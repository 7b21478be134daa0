// Generic strided/batched fp32 GEMM (CUDA cores) with a fused epilogue, plus the small reductions
// that go with it (split-K reduce, column sums).  Used for every contraction whose accuracy budget
// rules out single-pass TF32 (temporal attention, head) and for the weight-gradient reductions;
// the observation-propagation forward has its own tensor-core kernel (rd_obprop_tc.cu).
#include "rd_common.cuh"

namespace rd {

namespace {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;
constexpr int LDS_A = BM + 4, LDS_B = BN + 4;

__device__ __forceinline__ void epilogue_store(const GemmP& p, float* __restrict__ C, int i, int j,
                                               float v) {
  v *= p.alpha;
  if (p.bias) v += __ldg(p.bias + j);
  if (p.relu) v = fmaxf(v, 0.f);
  if (p.rowscale) v *= __ldg(p.rowscale + (i % p.rowscale_mod));
  if (p.gate) v *= (__ldg(p.gate + (long long)i * p.gate_ld + j) > 0.f) ? p.gate_scale : 0.f;
  if (p.drop_p > 0.f) {
    if (p.rep.B) {
      RngKey key;
      const uint64_t idx = rep_remap(p.rng, p.rep, (uint32_t)i, (uint64_t)p.N, (uint64_t)j, &key);
      v *= dropout_scale(key, p.drop_site, idx, p.drop_p, 1.f / (1.f - p.drop_p));
    } else {
      v *= dropout_scale(p.rng, p.drop_site, (uint64_t)i * (uint64_t)p.N + (uint64_t)j, p.drop_p,
                         1.f / (1.f - p.drop_p));
    }
  }
  if (p.resid) v += __ldg(p.resid + (long long)i * p.resid_ld + j);
  if (p.perm) {
    int b = i / p.pN, n = i - b * p.pN;
    int t = j / p.pdob, k = j - t * p.pdob;
    C[((long long)t * p.pB + b) * p.pD + n * p.pdob + k] = v;
  } else {
    C[(long long)i * p.sCi + (long long)j * p.sCj] = v;
  }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(NT) gemm_f32_kernel(GemmP p) {
  __shared__ __align__(16) float As[2][BK][LDS_A];
  __shared__ __align__(16) float Bs[2][BK][LDS_B];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  int z = blockIdx.z;
  int split = 0;
  if (p.nsplit > 1) { split = z; z = 0; }
  const int zo = z / p.nz_inner, zi = z - zo * p.nz_inner;
  const float* __restrict__ A = p.A + zo * p.sAzo + zi * p.sAzi;
  const float* __restrict__ B = p.B + zo * p.sBzo + zi * p.sBzi;
  const int i0 = blockIdx.x * BM, j0 = blockIdx.y * BN;
  int kbeg = 0, kend = p.K;
  if (p.nsplit > 1) {
    int chunk = ((p.K + p.nsplit - 1) / p.nsplit + BK - 1) / BK * BK;
    kbeg = split * chunk;
    kend = min(p.K, kbeg + chunk);
  }

  float ra[4], rb[4];
  auto load_tiles = [&](int kb) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int i, k;
      if (!TA) { i = (tid >> 4) + 16 * r; k = tid & 15; } else { k = (tid >> 6) + 4 * r; i = tid & 63; }
      int gi = i0 + i, gk = kb + k;
      float v = 0.f;
      if (gi < p.M && gk < kend) v = TA ? __ldg(A + (long long)gk * p.sAk + gi) : __ldg(A + (long long)gi * p.sAi + gk);
      ra[r] = v;
      int j, k2;
      if (!TB) { k2 = (tid >> 6) + 4 * r; j = tid & 63; } else { j = (tid >> 4) + 16 * r; k2 = tid & 15; }
      int gj = j0 + j, gk2 = kb + k2;
      float w = 0.f;
      if (gj < p.N && gk2 < kend) w = TB ? __ldg(B + (long long)gj * p.sBj + gk2) : __ldg(B + (long long)gk2 * p.sBk + gj);
      rb[r] = w;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int i, k;
      if (!TA) { i = (tid >> 4) + 16 * r; k = tid & 15; } else { k = (tid >> 6) + 4 * r; i = tid & 63; }
      As[buf][k][i] = ra[r];
      int j, k2;
      if (!TB) { k2 = (tid >> 6) + 4 * r; j = tid & 63; } else { j = (tid >> 4) + 16 * r; k2 = tid & 15; }
      Bs[buf][k2][j] = rb[r];
    }
  };

  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  // optional: asum[i] = sum_k A(i,k) (the bias gradient rides along with the weight-gradient GEMM)
  const bool do_asum = p.asum != nullptr && blockIdx.y == 0;
  float asum_acc[4] = {0.f, 0.f, 0.f, 0.f};

  int buf = 0;
  if (kbeg < kend) {
    load_tiles(kbeg);
    store_tiles(0);
  }
  __syncthreads();
  for (int kb = kbeg; kb < kend; kb += BK) {
    const bool more = kb + BK < kend;
    if (more) load_tiles(kb + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
      if (do_asum) {
#pragma unroll
        for (int r = 0; r < 4; ++r) asum_acc[r] += av[r];
      }
    }
    if (more) {
      store_tiles(buf ^ 1);
      __syncthreads();
      buf ^= 1;
    }
  }

  if (p.nsplit > 1) {
    const long long per_split = (long long)p.M * p.N + (p.asum ? p.M : 0);
    float* __restrict__ P = p.partial + (long long)split * per_split;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int i = i0 + ty * 4 + r;
      if (i >= p.M) continue;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        int j = j0 + tx * 4 + c;
        if (j < p.N) P[(long long)i * p.N + j] = acc[r][c] * p.alpha;
      }
      if (do_asum && tx == 0) P[(long long)p.M * p.N + i] = asum_acc[r];
    }
    return;
  }
  if (do_asum && tx == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
      if (i0 + ty * 4 + r < p.M) p.asum[i0 + ty * 4 + r] = asum_acc[r];
  }
  float* __restrict__ C = p.C + zo * p.sCzo + zi * p.sCzi;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int i = i0 + ty * 4 + r;
    if (i >= p.M) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      int j = j0 + tx * 4 + c;
      if (j < p.N) epilogue_store(p, C, i, j, acc[r][c]);
    }
  }
}

__global__ void reduce_partials_kernel(const float* __restrict__ partial, int nsplit, long long n, long long n1,
                                       float* __restrict__ out, float* __restrict__ out2) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int k = 0; k < nsplit; ++k) s += partial[(long long)k * n + i];  // fixed order: deterministic
  if (i < n1) out[i] = s; else out2[i - n1] = s;
}

constexpr int CS_ROWS = 32;  // rows per colsum chunk

__global__ void colsum_partial_kernel(const float* __restrict__ x, long long rows, int cols,
                                      long long ld, float* __restrict__ partial) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cols) return;
  long long r0 = (long long)blockIdx.y * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
  float s = 0.f;
  for (long long r = r0; r < r1; ++r) s += x[r * ld + j];
  partial[(long long)blockIdx.y * cols + j] = s;
}

}  // namespace

int64_t gemm_splitk_plan(int M, int N, int K, int* nsplit) {
  int64_t tiles = ceil_div(M, BM) * ceil_div(N, BN);
  int ns = (int)ceil_div(2 * 132, tiles);   // two CTAs per SM of an H100
  int maxs = (int)ceil_div(K, 4 * BK);  // at least 64 reduction steps per split
  if (ns > maxs) ns = maxs;
  if (ns > 256) ns = 256;
  if (ns < 1) ns = 1;
  // make sure no split is empty
  while (ns > 1) {
    int chunk = (int)round_up(ceil_div(K, ns), BK);
    if ((int64_t)(ns - 1) * chunk < K) break;
    --ns;
  }
  *nsplit = ns;
  return ns > 1 ? (int64_t)ns * ((int64_t)M * N + M) : 0;   // room for the fused A-column-sums too
}

int gemm(const GemmP& p, cudaStream_t st) {
  if (p.M <= 0 || p.N <= 0) return 0;
  if (p.nsplit > 1 && (p.nz != 1 || p.partial == nullptr)) {
    set_error("gemm: split-K needs nz == 1 and a partial buffer");
    return -2;
  }
  // the split kernel stores alpha-scaled partial sums and reduce_partials2 writes their sum to C[i*N + j]: no other
  // epilogue step runs, so a split-K call that asks for one (or for other C strides) would silently lose it
  if (p.nsplit > 1 && (p.bias || p.relu || p.rowscale || p.gate || p.drop_p > 0.f || p.resid || p.perm)) {
    set_error("gemm: split-K applies alpha only (bias, relu, rowscale, gate, dropout, resid and perm need nsplit == 1)");
    return -2;
  }
  if (p.nsplit > 1 && (p.sCi != p.N || p.sCj != 1)) {
    set_error("gemm: split-K stores C contiguously (sCi = N, sCj = 1), got sCi=%lld sCj=%lld", p.sCi, p.sCj);
    return -2;
  }
  if ((p.rowscale && p.rowscale_mod < 1) || (p.drop_p > 0.f && !p.rng) || (p.drop_p > 0.f && p.rep.B && p.rep.Bc < 1) ||
      (p.perm && (p.pB < 1 || p.pN < 1 || p.pdob < 1 || p.pD < 1))) {
    set_error("gemm: bad epilogue (rowscale_mod=%d, dropout without rng, replicate rows Bc=%d or perm sizes)", p.rowscale_mod,
              p.rep.Bc);
    return -2;
  }
  dim3 grid((unsigned)ceil_div(p.M, BM), (unsigned)ceil_div(p.N, BN), (unsigned)(p.nsplit > 1 ? p.nsplit : p.nz));
  if (grid.y > 65535 || grid.z > 65535) {
    set_error("gemm: grid too large (N tiles %u, z %u)", grid.y, grid.z);
    return -2;
  }
  if (p.ta) {
    if (p.tb) gemm_f32_kernel<true, true><<<grid, NT, 0, st>>>(p);
    else gemm_f32_kernel<true, false><<<grid, NT, 0, st>>>(p);
  } else {
    if (p.tb) gemm_f32_kernel<false, true><<<grid, NT, 0, st>>>(p);
    else gemm_f32_kernel<false, false><<<grid, NT, 0, st>>>(p);
  }
  RD_CHECK_LAUNCH("gemm_f32_kernel");
  if (p.nsplit > 1)
    return reduce_partials2(p.partial, p.nsplit, (int64_t)p.M * p.N, p.C, p.asum ? p.M : 0, p.asum, st);
  return 0;
}

int reduce_partials2(const float* partial, int nsplit, int64_t n1, float* out1, int64_t n2, float* out2,
                     cudaStream_t st) {
  int64_t n = n1 + n2;
  if (n <= 0) return 0;
  reduce_partials_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(partial, nsplit, n, n1, out1, out2);
  RD_CHECK_LAUNCH("reduce_partials_kernel");
  return 0;
}

int reduce_partials(const float* partial, int nsplit, int64_t n, float* out, cudaStream_t st) {
  return reduce_partials2(partial, nsplit, n, out, 0, nullptr, st);
}

int64_t colsum_scratch_floats(int64_t rows, int cols) { return ceil_div(rows, CS_ROWS) * cols; }

int colsum(const float* x, int64_t rows, int cols, int64_t ld, float* out, float* scratch, cudaStream_t st) {
  if (cols <= 0) return 0;
  int chunks = (int)ceil_div(rows, CS_ROWS);
  dim3 grid((unsigned)ceil_div(cols, 128), (unsigned)chunks);
  if (chunks > 65535) { set_error("colsum: too many row chunks"); return -2; }
  colsum_partial_kernel<<<grid, 128, 0, st>>>(x, rows, cols, ld, scratch);
  RD_CHECK_LAUNCH("colsum_partial_kernel");
  return reduce_partials(scratch, chunks, cols, out, st);
}

}  // namespace rd
