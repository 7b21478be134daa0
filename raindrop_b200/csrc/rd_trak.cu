// TRAK (Park et al. 2023): the margin seed of the gradient rows, the fp64 Gram of a projected training set and the
// rotation of projected rows into its eigenbasis.
//   trak_margin_seed_kernel  one thread per sample: d_logits[b] = grad_logits m_b / B and Q[b] = sigmoid(-m_b) (fp64),
//                            m_b = z_y - log sum_{c != y} exp(z_c), the softmax over c != y taken against its own max.
//   trak_gram_kernel         one CTA per 64 x 64 tile (bi <= bj) of K = Phi^T Phi: 4 warps of 32 x 32, fp32 rows staged
//                            to shared memory as fp64 (exact), mma.sync m16n8k16 f64 (DMMA) over 32-row k-blocks in row
//                            order; the tile is staged through shared memory and added to K at (bi, bj) and mirrored to
//                            (bj, bi) (a diagonal tile takes its upper triangle on both sides), so K is exactly symmetric.
//   trak_rotate_kernel       one CTA per 64 rows x 64 output columns of Phi V, the same warp tiling over 32-column
//                            k-blocks of V in order; each element rounded to fp32 once.
// Products of fp32 inputs are exact in fp64, and every element's k-order is fixed by the shapes alone: no split-K, no
// atomics.  Rows past n are staged as zeros.  A rotated row depends on its own row of Phi and on V alone.
#include <math.h>

#include "rd_dmma.cuh"

namespace rd {
namespace {

// rows [r0, r0 + 32) x columns [c0, c0 + 64) of Phi (fp32, ld = dim) -> s[k][m] (fp64); rows >= n are 0
struct GramLoader {
  float4 v[4];
  __device__ __forceinline__ void load(const float* __restrict__ Phi, long long n, int dim, long long r0, int c0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int idx = threadIdx.x + TK_THREADS * q, row = idx >> 4, c4 = idx & 15;
      v[q] = r0 + row < n ? __ldg(reinterpret_cast<const float4*>(Phi + (r0 + row) * dim + c0) + c4)
                          : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __device__ __forceinline__ void store(double* s) const {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int idx = threadIdx.x + TK_THREADS * q, row = idx >> 4, c4 = idx & 15;
      double2* d = reinterpret_cast<double2*>(s + row * TK_LD + 4 * c4);
      d[0] = make_double2((double)v[q].x, (double)v[q].y);
      d[1] = make_double2((double)v[q].z, (double)v[q].w);
    }
  }
};

__global__ void __launch_bounds__(TK_THREADS)
trak_gram_kernel(const float* __restrict__ Phi, long long n, int dim, double* __restrict__ K) {
  extern __shared__ double tk_smem[];
  pdl_launch_dependents();
  // tile (bi, bj), bi <= bj, numbered row by row over the upper triangle
  const int T = dim / TK_TILE;
  int bi = 0, z = blockIdx.x;
  while (z >= T - bi) { z -= T - bi; ++bi; }
  const int bj = bi + z, i0 = bi * TK_TILE, j0 = bj * TK_TILE;
  pdl_wait();
  GramLoader la, lb;
  double acc[2][4][4];
  tk_mainloop(
      tk_smem, (int)((n + TK_BK - 1) / TK_BK),
      [&](int kb) {
        la.load(Phi, n, dim, (long long)kb * TK_BK, i0);
        lb.load(Phi, n, dim, (long long)kb * TK_BK, j0);
      },
      [&](double* s) {
        la.store(s);
        lb.store(s + TK_OPERAND);
      },
      acc);
  // stage the tile, then add it to K at (bi, bj) and its transpose at (bj, bi)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  double* tile = tk_smem;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = (warp & 1) * 32 + 16 * mi + g + 8 * (e >> 1), c = (warp >> 1) * 32 + 8 * ni + 2 * t + (e & 1);
        tile[m * TK_OUT_LD + c] = acc[mi][ni][e];
      }
  __syncthreads();
  for (int idx = threadIdx.x; idx < TK_TILE * TK_TILE; idx += TK_THREADS) {
    const int a = idx / TK_TILE, b = idx % TK_TILE;
    const double v = bi == bj ? tile[min(a, b) * TK_OUT_LD + max(a, b)] : tile[a * TK_OUT_LD + b];
    K[(long long)(i0 + a) * dim + j0 + b] += v;
  }
  if (bi != bj) {
    for (int idx = threadIdx.x; idx < TK_TILE * TK_TILE; idx += TK_THREADS) {
      const int b = idx / TK_TILE, a = idx % TK_TILE;
      K[(long long)(j0 + b) * dim + i0 + a] += tile[a * TK_OUT_LD + b];
    }
  }
}

__global__ void __launch_bounds__(TK_THREADS)
trak_rotate_kernel(const float* __restrict__ Phi, long long n, int dim, const double* __restrict__ V,
                   float* __restrict__ out) {
  extern __shared__ double tk_smem[];
  pdl_launch_dependents();
  const int j0 = blockIdx.x * TK_TILE;
  const long long r0 = (long long)blockIdx.y * TK_TILE;
  pdl_wait();
  float4 va[4];
  double2 vb[8];
  double acc[2][4][4];
  tk_mainloop(
      tk_smem, dim / TK_BK,
      [&](int kb) {
        const int k0 = kb * TK_BK;
        // A: rows [r0, r0 + 64) x columns [k0, k0 + 32) of Phi, consecutive lanes on consecutive rows
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = threadIdx.x + TK_THREADS * q, c4 = idx >> 6, row = idx & 63;
          va[q] = r0 + row < n ? __ldg(reinterpret_cast<const float4*>(Phi + (r0 + row) * dim + k0) + c4)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // B: rows [k0, k0 + 32) x columns [j0, j0 + 64) of V
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int idx = threadIdx.x + TK_THREADS * q, row = idx >> 5, c2 = idx & 31;
          vb[q] = __ldg(reinterpret_cast<const double2*>(V + (long long)(k0 + row) * dim + j0) + c2);
        }
      },
      [&](double* s) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = threadIdx.x + TK_THREADS * q, c4 = idx >> 6, row = idx & 63;
          s[(4 * c4 + 0) * TK_LD + row] = (double)va[q].x;
          s[(4 * c4 + 1) * TK_LD + row] = (double)va[q].y;
          s[(4 * c4 + 2) * TK_LD + row] = (double)va[q].z;
          s[(4 * c4 + 3) * TK_LD + row] = (double)va[q].w;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int idx = threadIdx.x + TK_THREADS * q, row = idx >> 5, c2 = idx & 31;
          reinterpret_cast<double2*>(s + TK_OPERAND + row * TK_LD)[c2] = vb[q];
        }
      },
      acc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + (warp & 1) * 32 + 16 * mi + g + 8 * h;
        const int c = j0 + (warp >> 1) * 32 + 8 * ni + 2 * t;
        if (r < n)
          *reinterpret_cast<float2*>(out + r * dim + c) = make_float2((float)acc[mi][ni][2 * h], (float)acc[mi][ni][2 * h + 1]);
      }
}

__global__ void trak_margin_seed_kernel(const float* __restrict__ logits, int B, int ncls, const int64_t* __restrict__ y,
                                        float* __restrict__ dlog, double* __restrict__ Q) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* l = logits + (long long)b * ncls;
  float* d = dlog + (long long)b * ncls;
  const long long yb = y[b];
  if (yb < 0 || yb >= ncls) {            // refused on the host; NaN marks it should it get here
    for (int c = 0; c < ncls; ++c) d[c] = __int_as_float(0x7fc00000);
    Q[b] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  double m = -INFINITY;
  for (int c = 0; c < ncls; ++c)
    if (c != yb) m = fmax(m, (double)l[c]);
  double s = 0.0;
  for (int c = 0; c < ncls; ++c)
    if (c != yb) s += exp((double)l[c] - m);
  const double margin = (double)l[yb] - (m + log(s)), inv_b = 1.0 / (double)B;
  for (int c = 0; c < ncls; ++c) d[c] = c == yb ? (float)inv_b : (float)(-exp((double)l[c] - m) / s * inv_b);
  // sigmoid(-margin) without cancellation on either side
  const double e = exp(-fabs(margin));
  Q[b] = margin > 0.0 ? e / (1.0 + e) : 1.0 / (1.0 + e);
}

bool trak_dim_ok(int32_t dim) { return dim >= 128 && dim <= RD_TRAK_DIM_MAX && dim % 128 == 0; }

}  // namespace
}  // namespace rd

using namespace rd;

extern "C" {

int rd_trak_margin_seed(const float* logits, int32_t B, int32_t n_classes, const int64_t* y, float* d_logits, double* Q,
                        void* stream) {
  if (!logits || !y || !d_logits || !Q || B < 0 || n_classes < 2) {
    set_error("rd_trak_margin_seed: bad arguments (B=%d n_classes=%d; the margin needs 2 classes or more)", B, n_classes);
    return -2;
  }
  if (B == 0) return 0;
  launch_pdl(trak_margin_seed_kernel, dim3((unsigned)ceil_div(B, 128)), dim3(128), 0, (cudaStream_t)stream, logits,
             (int)B, (int)n_classes, y, d_logits, Q);
  RD_CHECK_LAUNCH("trak_margin_seed_kernel");
  return 0;
}

int rd_trak_gram(const float* Phi, int64_t n, int32_t dim, double* K, void* stream) {
  const char* fn = "rd_trak_gram";
  if (!Phi || !K) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 0 || !trak_dim_ok(dim)) {
    set_error("%s: bad sizes (n=%lld dim=%d; dim must be a multiple of 128 in [128, %d])", fn, (long long)n, dim,
              RD_TRAK_DIM_MAX);
    return -2;
  }
  if (reinterpret_cast<uintptr_t>(Phi) & 15) { set_error("%s: Phi must be 16-byte aligned", fn); return -2; }
  if (n == 0) return 0;
  RD_TRY(tc::ensure_max_smem((const void*)trak_gram_kernel, TK_SMEM));
  const int T = dim / TK_TILE;
  launch_pdl(trak_gram_kernel, dim3((unsigned)(T * (T + 1) / 2)), dim3(TK_THREADS), TK_SMEM, (cudaStream_t)stream, Phi,
             (long long)n, (int)dim, K);
  RD_CHECK_LAUNCH("trak_gram_kernel");
  return 0;
}

int rd_trak_rotate(const float* Phi, int64_t n, int32_t dim, const double* V, float* out, void* stream) {
  const char* fn = "rd_trak_rotate";
  if (!Phi || !V || !out) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 0 || !trak_dim_ok(dim) || ceil_div(n, TK_TILE) > 65535) {
    set_error("%s: bad sizes (n=%lld dim=%d; dim must be a multiple of 128 in [128, %d], n at most %d)", fn,
              (long long)n, dim, RD_TRAK_DIM_MAX, 65535 * TK_TILE);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(Phi) | reinterpret_cast<uintptr_t>(V) | reinterpret_cast<uintptr_t>(out)) & 15) {
    set_error("%s: Phi, V and out must be 16-byte aligned", fn);
    return -2;
  }
  if (n == 0) return 0;
  RD_TRY(tc::ensure_max_smem((const void*)trak_rotate_kernel, TK_SMEM));
  launch_pdl(trak_rotate_kernel, dim3((unsigned)(dim / TK_TILE), (unsigned)ceil_div(n, TK_TILE)), dim3(TK_THREADS),
             TK_SMEM, (cudaStream_t)stream, Phi, (long long)n, (int)dim, V, out);
  RD_CHECK_LAUNCH("trak_rotate_kernel");
  return 0;
}

}  // extern "C"
