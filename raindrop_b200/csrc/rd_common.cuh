// Shared device/host helpers for librd_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "raindrop_b200.h"

namespace rd {

// ---- error reporting across the C ABI (never throw) ---------------------------------------
void set_error(const char* fmt, ...);
const char* last_error();
unsigned long long launch_count();  // kernels launched by this library so far (host counter)
int check_launch(const char* what);  // cudaPeekAtLastError -> 0 / -1

#define RD_CHECK_LAUNCH(what)                    \
  do {                                           \
    if (rd::check_launch(what) != 0) return -1;  \
  } while (0)
#define RD_TRY(expr)             \
  do {                           \
    int _rc = (expr);            \
    if (_rc != 0) return _rc;    \
  } while (0)

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------
// A training step is ~40 dependent launches of 5-20 us each, so the ~2 us between "last CTA of kernel N exits" and
// "first CTA of kernel N+1 runs" is ~10 % of the step.  Kernels launched through launch_pdl() may be scheduled as soon
// as every CTA of the previous kernel has executed pdl_launch_dependents() (first instruction of our kernels): their
// CTAs take free SMs, run their prologue (barrier init, tensor-map prefetch) and then block in
// pdl_wait() until the previous kernel has COMPLETED and flushed its writes.  Every kernel calls pdl_wait() before its
// first global read of produced data and before its first global write, so the dependency semantics are unchanged.
// Stream capture records these as programmatic edges.  On by default; RD_PDL=0 turns it off (rd_kernels.cu).
bool pdl_enabled();
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// ---- dropout sites (ids are part of the debug ABI, see DESIGN.md) ---------------------------
enum DropSite : uint32_t {
  SITE_LIFT = 1,          // dropout on relu(src*R_u)          code/models_rd.py:296, index in [T,B,4N]
  SITE_ATTN = 16,         // + layer: attention probabilities  index in [B,H,T,T]
  SITE_RESID1 = 32,       // + layer: dropout1(out_proj)       index in [T*B, D]
  SITE_FFN = 48,          // + layer: dropout(relu(linear1))   index in [T*B, nhid]
  SITE_RESID2 = 64,       // + layer: dropout2(linear2)        index in [T*B, D]
};

// ---- Philox4x32-10, counter based: (seed, step) x (site, element index) ---------------------
__device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) { return __umulhi(a, b); }

__device__ __forceinline__ uint4 philox4(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = mulhi32(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = mulhi32(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  return make_uint4(c0, c1, c2, c3);
}

// One Philox block serves FOUR consecutive element indices: element idx uses word (idx & 3) of the block
// with counter idx >> 2.  rng[0] = seed, rng[1] = step counter captured by the forward.
__device__ __forceinline__ uint4 dropout_block(const uint64_t* __restrict__ rng, uint32_t site, uint64_t idx) {
  const uint64_t seed = rng[0], step = rng[1], blk = idx >> 2;
  return philox4((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)blk, (uint32_t)(blk >> 32),
                 site, (uint32_t)step);
}
__device__ __forceinline__ float keep_scale(uint32_t word, float p, float inv_keep) {
  return (float)(word >> 8) * (1.0f / 16777216.0f) >= p ? inv_keep : 0.0f;
}
// Returns 0 or 1/(1-p) for element idx.
__device__ __forceinline__ float dropout_scale(const uint64_t* __restrict__ rng, uint32_t site, uint64_t idx, float p,
                                               float inv_keep) {
  const uint4 b = dropout_block(rng, site, idx);
  const uint32_t sel = (uint32_t)idx & 3u;
  const uint32_t w = sel == 0 ? b.x : (sel == 1 ? b.y : (sel == 2 ? b.z : b.w));
  return keep_scale(w, p, inv_keep);
}
// Four consecutive elements idx .. idx+3 (idx % 4 == 0) from one Philox block.
__device__ __forceinline__ float4 dropout_scale4(const uint64_t* __restrict__ rng, uint32_t site, uint64_t idx, float p,
                                                 float inv_keep) {
  const uint4 b = dropout_block(rng, site, idx);
  return make_float4(keep_scale(b.x, p, inv_keep), keep_scale(b.y, p, inv_keep), keep_scale(b.z, p, inv_keep),
                     keep_scale(b.w, p, inv_keep));
}

// The same stream with the key held in registers: kernels that draw many blocks read (seed, step) from global memory
// ONCE per thread -- a load inside every call is an L2 round trip on the critical path whenever the compiler cannot
// hoist it (any "memory" clobber in between), which cost the attention kernels 2 us per CTA.
struct RngKey { uint32_t k0, k1, c3; };
__device__ __forceinline__ RngKey load_rng_key(const uint64_t* __restrict__ rng) {
  RngKey k{0u, 0u, 0u};
  if (rng) {
    const uint64_t seed = rng[0], step = rng[1];
    k.k0 = (uint32_t)seed; k.k1 = (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32); k.c3 = (uint32_t)step;
  }
  return k;
}
__device__ __forceinline__ uint4 dropout_block(const RngKey& k, uint32_t site, uint64_t idx) {
  const uint64_t blk = idx >> 2;
  return philox4(k.k0, k.k1, (uint32_t)blk, (uint32_t)(blk >> 32), site, k.c3);
}
__device__ __forceinline__ float dropout_scale(const RngKey& k, uint32_t site, uint64_t idx, float p, float inv_keep) {
  const uint4 b = dropout_block(k, site, idx);
  const uint32_t sel = (uint32_t)idx & 3u;
  const uint32_t w = sel == 0 ? b.x : (sel == 1 ? b.y : (sel == 2 ? b.z : b.w));
  return keep_scale(w, p, inv_keep);
}
__device__ __forceinline__ float4 dropout_scale4(const RngKey& k, uint32_t site, uint64_t idx, float p, float inv_keep) {
  const uint4 b = dropout_block(k, site, idx);
  return make_float4(keep_scale(b.x, p, inv_keep), keep_scale(b.y, p, inv_keep), keep_scale(b.z, p, inv_keep),
                     keep_scale(b.w, p, inv_keep));
}

// Two standard normals from two Philox words: u1 = ((a >> 8) + 1) 2^-24, u2 = (b >> 8) 2^-24, r = sqrt(-2 ln u1),
// (r cos(2 pi u2), r sin(2 pi u2)) in fp64, rounded to fp32.
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float* z0, float* z1) {
  const double u1 = ((double)(a >> 8) + 1.0) * (1.0 / 16777216.0), u2 = (double)(b >> 8) * (1.0 / 16777216.0);
  const double r = sqrt(-2.0 * log(u1)), t = 6.283185307179586 * u2;
  *z0 = (float)(r * cos(t));
  *z1 = (float)(r * sin(t));
}
// Standard normal of element idx at `site`: Box-Muller on the pair (x, y) of the block at counter idx >> 2 for
// idx & 3 in {0, 1}, (z, w) for {2, 3}; even idx takes the cosine, odd idx the sine (as rd_dp_add_noise draws them).
__device__ __forceinline__ float philox_normal(const RngKey& k, uint32_t site, uint64_t idx) {
  const uint4 w = dropout_block(k, site, idx);
  float z0, z1;
  if ((idx & 3u) < 2u) box_muller(w.x, w.y, &z0, &z1);
  else box_muller(w.z, w.w, &z0, &z1);
  return (idx & 1u) ? z1 : z0;
}

// ---- Monte Carlo dropout replicates in one forward ------------------------------------------------------------------
// A forward over Bc = cc*B rows, replicate-major (row j = m*B + b), in which row j draws exactly the words that the
// B-row forward at step (step + m) draws for row b.  Every site's index space is [T, Bc, width] (attention: T = 1,
// width = H*T*T), and rep_remap turns element `col` of row r = t*Bc + j into the key of step + m and the B-row index
// (t*B + b)*width + col.  A 4-word draw stays valid where width % 4 == 0 and col % 4 == 0 (the row maps to a row of the
// same width).  B == 0: off, every kernel draws as before.
struct DropRep { int B = 0, Bc = 0; };
__device__ __forceinline__ uint64_t rep_remap(const uint64_t* __restrict__ rng, const DropRep& rep, uint32_t r,
                                              uint64_t width, uint64_t col, RngKey* key) {
  const uint32_t t = r / (uint32_t)rep.Bc, j = r - t * (uint32_t)rep.Bc;
  const uint32_t m = j / (uint32_t)rep.B, b = j - m * (uint32_t)rep.B;
  const uint64_t seed = rng[0], step = rng[1] + m;
  *key = RngKey{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  return ((uint64_t)t * (uint32_t)rep.B + b) * width + col;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Sum of v over the CTA in a fixed order (butterfly within each warp, then the warps in order): deterministic.  red holds
// blockDim.x / 32 doubles; every thread returns the sum.
__device__ __forceinline__ double block_sum_fixed(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < nw; ++w) s += red[w];
  return s;
}

// ---- generic fp32 GEMM with a fused epilogue (rd_gemm.cu) ------------------------------------
// C(i,j) = epi( alpha * sum_k A(i,k) * B(k,j) ).  Element strides; exactly one of (sAi, sAk) and
// one of (sBk, sBj) must be 1 (ta / tb say which).  Batched over z = zo * nz_inner + zi.
struct GemmP {
  const float* A = nullptr; const float* B = nullptr; float* C = nullptr;
  int M = 0, N = 0, K = 0;
  int ta = 0;  // 0: A(i,k) = A[i*sAi + k]      1: A(i,k) = A[k*sAk + i]
  int tb = 0;  // 0: B(k,j) = B[k*sBk + j]      1: B(k,j) = B[j*sBj + k]
  long long sAi = 0, sAk = 0, sBk = 0, sBj = 0, sCi = 0, sCj = 1;
  int nz = 1, nz_inner = 1;
  long long sAzo = 0, sAzi = 0, sBzo = 0, sBzi = 0, sCzo = 0, sCzi = 0;
  // split-K (only for nz == 1): partial sums go to `partial` [nsplit][M][N], then reduced
  int nsplit = 1; float* partial = nullptr;
  float* asum = nullptr;   // optional extra output: asum[i] = sum_k A(i,k)  (bias gradient of a TN weight-grad GEMM)
  // epilogue, applied in this order
  float alpha = 1.f;
  const float* bias = nullptr;                         // + bias[j]
  int relu = 0;                                        // max(.,0)
  const float* rowscale = nullptr; int rowscale_mod = 1;  // * rowscale[i % mod]
  const float* gate = nullptr; long long gate_ld = 0; float gate_scale = 1.f;  // * (gate[i,j] > 0 ? gate_scale : 0)
  float drop_p = 0.f; const uint64_t* rng = nullptr; uint32_t drop_site = 0;   // dropout, index i*N + j
  DropRep rep;                                           // replicate rows (i = t*Bc + j): see rep_remap
  uint32_t* drop_mask = nullptr; int drop_mask_ld = 0;   // optional keep bits out: word [i*ld + j/32], bit j%32 (tensor-core path only)
  const float* resid = nullptr; long long resid_ld = 0;  // + resid[i*ld + j]
  // permuted store of the ob-prop output into the encoder input (code/models_rd.py:338-341):
  // row i = b*N + n, col j = t*d_ob + k  ->  C[((t*B + b)*D) + n*d_ob + k]
  int perm = 0, pB = 0, pN = 0, pdob = 0, pD = 0;
};
int gemm(const GemmP& p, cudaStream_t st);
// out[n] (+)= sum_s partial[s*n_elems + n]
int reduce_partials(const float* partial, int nsplit, int64_t n_elems, float* out, cudaStream_t st);
// same over a [nsplit][n1 + n2] buffer with two destinations
int reduce_partials2(const float* partial, int nsplit, int64_t n1, float* out1, int64_t n2, float* out2, cudaStream_t st);
// out[j] = sum_i x[i*ld + j], i < rows, j < cols; scratch >= colsum_scratch_floats(rows, cols)
int64_t colsum_scratch_floats(int64_t rows, int cols);
int colsum(const float* x, int64_t rows, int cols, int64_t ld, float* out, float* scratch, cudaStream_t st);
int64_t gemm_splitk_plan(int M, int N, int K, int* nsplit);  // returns partial floats needed

}  // namespace rd
