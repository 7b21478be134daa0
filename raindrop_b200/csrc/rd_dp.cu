// Differentially private training (DP-SGD) kernels: per-sample gradient norms, clipping, Gaussian noise.
//
// The per-sample norm pass runs the frozen-parameter backward (data gradients only) and, where the training path queues a
// weight-gradient item (dY, X), queues a per-sample norm item of the same operand pair instead.  The squared norm of
// sample b's gradient of a linear layer, weight [Nout, Kin] and bias [Nout], with the sample's R rows y_r, x_r, is
//   weight:  || sum_r y_r x_r^T ||_F^2            bias:  || sum_r y_r ||^2
// and comes in one of two forms, picked per item from the shape alone (dp_ghost):
//   ghost    sum_{r,r'} (y_r . y_r') (x_r . x_r')   and   sum_{r,r'} y_r . y_r'     R^2 (Nout + Kin + 1) MACs
//   explicit the sample's [Nout, Kin + 1] product (x extended by a column of ones), then its sum of squares
//                                                                                   R Nout (Kin + 1) MACs
// Both are 64 x 64 output tiles of a product staged through shared memory: Gram tiles of the R x R upper triangle (the
// off-diagonal ones count twice) or tiles of the [Nout, Kin + 1] product.  Each 16-deep slice of the contraction is
// summed in fp32 and added to fp64 accumulators; a CTA writes its tile's two sums (weight, bias) to a partial slot, and
// a second launch adds each (sample, tensor)'s slots in tile order.  No atomics: the result is bitwise reproducible and
// independent of anything but the shapes.
#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int DP_TILE = 64, DP_BK = 16, DP_THREADS = 256, DP_SMEM_LD = DP_TILE + 4;

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

// dst[k][m] = P[(m0 + m) * ms + k0 + k] for m0 + m < mlim, k0 + k < klim, else 0 (rows contiguous along k)
__device__ __forceinline__ void load_rows(float (*dst)[DP_SMEM_LD], const float* __restrict__ P, long long ms, int m0,
                                          int mlim, int k0, int klim) {
#pragma unroll
  for (int e = 0; e < DP_TILE * DP_BK / DP_THREADS; ++e) {
    const int idx = threadIdx.x + e * DP_THREADS, m = idx >> 4, k = idx & 15;
    dst[k][m] = (m0 + m < mlim && k0 + k < klim) ? __ldg(P + (long long)(m0 + m) * ms + k0 + k) : 0.f;
  }
}
// dst[k][n] = P[(k0 + k) * ks + n0 + n] for k0 + k < klim, n0 + n < nlim; a column of ones at n0 + n == ones_col
__device__ __forceinline__ void load_cols(float (*dst)[DP_SMEM_LD], const float* __restrict__ P, long long ks, int k0,
                                          int klim, int n0, int nlim, int ones_col) {
#pragma unroll
  for (int e = 0; e < DP_TILE * DP_BK / DP_THREADS; ++e) {
    const int idx = threadIdx.x + e * DP_THREADS, k = idx >> 6, n = idx & 63;
    float v = 0.f;
    if (k0 + k < klim) {
      if (n0 + n < nlim) v = __ldg(P + (long long)(k0 + k) * ks + n0 + n);
      else if (n0 + n == ones_col) v = 1.f;
    }
    dst[k][n] = v;
  }
}

__device__ __forceinline__ void mma_slice(const float (*As)[DP_SMEM_LD], const float (*Bs)[DP_SMEM_LD], double acc[4][4]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float c[4][4] = {};
#pragma unroll
  for (int k = 0; k < DP_BK; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
    const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) c[i][j] = fmaf(av[i], bv[j], c[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] += (double)c[i][j];
}

// acc = the [m0, m0+64) x [n0, n0+64) tile of the Gram matrix P P^T over the sample's R rows (row stride rs), width K
__device__ void gram_tile(float (*As)[DP_SMEM_LD], float (*Bs)[DP_SMEM_LD], const float* __restrict__ P, long long rs, int K,
                          int R, int m0, int n0, double acc[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < K; k0 += DP_BK) {
    __syncthreads();
    load_rows(As, P, rs, m0, R, k0, K);
    load_rows(Bs, P, rs, n0, R, k0, K);
    __syncthreads();
    mma_slice(As, Bs, acc);
  }
}

__global__ void __launch_bounds__(DP_THREADS) dp_norm_tile_kernel(const __grid_constant__ DpNormGroup g, double* __restrict__ partial) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) float As[DP_BK][DP_SMEM_LD];
  __shared__ __align__(16) float Bs[DP_BK][DP_SMEM_LD];
  __shared__ double red[DP_THREADS / 32];
  int ii = 0;
  for (int k = 1; k < g.n; ++k)
    if ((long long)blockIdx.x >= g.it[k].blk0) ii = k;
  const DpNormItem& o = g.it[ii];
  const long long local = (long long)blockIdx.x - o.blk0;
  const int b = (int)(local / o.ntiles), tile = (int)(local % o.ntiles);
  const float* Yb = o.Y + (long long)b * o.sstride * o.ldy;
  const float* Xb = o.X + (long long)b * o.sstride * o.ldx;
  const long long ys = o.rstride * o.ldy, xs = o.rstride * o.ldx;
  const int tx = threadIdx.x & 15;
  double pw = 0.0, pb = 0.0;
  if (o.ghost) {
    int i = 0, j = tile;                       // upper-triangle tile (i, j), i <= j, row by row
    while (j >= o.tm - i) { j -= o.tm - i; ++i; }
    j += i;
    double gy[4][4], gx[4][4];
    gram_tile(As, Bs, Yb, ys, o.Nout, o.R, i * DP_TILE, j * DP_TILE, gy);
    gram_tile(As, Bs, Xb, xs, o.Kin, o.R, i * DP_TILE, j * DP_TILE, gx);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) { pw += gy[u][v] * gx[u][v]; pb += gy[u][v]; }
    if (i != j) { pw *= 2.0; pb *= 2.0; }
  } else {
    const int m0 = (tile / o.tn) * DP_TILE, n0 = (tile % o.tn) * DP_TILE;
    double e[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) e[u][v] = 0.0;
    for (int r0 = 0; r0 < o.R; r0 += DP_BK) {
      __syncthreads();
      load_cols(As, Yb, ys, r0, o.R, m0, o.Nout, -1);
      load_cols(Bs, Xb, xs, r0, o.R, n0, o.Kin, o.Kin);
      __syncthreads();
      mma_slice(As, Bs, e);
    }
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int n = n0 + tx * 4 + v;
      double s = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u) s += e[u][v] * e[u][v];   // rows past Nout are 0
      if (n < o.Kin) pw += s;
      else if (n == o.Kin) pb += s;
    }
  }
  pw = block_sum_fixed(pw, red);
  pb = block_sum_fixed(pb, red);
  if (threadIdx.x == 0) {
    partial[2 * (long long)blockIdx.x] = pw;
    partial[2 * (long long)blockIdx.x + 1] = pb;
  }
}

// sqnorms[b, fw / fb] = the item's tile sums of sample b, in tile order; one thread per (item, sample)
__global__ void dp_norm_finalize_kernel(const __grid_constant__ DpNormGroup g, int B, const double* __restrict__ partial,
                                        double* __restrict__ sqn, int nf) {
  pdl_launch_dependents();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= g.n * B) return;
  const DpNormItem& o = g.it[idx / B];
  const int b = idx % B;
  const double* p = partial + 2 * (o.blk0 + (long long)b * o.ntiles);
  double w = 0.0, s = 0.0;
  for (int t = 0; t < o.ntiles; ++t) { w += p[2 * t]; s += p[2 * t + 1]; }
  sqn[(long long)b * nf + o.fw] = w;
  sqn[(long long)b * nf + o.fb] = s;
}

// LayerNorm gamma / beta of sample b: || sum_t dy (.) xhat ||^2 and || sum_t dy ||^2 over its rows r = t*B + b, xhat
// recomputed from the stored input and {mean, rstd}.  One CTA per sample, columns over the threads, rows in order.
__global__ void __launch_bounds__(DP_THREADS) dp_ln_sqnorm_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                                                  const float* __restrict__ dy, int T, int B, int D,
                                                                  double* __restrict__ sqn, int nf, int fw, int fb) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[DP_THREADS / 32];
  const int b = blockIdx.x;
  double sw = 0.0, sb = 0.0;
  for (int d = threadIdx.x; d < D; d += DP_THREADS) {
    double gw = 0.0, gb = 0.0;
    for (int t = 0; t < T; ++t) {
      const long long r = (long long)t * B + b;
      const float mean = stats[2 * r], rstd = stats[2 * r + 1];
      const float g = dy[r * D + d];
      gw += (double)(g * ((x[r * D + d] - mean) * rstd));
      gb += (double)g;
    }
    sw += gw * gw;
    sb += gb * gb;
  }
  sw = block_sum_fixed(sw, red);
  sb = block_sum_fixed(sb, red);
  if (threadIdx.x == 0) {
    sqn[(long long)b * nf + fw] = sw;
    sqn[(long long)b * nf + fb] = sb;
  }
}

__device__ double block_sqsum(const float* __restrict__ v, int n, double* red) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += DP_THREADS) s += (double)v[i] * (double)v[i];
  return block_sum_fixed(s, red);
}

// The head's layers see one row per sample: || a_b ||^2 (|| x_b ||^2 + 1) for mlp_static.2 (d_logits, h), mlp_static.0
// (dh, feat) and emb (dfeat[:, D:], static).  One CTA per sample.
__global__ void __launch_bounds__(DP_THREADS) dp_head_sqnorm_kernel(int D, int Df, int ds, int ncls, const float* __restrict__ dlogits,
                                                                    const float* __restrict__ hpre, const float* __restrict__ dh,
                                                                    const float* __restrict__ feat, const float* __restrict__ dfeat,
                                                                    const float* __restrict__ statics, double* __restrict__ sqn,
                                                                    int nf) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[DP_THREADS / 32];
  const int b = blockIdx.x;
  const long long rf = (long long)b * Df;
  const double a2 = block_sqsum(dlogits + (long long)b * ncls, ncls, red);
  const double h2 = block_sqsum(hpre + rf, Df, red);
  const double d2 = block_sqsum(dh + rf, Df, red);
  const double f2 = block_sqsum(feat + rf, Df, red);
  double e2 = 0.0, s2 = 0.0;
  if (ds > 0) {
    e2 = block_sqsum(dfeat + rf + D, Df - D, red);
    s2 = block_sqsum(statics + (long long)b * ds, ds, red);
  }
  if (threadIdx.x == 0) {
    double* o = sqn + (long long)b * nf;
    int f = 0;
    if (ds > 0) { o[f++] = e2 * s2; o[f++] = e2; }
    o[f++] = d2 * f2; o[f++] = d2;
    o[f++] = a2 * h2; o[f++] = a2;
  }
}

// n_b = B sqrt(sum_f sqnorms[b, f]) (the norms were taken of grad(loss_b / B)), c_b = min(1, C / (n_b + 1e-6)); d_logits
// row b *= w_b c_b B / L; clip[b] = c_b.  loss = sum_b w_b loss_b / sum_b w_b (0 for an empty batch), summed as the head
// kernel sums the batch-mean loss (lane-strided fp32 sums, then a butterfly), so with every weight 1 it is that loss
// bit for bit.  One CTA.
__global__ void __launch_bounds__(DP_THREADS) dp_clip_kernel(const double* __restrict__ sqn, int B, int nf, int ncls,
                                                             const float* __restrict__ weight, double max_norm, double L,
                                                             const float* __restrict__ loss_ps, float* __restrict__ dlogits,
                                                             float* __restrict__ clip, float* __restrict__ loss) {
  pdl_launch_dependents();
  pdl_wait();
  for (int b = threadIdx.x; b < B; b += DP_THREADS) {
    double s = 0.0;
    for (int f = 0; f < nf; ++f) s += sqn[(long long)b * nf + f];
    const double n = (double)B * sqrt(s);
    const double c = fmin(1.0, max_norm / (n + 1e-6));
    const float scale = (float)((double)weight[b] * c * (double)B / L);
    for (int k = 0; k < ncls; ++k) dlogits[(long long)b * ncls + k] *= scale;
    clip[b] = (float)c;
  }
  if (threadIdx.x < 32) {
    float s = 0.f, cnt = 0.f;
    for (int i = threadIdx.x; i < B; i += 32) { s += weight[i] * loss_ps[i]; cnt += weight[i]; }
    s = warp_sum(s);
    cnt = warp_sum(cnt);
    if (threadIdx.x == 0) *loss = cnt > 0.f ? s * (1.f / cnt) : 0.f;
  }
}

// g[i] += std * xi_i over the used elements of the bucket, xi_i = standard normal from Philox at key {seed, step}, site
// SITE_DP_NOISE, block i >> 2, Box-Muller on the block's word pairs (x, y) -> elements 4q, 4q+1 and (z, w) -> 4q+2, 4q+3:
//   u1 = ((w0 >> 8) + 1) 2^-24, u2 = (w1 >> 8) 2^-24, r = sqrt(-2 ln u1), (r cos(2 pi u2), r sin(2 pi u2)) in fp64,
// rounded to fp32.  key = {seed, step, ticket}: the last CTA to finish advances step (and resets the ticket).
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float* z0, float* z1) {
  const double u1 = ((double)(a >> 8) + 1.0) * (1.0 / 16777216.0), u2 = (double)(b >> 8) * (1.0 / 16777216.0);
  const double r = sqrt(-2.0 * log(u1)), t = 6.283185307179586 * u2;
  *z0 = (float)(r * cos(t));
  *z1 = (float)(r * sin(t));
}

__global__ void __launch_bounds__(DP_THREADS) dp_noise_kernel(float* __restrict__ g, long long n4, const __grid_constant__ DpFields fl,
                                                              float stdv, uint64_t* __restrict__ key) {
  pdl_launch_dependents();
  pdl_wait();
  const RngKey k = load_rng_key(key);
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  for (long long q = tid; q < n4; q += stride) {
    const long long i = 4 * q;
    int lo = 0, hi = fl.n - 1;                       // the field holding i: the last one with off <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (fl.off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    const long long end = fl.off[lo] + fl.numel[lo];
    if (i < fl.off[lo] || i >= end) continue;
    const uint4 w = dropout_block(k, SITE_DP_NOISE, (uint64_t)i);
    float z[4];
    box_muller(w.x, w.y, &z[0], &z[1]);
    box_muller(w.z, w.w, &z[2], &z[3]);
    float4 v = reinterpret_cast<float4*>(g)[q];
    v.x = fmaf(stdv, z[0], v.x);
    if (i + 1 < end) v.y = fmaf(stdv, z[1], v.y);
    if (i + 2 < end) v.z = fmaf(stdv, z[2], v.z);
    if (i + 3 < end) v.w = fmaf(stdv, z[3], v.w);
    reinterpret_cast<float4*>(g)[q] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned long long* ticket = reinterpret_cast<unsigned long long*>(key + 2);
    if (atomicAdd(ticket, 1ull) == (unsigned long long)(gridDim.x - 1)) {
      *ticket = 0ull;
      key[1] = key[1] + 1;
    }
  }
}

// ---- per-sample gradients, materialised ---------------------------------------------------------------------------
// The explicit form of dp_norm_tile_kernel, written out instead of squared: tile (m0, n0) of sample b's [Nout, Kin + 1]
// product dY_b^T [X_b | 1], 16-row fp32 slices summed in fp64, each value scaled and rounded to fp32 once.  kRotated
// (EK-FAC rows): X already holds Kin + 1 columns (the rotated [X | 1] Q_A), so no ones column is appended.
template <bool kRotated>
__global__ void __launch_bounds__(DP_THREADS) psg_tile_kernel(const __grid_constant__ PsgGroup g, float* __restrict__ G,
                                                              long long ldg, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) float As[DP_BK][DP_SMEM_LD];
  __shared__ __align__(16) float Bs[DP_BK][DP_SMEM_LD];
  int ii = 0;
  for (int k = 1; k < g.n; ++k)
    if ((long long)blockIdx.x >= g.it[k].blk0) ii = k;
  const PsgItem& o = g.it[ii];
  const long long local = (long long)blockIdx.x - o.blk0;
  const int b = (int)(local / o.ntiles), tile = (int)(local % o.ntiles);
  const float* Yb = o.Y + (long long)b * o.sstride * o.ldy;
  const float* Xb = o.X + (long long)b * o.sstride * o.ldx;
  const long long ys = o.rstride * o.ldy, xs = o.rstride * o.ldx;
  const int m0 = (tile / o.tn) * DP_TILE, n0 = (tile % o.tn) * DP_TILE;
  double e[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) e[u][v] = 0.0;
  for (int r0 = 0; r0 < o.R; r0 += DP_BK) {
    __syncthreads();
    load_cols(As, Yb, ys, r0, o.R, m0, o.Nout, -1);
    if (kRotated) load_cols(Bs, Xb, xs, r0, o.R, n0, o.Kin + 1, -1);
    else load_cols(Bs, Xb, xs, r0, o.R, n0, o.Kin, o.Kin);
    __syncthreads();
    mma_slice(As, Bs, e);
  }
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float* Gb = G + (long long)b * ldg;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int m = m0 + ty * 4 + u;
    if (m >= o.Nout) continue;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int n = n0 + tx * 4 + v;
      const float val = (float)(e[u][v] * (double)scale);
      if (n < o.Kin) Gb[o.gw + (long long)m * o.Kin + n] = val;
      else if (n == o.Kin) Gb[o.gb + m] = val;
    }
  }
}

// LayerNorm gamma / beta of sample b, written out (dp_ln_sqnorm_kernel's per-column sums)
__global__ void __launch_bounds__(DP_THREADS) psg_ln_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                                            const float* __restrict__ dy, int T, int B, int D,
                                                            float* __restrict__ G, long long ldg, long long gw, long long gb,
                                                            float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  float* Gb = G + (long long)b * ldg;
  for (int d = threadIdx.x; d < D; d += DP_THREADS) {
    double sw = 0.0, sb = 0.0;
    for (int t = 0; t < T; ++t) {
      const long long r = (long long)t * B + b;
      const float mean = stats[2 * r], rstd = stats[2 * r + 1];
      const float g = dy[r * D + d];
      sw += (double)(g * ((x[r * D + d] - mean) * rstd));
      sb += (double)g;
    }
    Gb[gw + d] = (float)(sw * (double)scale);
    Gb[gb + d] = (float)(sb * (double)scale);
  }
}

// a [n] (x) [x | 1] [m + 1] -> weight [n, m] at Gb + ow, bias [n] at Gb + ob; products in fp64, scaled, rounded once
__device__ void psg_outer(const float* __restrict__ a, int n, const float* __restrict__ x, int m, float* Gb, long long ow,
                          long long ob, double scale) {
  const long long nm = (long long)n * m;
  for (long long i = threadIdx.x; i < nm; i += DP_THREADS) {
    const int r = (int)(i / m), c = (int)(i - (long long)r * m);
    Gb[ow + i] = (float)((double)a[r] * (double)x[c] * scale);
  }
  for (int r = threadIdx.x; r < n; r += DP_THREADS) Gb[ob + r] = (float)((double)a[r] * scale);
}

// the head's one row per sample: mlp_static.2 (d_logits, h), mlp_static.0 (dh, feat), emb (dfeat[:, D:], static)
__global__ void __launch_bounds__(DP_THREADS) psg_head_kernel(int D, int Df, int ds, int ncls, const float* __restrict__ dlogits,
                                                              const float* __restrict__ hpre, const float* __restrict__ dh,
                                                              const float* __restrict__ feat, const float* __restrict__ dfeat,
                                                              const float* __restrict__ statics, float* __restrict__ G,
                                                              long long ldg, long long o0, long long o1, long long o2,
                                                              long long o3, long long o4, long long o5, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const long long rf = (long long)b * Df;
  float* Gb = G + (long long)b * ldg;
  if (ds > 0) psg_outer(dfeat + rf + D, Df - D, statics + (long long)b * ds, ds, Gb, o0, o1, scale);
  psg_outer(dh + rf, Df, feat + rf, Df, Gb, o2, o3, scale);
  psg_outer(dlogits + (long long)b * ncls, ncls, hpre + rf, Df, Gb, o4, o5, scale);
}

__global__ void psg_pad_kernel(const __grid_constant__ DpFields fl, int B, float* __restrict__ G, long long ldg) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)fl.n * B) return;
  const int f = (int)(idx % fl.n), b = (int)(idx / fl.n);
  const long long end = f + 1 < fl.n ? fl.off[f + 1] : ldg;
  float* Gb = G + (long long)b * ldg;
  for (long long i = fl.off[f] + fl.numel[f]; i < end; ++i) Gb[i] = 0.f;
}

}  // namespace

int psg_tiles(int Nout, int Kin, int* tn) {
  *tn = (int)ceil_div(Kin + 1, DP_TILE);
  return (int)ceil_div(Nout, DP_TILE) * *tn;
}

int psg_group(const PsgGroup& g, int B, float* G, long long ldg, float scale, cudaStream_t st, bool rotated) {
  if (g.n == 0) return 0;
  const PsgItem& last = g.it[g.n - 1];
  const long long blocks = last.blk0 + (long long)B * last.ntiles;
  if (blocks > 0x7FFFFFFFLL) { set_error("psg_group: %lld tiles, too many for one launch", blocks); return -2; }
  if (rotated) launch_pdl(psg_tile_kernel<true>, dim3((unsigned)blocks), dim3(DP_THREADS), 0, st, g, G, ldg, scale);
  else launch_pdl(psg_tile_kernel<false>, dim3((unsigned)blocks), dim3(DP_THREADS), 0, st, g, G, ldg, scale);
  RD_CHECK_LAUNCH("psg_tile_kernel");
  return 0;
}

int psg_ln(const float* x, const float* stats, const float* dy, int T, int B, int D, float* G, long long ldg, long long gw,
           long long gb, float scale, cudaStream_t st) {
  launch_pdl(psg_ln_kernel, dim3(B), dim3(DP_THREADS), 0, st, x, stats, dy, T, B, D, G, ldg, gw, gb, scale);
  RD_CHECK_LAUNCH("psg_ln_kernel");
  return 0;
}

int psg_head(int B, int D, int Df, int ds, int ncls, const float* dlogits, const float* hpre, const float* dh, const float* feat,
             const float* dfeat, const float* statics, float* G, long long ldg, const long long* off, float scale,
             cudaStream_t st) {
  const int h = ds > 0 ? 2 : 0;     // the first field past the static embedding
  const long long o0 = ds > 0 ? off[0] : 0, o1 = ds > 0 ? off[1] : 0;
  launch_pdl(psg_head_kernel, dim3(B), dim3(DP_THREADS), 0, st, D, Df, ds, ncls, dlogits, hpre, dh, feat, dfeat, statics, G,
             ldg, o0, o1, off[h], off[h + 1], off[h + 2], off[h + 3], scale);
  RD_CHECK_LAUNCH("psg_head_kernel");
  return 0;
}

int psg_pad(const DpFields& fields, int B, float* G, long long ldg, cudaStream_t st) {
  const long long n = (long long)fields.n * B;
  launch_pdl(psg_pad_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, fields, B, G, ldg);
  RD_CHECK_LAUNCH("psg_pad_kernel");
  return 0;
}

bool dp_ghost(int R, int Nout, int Kin) {
  return (int64_t)R * (Nout + Kin + 1) < (int64_t)Nout * (Kin + 1);
}

int dp_norm_tiles(int R, int Nout, int Kin, int* tm, int* tn) {
  if (dp_ghost(R, Nout, Kin)) {
    *tm = (int)ceil_div(R, DP_TILE); *tn = *tm;
    return *tm * (*tm + 1) / 2;
  }
  *tm = (int)ceil_div(Nout, DP_TILE); *tn = (int)ceil_div(Kin + 1, DP_TILE);
  return *tm * *tn;
}

int dp_norm_group(const DpNormGroup& g, int B, double* partial, double* sqnorms, int nf, cudaStream_t st) {
  if (g.n == 0) return 0;
  const DpNormItem& last = g.it[g.n - 1];
  const long long blocks = last.blk0 + (long long)B * last.ntiles;
  if (blocks > 0x7FFFFFFFLL) { set_error("dp_norm_group: %lld tiles, too many for one launch", blocks); return -2; }
  launch_pdl(dp_norm_tile_kernel, dim3((unsigned)blocks), dim3(DP_THREADS), 0, st, g, partial);
  RD_CHECK_LAUNCH("dp_norm_tile_kernel");
  const int n = g.n * B;
  launch_pdl(dp_norm_finalize_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, g, B, (const double*)partial, sqnorms, nf);
  RD_CHECK_LAUNCH("dp_norm_finalize_kernel");
  return 0;
}

int dp_ln_sqnorm(const float* x, const float* stats, const float* dy, int T, int B, int D, double* sqnorms, int nf, int fw,
                 int fb, cudaStream_t st) {
  launch_pdl(dp_ln_sqnorm_kernel, dim3(B), dim3(DP_THREADS), 0, st, x, stats, dy, T, B, D, sqnorms, nf, fw, fb);
  RD_CHECK_LAUNCH("dp_ln_sqnorm_kernel");
  return 0;
}

int dp_head_sqnorm(int B, int D, int Df, int ds, int ncls, const float* dlogits, const float* hpre, const float* dh,
                   const float* feat, const float* dfeat, const float* statics, double* sqnorms, int nf, cudaStream_t st) {
  launch_pdl(dp_head_sqnorm_kernel, dim3(B), dim3(DP_THREADS), 0, st, D, Df, ds, ncls, dlogits, hpre, dh, feat, dfeat, statics,
             sqnorms, nf);
  RD_CHECK_LAUNCH("dp_head_sqnorm_kernel");
  return 0;
}

int dp_clip(const double* sqnorms, int B, int nf, int ncls, const float* weight, double max_norm, double L,
            const float* loss_ps, float* dlogits, float* clip, float* loss, cudaStream_t st) {
  launch_pdl(dp_clip_kernel, dim3(1), dim3(DP_THREADS), 0, st, sqnorms, B, nf, ncls, weight, max_norm, L, loss_ps, dlogits,
             clip, loss);
  RD_CHECK_LAUNCH("dp_clip_kernel");
  return 0;
}

int dp_noise(float* g, int64_t n, const DpFields& fields, float stdv, uint64_t* key, cudaStream_t st) {
  const long long n4 = (long long)(n >> 2);
  long long blocks = ceil_div(n4, DP_THREADS);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  launch_pdl(dp_noise_kernel, dim3((unsigned)blocks), dim3(DP_THREADS), 0, st, g, n4, fields, stdv, key);
  RD_CHECK_LAUNCH("dp_noise_kernel");
  return 0;
}

}  // namespace rd
