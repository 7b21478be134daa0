// Worst-case sensor removal of Raindrop_v2 (rd_raindrop_v2_sensor_attack): the keep table of a beam round and the
// per-sample selection that run around each chunk's eval forward (rd_model.cu orchestrates them; ablate_expand writes
// the removed copies from the keep table, and exhaustive rounds take their keep rows from ablate_inputs' unranking).
//
// Score of a row with logits z against the reference class y (untargeted) or t (targeted): s = z_y - max_{c != y} z_c,
// resp. max_{c != t} z_c - z_t, in fp32; a row with a non-finite logit has s = +inf and never succeeds.  It succeeds
// when the first argmax of z is not y, resp. is t.  Candidates are ordered by (s, sorted tuple of removed players);
// within a round every set has the same size, so the tuples compare by the smallest player in which the two sets
// differ: the set that removes it is the smaller.  A keep row holds 1 for a kept player and 0 for a removed one.
//
// Per sample and round, fixed order and no atomics: the best and the best successful candidate (with their logits)
// and, in beam rounds, the list of the wsel smallest distinct candidates, built by wsel block-wide minimum searches
// over the old list and the chunk's rows, each for the smallest item strictly above the previous pick.  Equal sets
// evaluate to equal logits (every row is computed alike), so a duplicate ties its twin and is skipped.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int KEEP_TPB = 128, SELECT_TPB = 256;

// one thread per row j = m*B + b of the chunk
__global__ void __launch_bounds__(KEEP_TPB) sa_keep_kernel(const __grid_constant__ SaKeepArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)a.B * a.nc) return;
  const int m = (int)(j / a.B), b = (int)(j - (long long)m * a.B), P = a.P;
  const long long slot = a.s0 + m;
  const int w = (int)(slot / P), p = (int)(slot - (long long)w * P);
  uint8_t* out = a.keep + j * P;
  for (int q = 0; q < P; ++q) out[q] = 1;
  bool ok = w < a.beam_n[b];
  if (ok) {
    const int16_t* s = a.beam + ((long long)b * a.W + w) * a.R;
    for (int i = 0; i < a.r - 1; ++i) {
      out[s[i]] = 0;
      ok = ok && s[i] != p;
    }
  }
  out[p] = 0;
  a.valid[j] = ok ? 1 : 0;
}

struct Item { float s; const uint8_t* k; };

__device__ __forceinline__ bool item_less(const Item& x, const Item& y, int P) {
  if (x.s != y.s) return x.s < y.s;
  for (int p = 0; p < P; ++p) {
    if (x.k[p] != y.k[p]) return x.k[p] == 0;
  }
  return false;
}

__device__ __forceinline__ void row_score(const float* z, int C, int y, int targeted, float* s, bool* succ) {
  bool fin = true;
  float top = z[0], other = -INFINITY;
  int arg = 0;
  for (int c = 0; c < C; ++c) {
    const float v = z[c];
    fin = fin && isfinite(v);
    if (v > top) { top = v; arg = c; }
    if (c != y) other = fmaxf(other, v);
  }
  if (!fin) { *s = INFINITY; *succ = false; return; }
  *s = targeted ? other - z[y] : z[y] - other;
  *succ = targeted ? arg == y : arg != y;
}

// The smallest item of the threads' picks (-1: none), on every thread.
template <class F>
__device__ int block_min(int mine, const F& item, int P, int* red) {
  const int tid = threadIdx.x;
  red[tid] = mine;
  __syncthreads();
  for (int h = SELECT_TPB / 2; h > 0; h >>= 1) {
    if (tid < h) {
      const int x = red[tid], y = red[tid + h];
      if (y >= 0 && (x < 0 || item_less(item(y), item(x), P))) red[tid] = y;
    }
    __syncthreads();
  }
  const int r = red[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(SELECT_TPB) sa_select_kernel(const __grid_constant__ SaSelectArgs a) {
  __shared__ int red[SELECT_TPB];
  __shared__ int take[2];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x, B = a.B, C = a.C, P = a.P, W = a.W;
  if (a.r == 0) {                        // the clean row (nc = 1): the reference class and the clean logits
    const float* z = a.logits + (long long)b * C;
    if (tid == 0) {
      int y = 0;
      if (a.cls) {
        y = (int)a.cls[b];
      } else {
        float top = z[0];
        for (int c = 1; c < C; ++c) if (z[c] > top) { top = z[c]; y = c; }
      }
      a.yref[b] = y;
      a.done[b] = 0;
    }
    for (int c = tid; c < C; c += SELECT_TPB) a.clean_logits[(long long)b * C + c] = z[c];
    __syncthreads();
  }
  const int y = a.yref[b];
  float* cs = a.cscore + (long long)b * a.cc;
  uint8_t* cu = a.csucc + (long long)b * a.cc;
  auto valid = [&](int m) { return !a.valid || a.valid[(long long)m * B + b]; };
  auto cand = [&](int m) { return Item{cs[m], a.keep + ((long long)m * B + b) * P}; };

  // scores, and this chunk's best and best successful candidate
  int bi = -1, si = -1;
  for (int m = tid; m < a.nc; m += SELECT_TPB) {
    if (!valid(m)) continue;
    float s;
    bool ok;
    row_score(a.logits + ((long long)m * B + b) * C, C, y, a.targeted, &s, &ok);
    cs[m] = s;
    cu[m] = ok ? 1 : 0;
    if (bi < 0 || item_less(cand(m), cand(bi), P)) bi = m;
    if (ok && (si < 0 || item_less(cand(m), cand(si), P))) si = m;
  }
  const int win[2] = {block_min(bi, cand, P, red), block_min(si, cand, P, red)};
  if (tid == 0) {
    for (int t = 0; t < 2; ++t) {
      const long long o = (long long)t * B + b;
      const bool held = !a.first && a.trk_ok[o];
      take[t] = win[t] >= 0 && (!held || item_less(cand(win[t]), Item{a.trk_score[o], a.trk_keep + o * P}, P));
      if (a.first && !take[t]) a.trk_ok[o] = 0;
    }
  }
  __syncthreads();
  for (int t = 0; t < 2; ++t) {
    if (!take[t]) continue;
    const long long o = (long long)t * B + b, j = (long long)win[t] * B + b;
    for (int p = tid; p < P; p += SELECT_TPB) a.trk_keep[o * P + p] = a.keep[j * P + p];
    for (int c = tid; c < C; c += SELECT_TPB) a.trk_logits[o * C + c] = a.logits[j * C + c];
    if (tid == 0) { a.trk_score[o] = cs[win[t]]; a.trk_ok[o] = 1; }
  }

  // the list: the wsel smallest distinct items of the old list (items 0 .. n_old-1) and the chunk (n_old + m)
  int n_new = 0;
  if (a.wsel > 0) {
    const long long oc = (long long)a.cur * B + b, on = (long long)(a.cur ^ 1) * B + b;
    const int n_old = a.first ? 0 : a.top_n[oc];
    const float* os = a.top_score + oc * W;
    const uint8_t* ok = a.top_keep + oc * W * P;
    float* ns = a.top_score + on * W;
    uint8_t* nk = a.top_keep + on * W * P;
    auto item = [&](int i) { return i < n_old ? Item{os[i], ok + (long long)i * P} : cand(i - n_old); };
    __syncthreads();
    int last = -1;
    for (; n_new < a.wsel; ++n_new) {
      int mine = -1;
      for (int i = tid; i < n_old + a.nc; i += SELECT_TPB) {
        if (i >= n_old && !valid(i - n_old)) continue;
        const Item it = item(i);
        if (last >= 0 && !item_less(item(last), it, P)) continue;
        if (mine < 0 || item_less(it, item(mine), P)) mine = i;
      }
      const int got = block_min(mine, item, P, red);
      if (got < 0) break;
      const Item it = item(got);
      for (int p = tid; p < P; p += SELECT_TPB) nk[(long long)n_new * P + p] = it.k[p];
      if (tid == 0) ns[n_new] = it.s;
      last = got;
    }
    if (tid == 0) a.top_n[on] = n_new;
  }
  if (!a.last) return;

  // the round's end: its best score, the result in the first round with a success (or the best of the last round),
  // and the list promoted to the next round's beam
  __syncthreads();
  if (tid == 0) {
    a.best_score[(long long)b * (a.R + 1) + a.r] = a.trk_score[b];
    int res = -1;
    if (!a.done[b] && a.trk_ok[(long long)B + b]) {
      res = 1;
      a.done[b] = 1;
      a.n_removed[b] = a.r;
    } else if (!a.done[b] && a.r == a.R) {
      res = 0;
      a.n_removed[b] = -1;
    }
    take[0] = res;
  }
  __syncthreads();
  const int res = take[0];
  if (res >= 0) {
    const long long o = (long long)res * B + b;
    for (int p = tid; p < P; p += SELECT_TPB) a.removed[(long long)b * P + p] = a.trk_keep[o * P + p] ? 0 : 1;
    for (int c = tid; c < C; c += SELECT_TPB) a.logits_out[(long long)b * C + c] = a.trk_logits[o * C + c];
    if (tid == 0) a.score[b] = a.trk_score[o];
  }
  if (a.wsel > 0) {
    const uint8_t* nk = a.top_keep + ((long long)(a.cur ^ 1) * B + b) * W * P;
    for (int w = tid; w < n_new; w += SELECT_TPB) {
      int16_t* s = a.beam + ((long long)b * W + w) * a.R;
      int i = 0;
      for (int p = 0; p < P; ++p) if (!nk[(long long)w * P + p]) s[i++] = (int16_t)p;
    }
    if (tid == 0) a.beam_n[b] = n_new;
  }
}

}  // namespace

int sa_keep(const SaKeepArgs& a, cudaStream_t st) {
  const int64_t rows = (int64_t)a.B * a.nc;
  launch_pdl(sa_keep_kernel, dim3((unsigned)ceil_div(rows, KEEP_TPB)), dim3(KEEP_TPB), 0, st, a);
  RD_CHECK_LAUNCH("sa_keep_kernel");
  return 0;
}

int sa_select(const SaSelectArgs& a, cudaStream_t st) {
  launch_pdl(sa_select_kernel, dim3(a.B), dim3(SELECT_TPB), 0, st, a);
  RD_CHECK_LAUNCH("sa_select_kernel");
  return 0;
}

}  // namespace rd
