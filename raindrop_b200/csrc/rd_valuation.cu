// KNN-Shapley data valuation (Jia et al., VLDB 2019): rd_knn_shapley and rd_debug_knn_rank.
//
// For one query q with label y_q and the N candidate training records ranked by similarity, descending, ties to the
// lower index (alpha_1 .. alpha_N), the Shapley value of the record at rank r under the utility
//   U(S) = (1/K) #{the min(K, |S|) records of S nearest to q that carry label y_q}
// is, with m_r = 1[y(alpha_r) = y_q] and c_r = min(K, r) / (r K),
//   s_r = m_r c_r - sum_{j > r} t_j,   t_j = m_j / (j (j - 1)) for j > K and 0 otherwise
// (Theorem 1's recursion s_r = s_{r+1} + (m_r - m_{r+1}) c_r, s_N = m_N c_N, summed from the end; exact for K > N too).
// Per chunk of queries:
//   kv_sim_kernel         one CTA per 64 queries x 64 training records: the fp64 dots of the normalised fp32 rows on
//                         DMMA (rd_dmma.cuh), every element over the same k-blocks in the same order, written as 64-bit
//                         keys whose ascending order is descending similarity (-0 as +0, NaN after every number, the
//                         query's own record in leave-one-out mode after everything).
//   kv_rank_kernel        one CTA per query: a stable LSD radix sort of the keys with the index as payload, eight 8-bit
//                         passes through global scratch (a pass whose digit is the same for every key is the identity
//                         and is skipped).  The keys arrive in index order, so stability ranks ties by index.  Then
//                         the suffix sums of t in a fixed order (each thread a contiguous run of ranks from the end, the
//                         runs' totals summed from the last), s_r scattered to the record's column of the query's row,
//                         and utility[q] = (matches among the first min(K, N) ranks) / K.
//   kv_accumulate_kernel  values[i] (+)= the chunk's rows, one thread per record, queries in order.
// Every sum has one order fixed by (n_train, K) and the query index alone: the result is bitwise independent of the
// chunking and of how a query set is split across accumulating calls.
#include <math.h>

#include "rd_dmma.cuh"

namespace rd {
namespace {

constexpr int KV_THREADS = 256;               // the ranking CTA: one thread per radix bin
constexpr int KV_WARPS = KV_THREADS / 32;
constexpr int KV_BINS = 256, KV_PASSES = 8;
constexpr unsigned long long KV_SELF_KEY = ~0ull;
constexpr unsigned long long KV_NAN_KEY = ~0ull - 1;
static_assert(KV_BINS == KV_THREADS, "one thread per radix bin");

__device__ __forceinline__ unsigned long long kv_key(double s) {
  if (isnan(s)) return KV_NAN_KEY;
  unsigned long long u = (unsigned long long)__double_as_longlong(s + 0.0);
  u = (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);   // ascending with s
  return ~u;
}

__device__ __forceinline__ double kv_sim(unsigned long long key) {
  unsigned long long u = ~key;
  u = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
  return __longlong_as_double((long long)u);
}

// rows [r0, r0 + 64) x columns [k0, k0 + 32) of X [n, ld] (fp32) -> s[k][m] (fp64); rows >= n and columns >= ld are 0
struct RowLoader {
  float4 v[4];
  __device__ __forceinline__ void load(const float* __restrict__ X, long long n, int ld, long long r0, int k0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int idx = threadIdx.x + TK_THREADS * q, c4 = idx >> 6, row = idx & 63;
      v[q] = r0 + row < n && k0 + 4 * c4 < ld ? __ldg(reinterpret_cast<const float4*>(X + (r0 + row) * ld + k0) + c4)
                                              : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  __device__ __forceinline__ void store(double* s) const {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int idx = threadIdx.x + TK_THREADS * q, c4 = idx >> 6, row = idx & 63;
      s[(4 * c4 + 0) * TK_LD + row] = (double)v[q].x;
      s[(4 * c4 + 1) * TK_LD + row] = (double)v[q].y;
      s[(4 * c4 + 2) * TK_LD + row] = (double)v[q].z;
      s[(4 * c4 + 3) * TK_LD + row] = (double)v[q].w;
    }
  }
};

// keys[r, j] for the chunk's queries r < nq and records j < n; self0 >= 0: query r is record self0 + r.
__global__ void __launch_bounds__(TK_THREADS)
kv_sim_kernel(const float* __restrict__ Q, long long nq, const float* __restrict__ B, long long n, int ld, long long self0,
              unsigned long long* __restrict__ keys) {
  extern __shared__ double tk_smem[];
  pdl_launch_dependents();
  const long long j0 = (long long)blockIdx.x * TK_TILE, q0 = (long long)blockIdx.y * TK_TILE;
  pdl_wait();
  RowLoader la, lb;
  double acc[2][4][4];
  tk_mainloop(
      tk_smem, (ld + TK_BK - 1) / TK_BK,
      [&](int kb) {
        la.load(Q, nq, ld, q0, kb * TK_BK);
        lb.load(B, n, ld, j0, kb * TK_BK);
      },
      [&](double* s) {
        la.store(s);
        lb.store(s + TK_OPERAND);
      },
      acc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const long long r = q0 + (warp & 1) * 32 + 16 * mi + g + 8 * (e >> 1);
        const long long c = j0 + (warp >> 1) * 32 + 8 * ni + 2 * t + (e & 1);
        if (r < nq && c < n) keys[r * n + c] = self0 >= 0 && c == self0 + r ? KV_SELF_KEY : kv_key(acc[mi][ni][e]);
      }
}

// One CTA per query ql of the chunk: sorts keys0[ql, :n] (payload: the record index) and writes rows[ql, :n] (the
// Shapley values in record order, 0 at the query's own record) and utility[ql].  With y_train NULL only the debug
// outputs are written: dbg_order[ql, p] = the record at sorted position p, dbg_sim[ql, j] = record j's similarity.
__global__ void __launch_bounds__(KV_THREADS)
kv_rank_kernel(unsigned long long* __restrict__ keys0, unsigned long long* __restrict__ keys1, uint32_t* __restrict__ idx0,
               uint32_t* __restrict__ idx1, long long n, long long self0, const int64_t* __restrict__ y_train,
               const int64_t* __restrict__ y_query, int K, double* __restrict__ rows, double* __restrict__ utility,
               double* __restrict__ dbg_sim, int64_t* __restrict__ dbg_order) {
  __shared__ unsigned hist[KV_PASSES][KV_BINS];
  __shared__ unsigned wcnt[KV_WARPS][KV_BINS];
  __shared__ unsigned base[KV_BINS];
  __shared__ double seg[KV_THREADS];
  __shared__ int n_match;
  pdl_launch_dependents();
  pdl_wait();
  const long long ql = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned long long* src_k = keys0 + ql * n;
  unsigned long long* dst_k = keys1 + ql * n;
  uint32_t* src_i = idx0 + ql * n;
  uint32_t* dst_i = idx1 + ql * n;
  for (int i = tid; i < KV_PASSES * KV_BINS; i += KV_THREADS) (&hist[0][0])[i] = 0u;
  if (tid == 0) n_match = 0;
  __syncthreads();
  // the eight digits' histograms in one read: a stable pass permutes the keys, so each pass's histogram is known upfront
  for (long long e0 = 0; e0 < n; e0 += KV_THREADS) {
    const long long e = e0 + tid;
    const bool valid = e < n;
    const unsigned mask = __ballot_sync(0xffffffffu, valid);
    if (valid) {
      const unsigned long long key = src_k[e];
#pragma unroll
      for (int p = 0; p < KV_PASSES; ++p) {
        const unsigned d = (unsigned)(key >> (8 * p)) & 255u;
        const unsigned peers = __match_any_sync(mask, d);
        if (lane == __ffs(peers) - 1) atomicAdd(&hist[p][d], (unsigned)__popc(peers));
      }
    }
  }
  bool implied = true;                        // the payload is still the position (the keys arrive in index order)
  for (int p = 0; p < KV_PASSES; ++p) {
    if (__syncthreads_or(hist[p][tid] == (unsigned)n)) continue;   // one digit value: the stable pass is the identity
    if (tid == 0) {
      unsigned s = 0;
      for (int b = 0; b < KV_BINS; ++b) { base[b] = s; s += hist[p][b]; }
    }
    __syncthreads();
    for (long long e0 = 0; e0 < n; e0 += KV_THREADS) {
      const long long e = e0 + tid;
      const bool valid = e < n;
      const unsigned mask = __ballot_sync(0xffffffffu, valid);
      unsigned long long key = 0;
      uint32_t id = 0;
      unsigned d = 0, peers = 0;
      if (valid) {
        key = src_k[e];
        id = implied ? (uint32_t)e : src_i[e];
        d = (unsigned)(key >> (8 * p)) & 255u;
        peers = __match_any_sync(mask, d);
      }
#pragma unroll
      for (int w = 0; w < KV_WARPS; ++w) wcnt[w][tid] = 0u;
      __syncthreads();
      if (valid && lane == __ffs(peers) - 1) wcnt[warp][d] = (unsigned)__popc(peers);
      __syncthreads();
      if (valid) {
        unsigned off = base[d] + (unsigned)__popc(peers & ((1u << lane) - 1u));
        for (int w = 0; w < warp; ++w) off += wcnt[w][d];
        dst_k[off] = key;
        dst_i[off] = id;
      }
      __syncthreads();
      unsigned tile = 0;
#pragma unroll
      for (int w = 0; w < KV_WARPS; ++w) tile += wcnt[w][tid];
      base[tid] += tile;
    }
    __syncthreads();                          // the pass's stores are visible to the whole CTA
    unsigned long long* tk = src_k; src_k = dst_k; dst_k = tk;
    uint32_t* ti = src_i; src_i = dst_i; dst_i = ti;
    implied = false;
  }
  if (dbg_order || dbg_sim) {
    for (long long p = tid; p < n; p += KV_THREADS) {
      const uint32_t id = implied ? (uint32_t)p : src_i[p];
      if (dbg_order) dbg_order[ql * n + p] = (int64_t)id;
      if (dbg_sim) dbg_sim[ql * n + id] = kv_sim(src_k[p]);
    }
  }
  if (!y_train) return;
  // ranks r = p + 1 for p < N; the query's own record, when excluded, sorted last
  const long long N = self0 >= 0 ? n - 1 : n;
  const int64_t yq = y_query[ql];
  const long long per = (N + KV_THREADS - 1) / KV_THREADS;
  const long long p0 = min(N, tid * per), p1 = min(N, p0 + per);
  double tot = 0.0;
  int cnt = 0;
  for (long long p = p1 - 1; p >= p0; --p) {
    const long long r = p + 1;
    const bool m = y_train[implied ? p : (long long)src_i[p]] == yq;
    if (m && r > K) tot += 1.0 / ((double)r * (double)(r - 1));
    cnt += m && r <= K;
  }
  seg[tid] = tot;
  if (cnt) atomicAdd(&n_match, cnt);
  __syncthreads();
  if (tid == 0) {                             // seg[t] = the runs after run t, summed from the last
    double s = 0.0;
    for (int t = KV_THREADS - 1; t >= 0; --t) { const double v = seg[t]; seg[t] = s; s += v; }
  }
  __syncthreads();
  double* row = rows + ql * n;
  double acc = seg[tid];                      // sum of t_j over j > r
  const double invK = 1.0 / (double)K;
  for (long long p = p1 - 1; p >= p0; --p) {
    const long long r = p + 1;
    const uint32_t id = implied ? (uint32_t)p : src_i[p];
    const bool m = y_train[id] == yq;
    row[id] = (m ? (r <= K ? invK : 1.0 / (double)r) : 0.0) - acc;
    if (m && r > K) acc += 1.0 / ((double)r * (double)(r - 1));
  }
  if (tid == 0) {
    if (self0 >= 0) row[self0 + ql] = 0.0;
    if (utility) utility[ql] = (double)n_match / (double)K;
  }
}

__global__ void kv_accumulate_kernel(const double* __restrict__ rows, long long nq, long long n, int accumulate,
                                     double* __restrict__ values) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double v = accumulate ? values[i] : 0.0;
  for (long long q = 0; q < nq; ++q) v += rows[q * n + i];
  values[i] = v;
}

struct KvLayout { size_t keys0, keys1, idx0, idx1, rows, total; };

bool kv_args_ok(int64_t n_train, int32_t ld, int64_t qc) {
  return n_train >= 1 && n_train < (1ll << 31) && ld >= 4 && ld % 4 == 0 && qc >= 1 && qc <= (1ll << 56) / n_train;
}

KvLayout kv_layout(int64_t n_train, int64_t qc) {
  KvLayout l{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  const size_t e = (size_t)qc * (size_t)n_train;
  l.keys0 = take(e * 8);
  l.keys1 = take(e * 8);
  l.idx0 = take(e * 4);
  l.idx1 = take(e * 4);
  l.rows = take(e * 8);
  l.total = off;
  return l;
}

constexpr int64_t KV_MAX_CHUNK = 65535ll * TK_TILE;   // grid.y of the similarity launch

// The similarity and ranking launches of one chunk of nq queries.
int kv_chunk(const float* bank, int64_t n, int32_t ld, const float* queries, int64_t nq, int64_t self0,
             const KvLayout& l, uint8_t* sb, const int64_t* y_train, const int64_t* y_query, int32_t k, double* rows,
             double* utility, double* dbg_sim, int64_t* dbg_order, cudaStream_t st) {
  auto* keys0 = reinterpret_cast<unsigned long long*>(sb + l.keys0);
  auto* keys1 = reinterpret_cast<unsigned long long*>(sb + l.keys1);
  launch_pdl(kv_sim_kernel, dim3((unsigned)ceil_div(n, TK_TILE), (unsigned)ceil_div(nq, TK_TILE)), dim3(TK_THREADS),
             TK_SMEM, st, queries, (long long)nq, bank, (long long)n, (int)ld, (long long)self0, keys0);
  RD_CHECK_LAUNCH("kv_sim_kernel");
  launch_pdl(kv_rank_kernel, dim3((unsigned)nq), dim3(KV_THREADS), 0, st, keys0, keys1,
             reinterpret_cast<uint32_t*>(sb + l.idx0), reinterpret_cast<uint32_t*>(sb + l.idx1), (long long)n,
             (long long)self0, y_train, y_query, (int)k, rows, utility, dbg_sim, dbg_order);
  RD_CHECK_LAUNCH("kv_rank_kernel");
  return 0;
}

}  // namespace
}  // namespace rd

using namespace rd;

extern "C" {

size_t rd_knn_shapley_scratch_bytes(int64_t n_train, int32_t ld, int32_t queries_per_chunk) {
  if (!kv_args_ok(n_train, ld, queries_per_chunk)) return 0;
  return kv_layout(n_train, queries_per_chunk < KV_MAX_CHUNK ? queries_per_chunk : KV_MAX_CHUNK).total;
}

int rd_knn_shapley(const float* bank, int64_t n_train, int32_t ld, const int64_t* y_train, const float* queries,
                   int64_t n_query, const int64_t* y_query, int32_t k, int64_t self_offset, int32_t queries_per_chunk,
                   int32_t accumulate, void* scratch, double* values, double* per_query, double* utility, void* stream) {
  const char* fn = "rd_knn_shapley";
  if (!bank || !y_train || !scratch || !values || (n_query > 0 && (!queries || !y_query))) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (k < 1 || n_query < 0 || !kv_args_ok(n_train, ld, queries_per_chunk)) {
    set_error("%s: bad sizes (n_train=%lld ld=%d n_query=%lld k=%d queries_per_chunk=%d; 1 <= n_train < 2^31, ld a "
              "multiple of 4, k >= 1)", fn, (long long)n_train, ld, (long long)n_query, k, queries_per_chunk);
    return -2;
  }
  if (self_offset < -1 || (self_offset >= 0 && (n_train < 2 || self_offset > n_train - n_query))) {
    set_error("%s: self range [%lld, %lld) must lie in the bank of %lld records (at least 2)", fn,
              (long long)self_offset, (long long)(self_offset + n_query), (long long)n_train);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(bank) | reinterpret_cast<uintptr_t>(queries)) & 15) {
    set_error("%s: bank and queries must be 16-byte aligned", fn);
    return -2;
  }
  if (reinterpret_cast<uintptr_t>(scratch) & 255) { set_error("%s: scratch must be 256-byte aligned", fn); return -2; }
  const int64_t qc = queries_per_chunk < KV_MAX_CHUNK ? queries_per_chunk : KV_MAX_CHUNK;
  const KvLayout l = kv_layout(n_train, qc);
  uint8_t* sb = static_cast<uint8_t*>(scratch);
  const cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(tc::ensure_max_smem((const void*)kv_sim_kernel, TK_SMEM));
  const dim3 agrid((unsigned)ceil_div(n_train, 256));
  if (n_query == 0) {
    launch_pdl(kv_accumulate_kernel, agrid, dim3(256), 0, st, (const double*)nullptr, 0ll, (long long)n_train,
               (int)accumulate, values);
    RD_CHECK_LAUNCH("kv_accumulate_kernel");
  }
  for (int64_t q0 = 0; q0 < n_query; q0 += qc) {
    const int64_t nq = n_query - q0 < qc ? n_query - q0 : qc;
    double* rows = per_query ? per_query + q0 * n_train : reinterpret_cast<double*>(sb + l.rows);
    RD_TRY(kv_chunk(bank, n_train, ld, queries + q0 * ld, nq, self_offset >= 0 ? self_offset + q0 : -1, l, sb, y_train,
                    y_query + q0, k, rows, utility ? utility + q0 : nullptr, nullptr, nullptr, st));
    launch_pdl(kv_accumulate_kernel, agrid, dim3(256), 0, st, (const double*)rows, (long long)nq, (long long)n_train,
               (int)(accumulate || q0 > 0), values);
    RD_CHECK_LAUNCH("kv_accumulate_kernel");
  }
  return 0;
}

int rd_debug_knn_rank(const float* bank, int64_t n_train, int32_t ld, const float* queries, int64_t n_query,
                      int64_t self_offset, void* scratch, double* sim, int64_t* order, void* stream) {
  const char* fn = "rd_debug_knn_rank";
  if (!bank || !queries || !scratch || !sim || !order) { set_error("%s: NULL argument", fn); return -2; }
  if (n_query < 1 || n_query > KV_MAX_CHUNK || !kv_args_ok(n_train, ld, n_query) || self_offset < -1 ||
      (self_offset >= 0 && self_offset > n_train - n_query)) {
    set_error("%s: bad sizes (n_train=%lld ld=%d n_query=%lld self_offset=%lld)", fn, (long long)n_train, ld,
              (long long)n_query, (long long)self_offset);
    return -2;
  }
  if (((reinterpret_cast<uintptr_t>(bank) | reinterpret_cast<uintptr_t>(queries)) & 15) ||
      (reinterpret_cast<uintptr_t>(scratch) & 255)) {
    set_error("%s: bank and queries must be 16-byte aligned, scratch 256-byte aligned", fn);
    return -2;
  }
  RD_TRY(tc::ensure_max_smem((const void*)kv_sim_kernel, TK_SMEM));
  return kv_chunk(bank, n_train, ld, queries, n_query, self_offset, kv_layout(n_train, n_query),
                  static_cast<uint8_t*>(scratch), nullptr, nullptr, 1, nullptr, nullptr, sim, order, (cudaStream_t)stream);
}

}  // extern "C"
