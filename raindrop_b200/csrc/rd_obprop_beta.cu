// Observation_progation.forward with use_beta=True (code/Ob_propagation.py:161-186,191,195-228): the
// dormant but selectable branch of the operator.  Everything that the reference evaluates per EDGE
// depends on the edge's TARGET node only (x_i = x[edge_index[1]]), so we evaluate it per NODE:
//   Hn      = increase_dim(x)                       [N, 8C] viewed [N, T, 32]      (:166)
//   beta[n,t] = mean_k( Hn[n,t,k] * [map_weights[n] || p_t[t]]_k )                   (:167-172)
//   gamma[e,t] = beta[tgt(e), t] * w[e], repeated d_ob times along channels          (:176-177)
//   score[e] = mean_c gamma[e, c]; keep the K = int(E/2) highest edges, in that order (:180-186)
//   gamma'  = per-channel segment softmax over the kept edges grouped by SOURCE      (:183,195)
//   out[s]  = sum_{kept e: src(e)=s} relu(lin_value(x[tgt(e)])) * gamma'[e]          (:200,208,226-228)
// returned: out [N, C], pruned edge_index [2, K], alpha[K] = score of the kept edges (:191).
#include "rd_kernels.cuh"

namespace rd {
namespace {

__global__ void beta_node_kernel(const float* __restrict__ Hn, const float* __restrict__ map_w,
                                 const float* __restrict__ p_t, int N, int T, float* __restrict__ beta) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * T) return;
  int n = i / T, t = i - n * T;
  const float* h = Hn + ((long long)n * T + t) * 32;
  float s = 0.f;
  for (int k = 0; k < 16; ++k) s += h[k] * map_w[n * 16 + k];
  for (int k = 0; k < 16; ++k) s += h[16 + k] * p_t[t * 16 + k];
  beta[i] = s / 32.f;
}

// score[e] = mean over channels of beta[tgt,t]*w[e] repeated d_ob times == w[e] * mean_t beta[tgt, t]
__global__ void edge_score_kernel(const float* __restrict__ beta, const int64_t* __restrict__ tgt,
                                  const float* __restrict__ w, int E, int T, int d_ob, float* __restrict__ score) {
  int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (e >= E) return;
  const float* b = beta + (long long)tgt[e] * T;
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += (b[t] * w[e]) * (float)d_ob;   // sum over the C = T*d_ob repeated entries
  s = warp_sum(s);
  if (lane == 0) score[e] = s / (float)(T * d_ob);
}

// descending stable rank (== torch.argsort(descending=True) for distinct scores); writes the kept edges
__global__ void rank_and_prune_kernel(const float* __restrict__ score, const int64_t* __restrict__ src,
                                      const int64_t* __restrict__ tgt, int E, int K, int* __restrict__ rank,
                                      int64_t* __restrict__ src_out, int64_t* __restrict__ tgt_out,
                                      float* __restrict__ alpha_out, int* __restrict__ eid_out) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  float s = score[e];
  int r = 0;
  for (int j = 0; j < E; ++j) {
    float sj = score[j];
    r += (sj > s) || (sj == s && j < e);
  }
  rank[e] = r;
  if (r < K) { src_out[r] = src[e]; tgt_out[r] = tgt[e]; alpha_out[r] = s; if (eid_out) eid_out[r] = e; }
}

// one block per source node; threads over channels; kept edges = rank < K
__global__ void beta_aggregate_kernel(const float* __restrict__ V, const float* __restrict__ beta,
                                      const int64_t* __restrict__ src, const int64_t* __restrict__ tgt,
                                      const float* __restrict__ w, const int* __restrict__ rank, int E, int K, int C,
                                      int T, int d_ob, float* __restrict__ out) {
  const int s = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int t = c / d_ob;
    float mx = -INFINITY;
    for (int e = 0; e < E; ++e)
      if (rank[e] < K && src[e] == s) mx = fmaxf(mx, beta[(long long)tgt[e] * T + t] * w[e]);
    float acc = 0.f;
    if (mx != -INFINITY) {
      float den = 0.f;
      for (int e = 0; e < E; ++e)
        if (rank[e] < K && src[e] == s) den += expf(beta[(long long)tgt[e] * T + t] * w[e] - mx);
      den += 1e-16f;
      // (the reference's scatter-add runs over the kept list in descending-score order; we sum in edge
      //  order -- same terms, fp32 rounding differs at the 1e-7 level)
      for (int e = 0; e < E; ++e)
        if (rank[e] < K && src[e] == s)
          acc += V[(long long)tgt[e] * C + c] * (expf(beta[(long long)tgt[e] * T + t] * w[e] - mx) / den);
    }
    out[(long long)s * C + c] = acc;
  }
}

// ---- backward ---------------------------------------------------------------------------------------
// per (source s, channel c) over the kept edges leaving s: mx, den of the softmax and dot = sum_e g'[e] dg'[e] with
// g' = exp(gamma - mx) / den, dg' = d_out[s, c] * V[tgt e, c]
__global__ void beta_bwd_stats_kernel(const float* __restrict__ V, const float* __restrict__ beta, const int64_t* __restrict__ ksrc,
                                      const int64_t* __restrict__ ktgt, const float* __restrict__ kw, int K, int C, int T, int d_ob,
                                      const float* __restrict__ dout, float* __restrict__ mx_o, float* __restrict__ den_o,
                                      float* __restrict__ dot_o) {
  const int s = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int t = c / d_ob;
    float mx = -INFINITY;
    for (int r = 0; r < K; ++r) if (ksrc[r] == s) mx = fmaxf(mx, beta[(long long)ktgt[r] * T + t] * kw[r]);
    float den = 0.f, dot = 0.f;
    if (mx != -INFINITY) {
      for (int r = 0; r < K; ++r) if (ksrc[r] == s) den += expf(beta[(long long)ktgt[r] * T + t] * kw[r] - mx);
      den += 1e-16f;
      const float go = dout[(long long)s * C + c];
      for (int r = 0; r < K; ++r)
        if (ksrc[r] == s) dot += (expf(beta[(long long)ktgt[r] * T + t] * kw[r] - mx) / den) * (go * V[(long long)ktgt[r] * C + c]);
    }
    mx_o[(long long)s * C + c] = mx; den_o[(long long)s * C + c] = den; dot_o[(long long)s * C + c] = dot;
  }
}
// per kept edge r and channel c: gp[r, c] = g'  and  dgam[r, c] = g' * (dg' - dot[src, c])
__global__ void beta_bwd_edge_kernel(const float* __restrict__ V, const float* __restrict__ beta, const int64_t* __restrict__ ksrc,
                                     const int64_t* __restrict__ ktgt, const float* __restrict__ kw, int K, int C, int T, int d_ob,
                                     const float* __restrict__ dout, const float* __restrict__ mx, const float* __restrict__ den,
                                     const float* __restrict__ dot, float* __restrict__ gp, float* __restrict__ dgam) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)K * C) return;
  const int r = (int)(o / C), c = (int)(o - (long long)r * C), t = c / d_ob;
  const long long s = ksrc[r], i = ktgt[r];
  const float g = expf(beta[i * T + t] * kw[r] - mx[s * C + c]) / den[s * C + c];
  const float dg = dout[s * C + c] * V[i * C + c];
  gp[o] = g;
  dgam[o] = g * (dg - dot[s * C + c]);
}
// per TARGET node i: d(pre-activation of lin_value)[i, c] = [V > 0] * sum_{kept r: tgt = i} d_out[src r, c] * g'[r, c]
__global__ void beta_bwd_value_kernel(const float* __restrict__ V, const int64_t* __restrict__ ksrc, const int64_t* __restrict__ ktgt,
                                      int K, int C, const float* __restrict__ dout, const float* __restrict__ gp,
                                      float* __restrict__ dpre) {
  const int i = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f;
    for (int r = 0; r < K; ++r) if (ktgt[r] == i) a += dout[ksrc[r] * C + c] * gp[(long long)r * C + c];
    dpre[(long long)i * C + c] = V[(long long)i * C + c] > 0.f ? a : 0.f;
  }
}
// d_edge_w[eid r] = sum_c dgam[r, c] * beta[tgt, t(c)] + d_alpha[r] * mean_t beta[tgt, t]       one warp per kept edge
__global__ void beta_bwd_edgew_kernel(const float* __restrict__ beta, const int64_t* __restrict__ ktgt, const int* __restrict__ eid,
                                      int K, int C, int T, int d_ob, const float* __restrict__ dgam,
                                      const float* __restrict__ dalpha, float* __restrict__ dw) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= K) return;
  const float* b = beta + (long long)ktgt[r] * T;
  float a = 0.f, m = 0.f;
  for (int c = lane; c < C; c += 32) a += dgam[(long long)r * C + c] * b[c / d_ob];
  for (int t = lane; t < T; t += 32) m += b[t];
  a = warp_sum(a); m = warp_sum(m);
  if (lane == 0) dw[eid[r]] = a + (dalpha ? dalpha[r] * (m / (float)T) : 0.f);
}
// d_beta[i, t] = sum_{kept r: tgt = i} w_r * ( sum_{k < d_ob} dgam[r, t*d_ob + k] + d_alpha[r] / T )
__global__ void beta_bwd_beta_kernel(const int64_t* __restrict__ ktgt, const float* __restrict__ kw, int K, int N, int C, int T,
                                     int d_ob, const float* __restrict__ dgam, const float* __restrict__ dalpha,
                                     float* __restrict__ dbeta) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N * T) return;
  const int i = o / T, t = o - i * T;
  float a = 0.f;
  for (int r = 0; r < K; ++r) {
    if (ktgt[r] != i) continue;
    float g = 0.f;
    for (int k = 0; k < d_ob; ++k) g += dgam[(long long)r * C + t * d_ob + k];
    if (dalpha) g += dalpha[r] / (float)T;
    a += kw[r] * g;
  }
  dbeta[o] = a;
}
// beta[n, t] = mean_k( Hn[n, t, k] * [map_w[n] || p_t[t]]_k ):  d_Hn, d_map_w[n, k], d_p_t[t, k]
__global__ void beta_bwd_hn_kernel(const float* __restrict__ map_w, const float* __restrict__ p_t, int N, int T,
                                   const float* __restrict__ dbeta, float* __restrict__ dHn) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)N * T * 32) return;
  const int k = (int)(o & 31);
  const long long nt = o >> 5;
  const int n = (int)(nt / T), t = (int)(nt - (long long)n * T);
  const float a = k < 16 ? map_w[n * 16 + k] : p_t[t * 16 + (k - 16)];
  dHn[o] = dbeta[nt] * a * (1.f / 32.f);
}
__global__ void beta_bwd_mapw_kernel(const float* __restrict__ Hn, int N, int T, const float* __restrict__ dbeta,
                                     float* __restrict__ dmap, float* __restrict__ dpt) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o < N * 16) {
    const int n = o / 16, k = o - n * 16;
    float a = 0.f;
    for (int t = 0; t < T; ++t) a += dbeta[n * T + t] * Hn[((long long)n * T + t) * 32 + k];
    dmap[o] = a * (1.f / 32.f);
  } else if (dpt && o < N * 16 + T * 16) {
    const int q = o - N * 16, t = q / 16, k = q - t * 16;
    float a = 0.f;
    for (int n = 0; n < N; ++n) a += dbeta[n * T + t] * Hn[((long long)n * T + t) * 32 + 16 + k];
    dpt[q] = a * (1.f / 32.f);
  }
}

struct BLay { long long Hn, V, beta, score, rank, eid, kw, klist, mx, den, dot, gp, dgam, dpre, dbeta, dHn, partial, total; };
BLay blayout(int N, int T, int d_ob, int E) {
  const long long C = (long long)T * d_ob, K = E / 2;
  BLay l;
  long long o = 0;
  auto take = [&](long long n) { long long r = o; o += round_up(n > 0 ? n : 1, 64); return r; };
  l.Hn = take((long long)N * 8 * C); l.V = take((long long)N * C); l.beta = take((long long)N * T);
  l.score = take(E); l.rank = take(E); l.eid = take(K); l.kw = take(K);
  l.klist = take(5 * K + 16);          // kept edges: int64 src[K], int64 tgt[K], float alpha[K]
  l.mx = take((long long)N * C); l.den = take((long long)N * C); l.dot = take((long long)N * C);
  l.gp = take(K * C); l.dgam = take(K * C); l.dpre = take((long long)N * C); l.dbeta = take((long long)N * T);
  l.dHn = take((long long)N * 8 * C);
  // both weight gradients share `partial`; the [C, C] one has fewer tiles, so it may split where the [8C, C] one does not
  int ns;
  const int64_t p_inc = gemm_splitk_plan((int)(8 * C), (int)C, N, &ns), p_val = gemm_splitk_plan((int)C, (int)C, N, &ns);
  l.partial = take(p_inc > p_val ? p_inc : p_val);
  l.total = o;
  return l;
}

__global__ void gather_kept_w_kernel(const float* __restrict__ w, const int* __restrict__ eid, int K, float* __restrict__ kw) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < K) kw[r] = w[eid[r]];
}

}  // namespace
}  // namespace rd

using namespace rd;

extern "C" size_t rd_obprop_beta_bwd_scratch_bytes(int32_t N, int32_t T, int32_t d_ob, int32_t E) {
  if (N < 1 || T < 1 || d_ob < 1 || E < 2) return 0;
  return (size_t)blayout(N, T, d_ob, E).total * sizeof(float);
}

// Backward of rd_obprop_beta_fwd (same inputs; the forward is recomputed, the kept-edge selection is piecewise
// constant and gets no gradient).  d_out [N, C]; d_alpha [K] or NULL (gradient w.r.t. the returned alpha = mean gamma
// of the kept edges, which Raindrop_v2 would feed into layer 2 as edge weights, code/models_rd.py:332-336).
// Writes d_x [N, C] (may be NULL), d_edge_w [E], d_p_t [T, 16] (may be NULL), d_increase_dim_{w [8C, C], b [8C]},
// d_map_weights [N, 16], d_value_{w [C, C], b [C]}.
extern "C" int rd_obprop_beta_bwd(const float* x, const float* p_t, const int64_t* edge_src, const int64_t* edge_tgt,
                                  const float* edge_w, int32_t E, int32_t N, int32_t T, int32_t d_ob,
                                  const float* increase_dim_w, const float* increase_dim_b, const float* map_weights,
                                  const float* value_w, const float* value_b, const float* d_out, const float* d_alpha,
                                  float* d_x, float* d_edge_w, float* d_p_t, float* d_inc_w, float* d_inc_b, float* d_map_w,
                                  float* d_val_w, float* d_val_b, void* scratch, void* stream) {
  if (!x || !p_t || !edge_src || !edge_tgt || !edge_w || !increase_dim_w || !increase_dim_b || !map_weights || !value_w ||
      !value_b || !d_out || !d_edge_w || !d_inc_w || !d_inc_b || !d_map_w || !d_val_w || !d_val_b || !scratch || N < 1 || T < 1) {
    set_error("rd_obprop_beta_bwd: bad arguments");
    return -2;
  }
  if (E < 2) { set_error("rd_obprop_beta_bwd: E = %d, but keeping the top E / 2 edges needs E >= 2", E); return -2; }
  if (d_ob * 8 != 32) { set_error("use_beta needs d_ob == 4 (code/Ob_propagation.py:166)"); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  const int C = T * d_ob, K = E / 2;
  const BLay l = blayout(N, T, d_ob, E);
  float* sc = (float*)scratch;
  float* Hn = sc + l.Hn; float* V = sc + l.V; float* beta = sc + l.beta; float* score = sc + l.score;
  int* rank = (int*)(sc + l.rank); int* eid = (int*)(sc + l.eid); float* kw = sc + l.kw;
  float* mx = sc + l.mx; float* den = sc + l.den; float* dot = sc + l.dot; float* gp = sc + l.gp; float* dgam = sc + l.dgam;
  float* dpre = sc + l.dpre; float* dbeta = sc + l.dbeta; float* dHn = sc + l.dHn; float* partial = sc + l.partial;
  int64_t* ksrc = (int64_t*)(sc + l.klist);
  int64_t* ktgt = ksrc + K;
  float* kalpha = (float*)(ktgt + K);
  // ---- recompute the forward up to the pruned edge list -----------------------------------------------
  GemmP g;
  g.A = x; g.ta = 0; g.sAi = C; g.sAk = 1; g.B = increase_dim_w; g.tb = 1; g.sBj = C; g.sBk = 1;
  g.C = Hn; g.sCi = 8 * C; g.sCj = 1; g.M = N; g.N = 8 * C; g.K = C; g.bias = increase_dim_b;
  RD_TRY(gemm(g, st));
  g.B = value_w; g.C = V; g.sCi = C; g.N = C; g.bias = value_b; g.relu = 1;
  RD_TRY(gemm(g, st));
  beta_node_kernel<<<(unsigned)ceil_div((int64_t)N * T, 256), 256, 0, st>>>(Hn, map_weights, p_t, N, T, beta);
  RD_CHECK_LAUNCH("beta_node_kernel");
  edge_score_kernel<<<(unsigned)ceil_div((int64_t)E * 32, 256), 256, 0, st>>>(beta, edge_tgt, edge_w, E, T, d_ob, score);
  RD_CHECK_LAUNCH("edge_score_kernel");
  rank_and_prune_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(score, edge_src, edge_tgt, E, K, rank, ksrc, ktgt, kalpha, eid);
  RD_CHECK_LAUNCH("rank_and_prune_kernel");
  gather_kept_w_kernel<<<(unsigned)ceil_div(K, 256), 256, 0, st>>>(edge_w, eid, K, kw);
  RD_CHECK_LAUNCH("gather_kept_w_kernel");
  // ---- backward of the softmax-weighted aggregation ---------------------------------------------------------
  beta_bwd_stats_kernel<<<N, 256, 0, st>>>(V, beta, ksrc, ktgt, kw, K, C, T, d_ob, d_out, mx, den, dot);
  RD_CHECK_LAUNCH("beta_bwd_stats_kernel");
  beta_bwd_edge_kernel<<<(unsigned)ceil_div((int64_t)K * C, 256), 256, 0, st>>>(V, beta, ksrc, ktgt, kw, K, C, T, d_ob, d_out, mx, den,
                                                                              dot, gp, dgam);
  RD_CHECK_LAUNCH("beta_bwd_edge_kernel");
  beta_bwd_value_kernel<<<N, 256, 0, st>>>(V, ksrc, ktgt, K, C, d_out, gp, dpre);
  RD_CHECK_LAUNCH("beta_bwd_value_kernel");
  if (cudaMemsetAsync(d_edge_w, 0, sizeof(float) * (size_t)E, st) != cudaSuccess) { set_error("rd_obprop_beta_bwd: memset failed"); return -1; }
  beta_bwd_edgew_kernel<<<(unsigned)ceil_div((int64_t)K * 32, 256), 256, 0, st>>>(beta, ktgt, eid, K, C, T, d_ob, dgam, d_alpha, d_edge_w);
  RD_CHECK_LAUNCH("beta_bwd_edgew_kernel");
  beta_bwd_beta_kernel<<<(unsigned)ceil_div((int64_t)N * T, 256), 256, 0, st>>>(ktgt, kw, K, N, C, T, d_ob, dgam, d_alpha, dbeta);
  RD_CHECK_LAUNCH("beta_bwd_beta_kernel");
  beta_bwd_mapw_kernel<<<(unsigned)ceil_div((int64_t)N * 16 + T * 16, 256), 256, 0, st>>>(Hn, N, T, dbeta, d_map_w, d_p_t);
  RD_CHECK_LAUNCH("beta_bwd_mapw_kernel");
  beta_bwd_hn_kernel<<<(unsigned)ceil_div((int64_t)N * T * 32, 256), 256, 0, st>>>(map_weights, p_t, N, T, dbeta, dHn);
  RD_CHECK_LAUNCH("beta_bwd_hn_kernel");
  // ---- the two linear layers --------------------------------------------------------------------------------
  auto wgrad = [&](const float* dy, int out_f, float* dW, float* db) -> int {
    GemmP w;
    w.A = dy; w.ta = 1; w.sAk = out_f; w.sAi = 1;
    w.B = x; w.tb = 0; w.sBk = C; w.sBj = 1;
    w.C = dW; w.sCi = C; w.sCj = 1;
    w.M = out_f; w.N = C; w.K = N;
    int ns;
    gemm_splitk_plan(out_f, C, N, &ns);
    w.nsplit = ns; w.partial = partial; w.asum = db;
    return gemm(w, st);
  };
  RD_TRY(wgrad(dHn, 8 * C, d_inc_w, d_inc_b));
  RD_TRY(wgrad(dpre, C, d_val_w, d_val_b));
  if (d_x) {
    GemmP b1;
    b1.A = dHn; b1.ta = 0; b1.sAi = 8 * C; b1.sAk = 1; b1.B = increase_dim_w; b1.tb = 0; b1.sBk = C; b1.sBj = 1;
    b1.C = d_x; b1.sCi = C; b1.sCj = 1; b1.M = N; b1.N = C; b1.K = 8 * C;
    RD_TRY(gemm(b1, st));
    GemmP b2 = b1;
    b2.A = dpre; b2.sAi = C; b2.B = value_w; b2.K = C; b2.resid = d_x; b2.resid_ld = C;
    RD_TRY(gemm(b2, st));
  }
  return 0;
}

extern "C" size_t rd_obprop_beta_scratch_bytes(int32_t N, int32_t T, int32_t d_ob, int32_t E) {
  if (N < 1 || T < 1 || d_ob < 1 || E < 2) return 0;
  return (size_t)blayout(N, T, d_ob, E).eid * sizeof(float);   // the forward uses the layout up to `rank`
}

extern "C" int rd_obprop_beta_fwd(const float* x, const float* p_t, const int64_t* edge_src, const int64_t* edge_tgt,
                                  const float* edge_w, int32_t E, int32_t N, int32_t T, int32_t d_ob,
                                  const float* increase_dim_w, const float* increase_dim_b, const float* map_weights,
                                  const float* value_w, const float* value_b, float* out, int64_t* edge_src_out,
                                  int64_t* edge_tgt_out, float* alpha_out, void* scratch, void* stream) {
  if (!x || !p_t || !edge_src || !edge_tgt || !edge_w || !increase_dim_w || !increase_dim_b || !map_weights || !value_w ||
      !value_b || !out || !edge_src_out || !edge_tgt_out || !alpha_out || !scratch || N < 1 || T < 1) {
    set_error("rd_obprop_beta_fwd: bad arguments");
    return -2;
  }
  if (E < 2) { set_error("rd_obprop_beta_fwd: E = %d, but keeping the top E / 2 edges needs E >= 2", E); return -2; }
  if (d_ob * 8 != 32) { set_error("use_beta needs out_channels*8 == T*32, i.e. d_ob == 4 (code/Ob_propagation.py:166)"); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  const int C = T * d_ob, K = E / 2;
  const BLay l = blayout(N, T, d_ob, E);
  float* sc = (float*)scratch;
  float* Hn = sc + l.Hn; float* V = sc + l.V; float* beta = sc + l.beta; float* score = sc + l.score;
  int* rank = (int*)(sc + l.rank);
  GemmP g;
  g.A = x; g.ta = 0; g.sAi = C; g.sAk = 1; g.B = increase_dim_w; g.tb = 1; g.sBj = C; g.sBk = 1;
  g.C = Hn; g.sCi = 8 * C; g.sCj = 1; g.M = N; g.N = 8 * C; g.K = C; g.bias = increase_dim_b;
  RD_TRY(gemm(g, st));
  g.B = value_w; g.C = V; g.sCi = C; g.N = C; g.bias = value_b; g.relu = 1;
  RD_TRY(gemm(g, st));
  beta_node_kernel<<<(unsigned)ceil_div((int64_t)N * T, 256), 256, 0, st>>>(Hn, map_weights, p_t, N, T, beta);
  RD_CHECK_LAUNCH("beta_node_kernel");
  edge_score_kernel<<<(unsigned)ceil_div((int64_t)E * 32, 256), 256, 0, st>>>(beta, edge_tgt, edge_w, E, T, d_ob, score);
  RD_CHECK_LAUNCH("edge_score_kernel");
  rank_and_prune_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(score, edge_src, edge_tgt, E, K, rank, edge_src_out,
                                                                   edge_tgt_out, alpha_out, nullptr);
  RD_CHECK_LAUNCH("rank_and_prune_kernel");
  beta_aggregate_kernel<<<N, 256, 0, st>>>(V, beta, edge_src, edge_tgt, edge_w, rank, E, K, C, T, d_ob, out);
  RD_CHECK_LAUNCH("beta_aggregate_kernel");
  return 0;
}
