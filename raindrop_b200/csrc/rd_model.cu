// Host-side orchestration of the Raindrop_v2 hot path and the C ABI (include/raindrop_b200.h).
//
// Data layout in HBM (all fp32, row-major, 256-byte aligned sub-buffers of one caller-provided
// workspace so that nothing is allocated between forward and backward):
//   X0, H1          [B*N, C]   sensor-major rows, C = T*d_ob  (observation propagation operands)
//   Z[l]            [T, B, D]  encoder layer inputs/outputs, seq-first exactly like the reference
//   qkv, ctx, r1, x1, f, r2    per encoder layer, token-major [T*B, .]
//   P (and Pd)      [B, H, T, T] attention probabilities (and their dropped copy when training)
#include <math.h>
#include <string.h>

#include "rd_kernels.cuh"
#include "rd_obprop_tc.cuh"
#include "rd_tc_gemm.cuh"

namespace rd {
int grad_lo_image(const float* G, long long n, float* lo, cudaStream_t st);     // rd_influence.cu
namespace {

struct Shape {
  int B, T, N, dob, H, nhid, L, ds, ncls;
  int C, Dm, D, Df, hd, dpe, emb;
  int64_t M1, M2;
  float p;  // effective dropout probability (0 in eval)
  int tc, exact;   // ob-prop layers: tensor-core kernel usable / error-compensated (3xTF32) mode chosen
};

int make_shape(const rd_dims* d, Shape* s) {
  if (!d) { set_error("dims is NULL"); return -2; }
  s->B = d->B; s->T = d->T; s->N = d->N; s->dob = d->d_ob; s->H = d->nhead; s->nhid = d->nhid;
  s->L = d->nlayers; s->ds = d->d_static; s->ncls = d->n_classes;
  if (s->B < 1 || s->T < 1 || s->N < 1 || s->dob < 1 || s->H < 1 || s->nhid < 1 || s->L < 1 ||
      s->L > RD_MAX_LAYERS || s->ncls < 1 || s->ds < 0) {
    set_error("invalid dims (B=%d T=%d N=%d d_ob=%d nhead=%d nhid=%d nlayers=%d d_static=%d n_classes=%d)",
              s->B, s->T, s->N, s->dob, s->H, s->nhid, s->L, s->ds, s->ncls);
    return -2;
  }
  s->dpe = d->d_pe > 0 ? d->d_pe : RD_D_PE;
  s->emb = d->emb_dim > 0 ? d->emb_dim : s->N;
  if (s->dpe > 64 || (s->dpe & 3)) { set_error("d_pe = %d must be a multiple of 4 and <= 64", s->dpe); return -2; }
  s->C = s->T * s->dob; s->Dm = s->N * s->dob; s->D = s->Dm + s->dpe;
  if (s->D % s->H != 0) { set_error("d_model+16 = %d not divisible by nhead = %d", s->D, s->H); return -2; }
  s->hd = s->D / s->H;
  s->Df = s->D + (s->ds > 0 ? s->emb : 0);
  s->M1 = (int64_t)s->B * s->N; s->M2 = (int64_t)s->T * s->B;
  s->p = (d->training && d->dropout_p > 0.f) ? d->dropout_p : 0.f;
  if (s->p >= 1.f) { set_error("dropout_p must be < 1"); return -2; }
  if (d->obprop_mode < 0 || d->obprop_mode > 2) { set_error("obprop_mode must be 0 (auto), 1 (tf32) or 2 (3xtf32)"); return -2; }
  s->tc = obprop_tc_supported(s->C) ? 1 : 0;
  s->exact = (s->tc && obprop_tc_exact(s->M1, s->C, d->obprop_mode)) ? 1 : 0;
  return 0;
}

// Raindrop_v2 embeds positions in d_pe = 16 columns and the statics in d_inp: the only embedding its entry points take.
int check_raindrop_v2(const char* fn, const Shape& s) {
  if (s.dpe == RD_D_PE && s.emb == s.N) return 0;
  set_error("%s: Raindrop_v2 has d_pe = 16 and emb_dim = d_inp", fn);
  return -2;
}

// The checks every Raindrop_v2 model entry point makes before it writes anything: dims, params, lengths and node_scale
// not NULL, dims->training == 0 when `eval` (the entry point runs eval arithmetic), a valid Raindrop_v2 shape, and
// statics when d_static > 0.  The caller checks its own pointer arguments after these.
int check_model_call(const char* fn, const rd_dims* dims, const rd_params* params, const int64_t* lengths,
                     const float* node_scale, const float* statics, bool eval, Shape* s) {
  if (!dims || !params || !lengths || !node_scale) { set_error("%s: NULL argument", fn); return -2; }
  if (eval && dims->training) { set_error("%s: runs eval arithmetic, dims->training must be 0", fn); return -2; }
  RD_TRY(make_shape(dims, s));
  RD_TRY(check_raindrop_v2(fn, *s));
  if (s->ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  return 0;
}

struct Arena {
  int64_t off = 0;  // floats
  int64_t take(int64_t n) { int64_t o = off; off += round_up(n > 0 ? n : 1, 64); return o; }
};

struct WsLayout {
  int64_t rng, cnt, loss_ps, X0, H1, W1r, W2r, W2t, W1lo, W2lo, W2tlo, Z[RD_MAX_LAYERS + 1], feat, hpre, total;
  struct { int64_t qkv, P, Pd, ctx, r1, st1, x1, f, r2, st2, m1, m2; } l[RD_MAX_LAYERS];   // m1, m2: dropout keep bits of r1, r2
  // error-compensation remainders and transposes of the encoder weights (rd_tc_gemm.cuh)
  struct { int64_t in_lo, in_t, in_tlo, out_lo, out_t, out_tlo, l1_lo, l1_t, l1_tlo, l2_lo, l2_t, l2_tlo; } wsp[RD_MAX_LAYERS];
};

WsLayout ws_layout(const Shape& s) {
  WsLayout w;
  Arena a;
  w.rng = a.take(4);
  w.cnt = a.take(64);                   // ticket word of the fused loss reduction (zeroed by the step prologue)
  w.loss_ps = a.take(s.B);              // per-sample cross-entropy terms
  w.X0 = a.take(s.M1 * s.C);
  w.H1 = a.take(s.M1 * s.C);
  w.W1r = a.take((int64_t)s.C * s.C);   // TF32-rounded copies of the two lin_value weights
  w.W2r = a.take((int64_t)s.C * s.C);
  w.W2t = a.take((int64_t)s.C * s.C);   // (rounded) W2^T for the backward d(input) GEMM
  const int64_t nlo = s.exact ? (int64_t)s.C * s.C : 0;     // error-compensated mode: remainders of W1, W2, W2^T
  w.W1lo = a.take(nlo); w.W2lo = a.take(nlo); w.W2tlo = a.take(nlo);
  for (int i = 0; i <= s.L; ++i) w.Z[i] = a.take(s.M2 * s.D);
  // the T x T probabilities only reach HBM on the long-sequence path (the fused short-sequence kernels
  // keep them in shared memory and recompute them in backward)
  const int64_t pp = attn_small_supported(s.T, s.hd) ? 0 : (int64_t)s.B * s.H * s.T * s.T;
  for (int i = 0; i < s.L; ++i) {
    w.l[i].qkv = a.take(s.M2 * 3 * s.D);
    w.l[i].P = a.take(pp);
    w.l[i].Pd = a.take(s.p > 0.f ? pp : 0);
    w.l[i].ctx = a.take(s.M2 * s.D);
    w.l[i].r1 = a.take(s.M2 * s.D);
    w.l[i].st1 = a.take(s.M2 * 2);
    w.l[i].x1 = a.take(s.M2 * s.D);
    w.l[i].f = a.take(s.M2 * s.nhid);
    w.l[i].r2 = a.take(s.M2 * s.D);
    w.l[i].st2 = a.take(s.M2 * 2);
    const int64_t mw = s.p > 0.f ? s.M2 * ((s.D + 31) / 32) : 0;     // one 32-bit word per 32 columns
    w.l[i].m1 = a.take(mw); w.l[i].m2 = a.take(mw);
    const int64_t nin = 3LL * s.D * s.D, nout = (int64_t)s.D * s.D, nff = (int64_t)s.nhid * s.D;
    w.wsp[i].in_lo = a.take(nin); w.wsp[i].in_t = a.take(nin); w.wsp[i].in_tlo = a.take(nin);
    w.wsp[i].out_lo = a.take(nout); w.wsp[i].out_t = a.take(nout); w.wsp[i].out_tlo = a.take(nout);
    w.wsp[i].l1_lo = a.take(nff); w.wsp[i].l1_t = a.take(nff); w.wsp[i].l1_tlo = a.take(nff);
    w.wsp[i].l2_lo = a.take(nff); w.wsp[i].l2_t = a.take(nff); w.wsp[i].l2_tlo = a.take(nff);
  }
  w.feat = a.take((int64_t)s.B * s.Df);
  w.hpre = a.take((int64_t)s.B * s.Df);
  w.total = a.off;
  return w;
}

// ---- the trained tensors ------------------------------------------------------------------------------------------
// Every trained tensor, in flat-bucket order (TrainStep's layout, used_param_fields in functional.py), each at a
// 4-aligned offset: the head (emb when d_static > 0, mlp_static.0, mlp_static.2; dp_head_sqnorm_kernel and psg_head in
// rd_dp.cu number these fields themselves, in this order), 12 per encoder layer (in_proj, out_proj, linear1, linear2,
// norm1, norm2; weight then bias), the lin_value pairs of ob-prop layers 1 and 2.  A linear's bias field follows its
// weight, and ord numbers the linears in the same order (the backward's partial buffer, the EK-FAC block).  Sample b's
// R rows of a linear's operands are b*sstride + t*rstride, t < R; ob: the ob-prop phase queues it.  EK-FAC block:
// offsets a, s (doubles) of A [(Kin + 1)^2] and S [Nout^2] in the factors, qs, qa, qb (floats) of Q_S^T [Nout, Nout],
// Q_A[:Kin]^T [Np, Kin] and Q_A[Kin] [Np] in the bases, Np = Kin + 1 rounded up to 4 (rows past Kin + 1 are 0).
enum Role { IN_PROJ, OUT_PROJ, LINEAR1, LINEAR2 };     // an encoder layer's linears, in bucket order
struct Linear { int Nout, Kin, R, fw, ord, ob, Np; int64_t rows, sstride, rstride, a, s, qs, qa, qb; };
struct Trained {
  DpFields f;                          // bucket offset and size of every field
  int64_t bucket;                      // the bucket length
  float* grad[DP_MAX_FIELDS];          // each field's rd_grads member (NULL when built without one)
  Linear lin[4 * RD_MAX_LAYERS + 2];   // lin[ord]
  int nlin, L;
  int norm1[RD_MAX_LAYERS], norm2[RD_MAX_LAYERS];   // weight fields of encoder layer l's LayerNorms
  int64_t factor_doubles, base_floats;              // EK-FAC factors and bases of all blocks
  const Linear& layer(int l, Role r) const { return lin[4 * l + r]; }
  const Linear& obprop(int k) const { return lin[4 * L + k - 1]; }   // lin_value of ob-prop layer k = 1, 2
};

const rd_grads kNoGrads = {};

Trained trained(const Shape& s, const rd_grads* G = nullptr) {
  const rd_grads& g = G ? *G : kNoGrads;
  Trained t;
  t.f.n = 0; t.bucket = 0; t.nlin = 0; t.L = s.L; t.factor_doubles = 0; t.base_floats = 0;
  auto field = [&](int64_t numel, float* grad) {
    t.f.off[t.f.n] = t.bucket; t.f.numel[t.f.n] = numel; t.grad[t.f.n] = grad;
    t.bucket += round_up(numel, 4);
    return t.f.n++;
  };
  auto linear = [&](int Nout, int Kin, int ob, float* gw, float* gb) {
    Linear& o = t.lin[t.nlin];
    o.Nout = Nout; o.Kin = Kin; o.ord = t.nlin++; o.ob = ob;
    o.R = ob ? s.N : s.T; o.sstride = ob ? s.N : 1; o.rstride = ob ? 1 : s.B; o.rows = (int64_t)s.B * o.R;
    o.fw = field((int64_t)Nout * Kin, gw); field(Nout, gb);
    o.Np = (int)round_up(Kin + 1, 4);     // each EK-FAC piece starts 4-aligned
    o.a = t.factor_doubles; t.factor_doubles += (int64_t)(Kin + 1) * (Kin + 1);
    o.s = t.factor_doubles; t.factor_doubles += (int64_t)Nout * Nout;
    o.qs = t.base_floats; t.base_floats += round_up((int64_t)Nout * Nout, 4);
    o.qa = t.base_floats; t.base_floats += (int64_t)o.Np * Kin;
    o.qb = t.base_floats; t.base_floats += o.Np;
  };
  if (s.ds > 0) { field((int64_t)s.emb * s.ds, g.emb_weight); field(s.emb, g.emb_bias); }
  field((int64_t)s.Df * s.Df, g.mlp0_weight); field(s.Df, g.mlp0_bias);
  field((int64_t)s.ncls * s.Df, g.mlp2_weight); field(s.ncls, g.mlp2_bias);
  for (int l = 0; l < s.L; ++l) {
    const rd_encoder_layer_grads& e = g.layer[l];
    linear(3 * s.D, s.D, 0, e.in_proj_weight, e.in_proj_bias);
    linear(s.D, s.D, 0, e.out_proj_weight, e.out_proj_bias);
    linear(s.nhid, s.D, 0, e.linear1_weight, e.linear1_bias);
    linear(s.D, s.nhid, 0, e.linear2_weight, e.linear2_bias);
    t.norm1[l] = field(s.D, e.norm1_weight); field(s.D, e.norm1_bias);
    t.norm2[l] = field(s.D, e.norm2_weight); field(s.D, e.norm2_bias);
  }
  linear(s.C, s.C, 1, g.ob1_value_weight, g.ob1_value_bias);
  linear(s.C, s.C, 1, g.ob2_value_weight, g.ob2_value_bias);
  return t;
}

// the larger of the two backward phases' sums of cost(linear)
template <class F> int64_t phase_max(const Trained& t, F cost) {
  int64_t sum[2] = {0, 0};
  for (int i = 0; i < t.nlin; ++i) sum[t.lin[i].ob] += cost(t.lin[i]);
  return sum[0] > sum[1] ? sum[0] : sum[1];
}

// Backward scratch.  The weight gradients are DEFERRED: every linear layer's (dY, X) operand pair stays alive in
// its own buffer until one grouped tensor-core launch (tc_wgrad_group) reduces them all, so dY buffers and the
// split-K partial buffers are per layer / per problem instead of ping-pong.
struct BwLayout {
  int64_t dfeat, dhpre, gA, gB, gD, dP, gO2, gO1, partial, total;
  struct { int64_t K2, gF, K1, dqkv, ln[2]; } l[RD_MAX_LAYERS];   // ln: norm2, norm1
  int64_t wp[4 * RD_MAX_LAYERS + 2];   // tensor-core partial buffer of each linear, by ord
};

int64_t splitk_partial_floats(int Nout, int Kin, int64_t rows) {
  int ns;
  return gemm_splitk_plan(Nout, Kin, (int)rows, &ns);
}

BwLayout bw_layout(const Shape& s) {
  const Trained t = trained(s);
  BwLayout b;
  Arena a;
  auto wp = [&](const Linear& o) { b.wp[o.ord] = a.take(tc_wgrad_partial_floats(o.Nout, o.Kin, o.rows)); };
  b.dfeat = a.take((int64_t)s.B * s.Df);
  b.dhpre = a.take((int64_t)s.B * s.Df);
  b.gA = a.take(s.M2 * s.D);
  b.gB = a.take(s.M2 * s.D);
  b.gD = a.take(s.M2 * s.D);
  b.dP = a.take(attn_small_supported(s.T, s.hd) ? 0 : (int64_t)s.B * s.H * s.T * s.T);
  for (int l = 0; l < s.L; ++l) {
    b.l[l].K2 = a.take(s.M2 * s.D);
    b.l[l].gF = a.take(s.M2 * s.nhid);
    b.l[l].K1 = a.take(s.M2 * s.D);
    b.l[l].dqkv = a.take(s.M2 * 3 * s.D);
    wp(t.layer(l, LINEAR2)); wp(t.layer(l, LINEAR1)); wp(t.layer(l, OUT_PROJ)); wp(t.layer(l, IN_PROJ));
    b.l[l].ln[0] = a.take(ln_bwd_scratch_floats(s.M2, s.D));      // per-CTA dgamma/dbeta partial rows, reduced with the group
    b.l[l].ln[1] = a.take(ln_bwd_scratch_floats(s.M2, s.D));
  }
  b.gO2 = a.take(s.M1 * s.C);
  b.gO1 = a.take(s.M1 * s.C);
  wp(t.obprop(2)); wp(t.obprop(1));
  // shared split-K scratch of the CUDA-core fallback (shapes the tensor-core kernel does not take)
  int64_t pf = 0;
  for (int i = 0; i < t.nlin; ++i) { const int64_t v = splitk_partial_floats(t.lin[i].Nout, t.lin[i].Kin, t.lin[i].rows); if (v > pf) pf = v; }
  b.partial = a.take(pf);
  b.total = a.off;
  return b;
}

// CTAs (= partial pairs) of the larger of the two phases' group launches
int64_t dp_partial_blocks(const Shape& s) {
  int tm, tn;
  return (int64_t)s.B * phase_max(trained(s), [&](const Linear& o) {
    return (int64_t)dp_norm_tiles(o.R, o.Nout, o.Kin, dp_ghost(o.R, o.Nout, o.Kin), &tm, &tn);
  });
}

// Scratch of rd_raindrop_v2_per_sample_grad_sqnorms: the backward scratch of the data-gradient chain, then the partial
// sums (2 doubles per CTA of a group launch)
struct DpLayout { int64_t bw, partial, total; };
DpLayout dp_layout(const Shape& s) {
  DpLayout l;
  Arena a;
  l.bw = a.take(bw_layout(s).total);
  l.partial = a.take(4 * dp_partial_blocks(s));
  l.total = a.off;
  return l;
}

// Scratch of rd_raindrop_v2_input_grad: W1^T with its error-compensation remainder, and dX0 = d(loss)/d(X0) [B*N, C]
struct IgLayout { int64_t W1t, W1tlo, dX0, total; };
IgLayout input_grad_layout(const Shape& s) {
  IgLayout l;
  Arena a;
  l.W1t = a.take((int64_t)s.C * s.C);
  l.W1tlo = a.take((int64_t)s.C * s.C);
  l.dX0 = a.take(s.M1 * s.C);
  l.total = a.off;
  return l;
}

// ---- chunked drivers ------------------------------------------------------------------------------------------------
// Integrated gradients, PGD, coalition attribution, KernelSHAP, Monte Carlo dropout and smoothing run the model on chunks
// of rows expanded from the batch.  The arithmetic of a chunk's ob-prop GEMMs is resolved once, from the row count
// pin_rows of a FULL chunk (obprop_mode 0 depends on it), and every chunk and endpoint forward runs with that explicit
// mode: a ragged tail chunk with fewer rows cannot switch arithmetic.
rd_dims chunk_dims(const rd_dims* d, int rows, int64_t pin_rows, int training) {
  rd_dims e = *d;
  e.obprop_mode = obprop_tc_exact(pin_rows * d->N, d->T * d->d_ob, d->obprop_mode) ? 2 : 1;
  e.B = rows;
  e.training = training;
  return e;
}

// The expanded inputs of a chunk; statics is nullptr without a static branch.
struct Expanded { float* src; float* statics; float* times; int64_t* lengths; };

// Scratch of a chunked driver whose chunk is n units of `per` rows (`what` names n in the range check): the forward
// workspace and the expanded inputs of the forward's rows (the chunk's, or at least 2B with an endpoint forward), the
// chunk's logits and, when the chunk runs a backward, its backward scratch, W1^T with its remainder, dX0 and d_logits.
// A driver takes its own pieces from `a` after these.
struct ChunkLayout {
  Arena a;
  int64_t ws, sc, W1t, W1tlo, dX0, dlogits, src, statics, times, lengths, logits;
  Expanded inputs(float* S, int ds) const {
    return {S + src, ds > 0 ? S + statics : nullptr, S + times, reinterpret_cast<int64_t*>(S + lengths)};
  }
};
int chunk_layout(const rd_dims* dims, const char* what, int n, int per, bool endpoints, int training, bool bwd,
                 ChunkLayout* l) {
  if (n < 1 || (int64_t)per * n > (1LL << 30)) { set_error("%s = %d out of range", what, n); return -2; }
  const int rows = per * n, fwd_rows = endpoints && rows < 2 * dims->B ? 2 * dims->B : rows;
  const rd_dims dc = chunk_dims(dims, rows, rows, training), dx = chunk_dims(dims, fwd_rows, rows, training);
  Shape sc, sx;
  RD_TRY(make_shape(&dc, &sc));
  RD_TRY(make_shape(&dx, &sx));
  Arena& a = l->a;
  l->ws = a.take(ws_layout(sx).total);
  if (bwd) {
    l->sc = a.take(bw_layout(sc).total);
    l->W1t = a.take((int64_t)sc.C * sc.C);
    l->W1tlo = a.take((int64_t)sc.C * sc.C);
    l->dX0 = a.take(sc.M1 * sc.C);
    l->dlogits = a.take((int64_t)rows * sc.ncls);
  }
  l->src = a.take(sx.M2 * 2 * sx.N);
  l->statics = a.take((int64_t)fwd_rows * sx.ds);
  l->times = a.take(sx.M2);
  l->lengths = a.take(2LL * fwd_rows);
  l->logits = a.take((int64_t)rows * sx.ncls);
  return 0;
}

// Integrated gradients: chunks of mc path steps (B*mc rows) with a backward, the endpoint forward on 2B rows, and the
// running sums [B*N*T] and [B, d_static].
struct IgScratch : ChunkLayout { int64_t acc_src, acc_static; };
int ig_scratch(const rd_dims* dims, int mc, IgScratch* l) {
  RD_TRY(chunk_layout(dims, "steps_per_chunk", mc, dims->B, true, 0, true, l));
  l->acc_src = l->a.take((int64_t)dims->B * dims->N * dims->T);
  l->acc_static = l->a.take((int64_t)dims->B * dims->d_static);
  return 0;
}

// PGD: chunks of spc samples with a backward, the perturbation and l2 gradient [spc, T*N + ds] and the best losses (fp64).
struct PgdScratch : ChunkLayout { int64_t delta, grad, best; };
int pgd_scratch(const rd_dims* dims, int spc, PgdScratch* l) {
  RD_TRY(chunk_layout(dims, "samples_per_chunk", spc, 1, false, 0, true, l));
  const int64_t E = (int64_t)dims->T * dims->N + dims->d_static;
  l->delta = l->a.take(spc * E);
  l->grad = l->a.take(spc * E);
  l->best = l->a.take(2LL * spc);
  return 0;
}

// Counterfactuals: chunks of spc samples on spc*R rows with a backward, the deltas of x_k and y_k [spc*R, T*N + ds], the
// per-row state [spc*R, CF_ROW] and the per-sample best distances (fp64).
struct CfScratch : ChunkLayout { int64_t xd, yd, row, best; };
int cf_scratch(const rd_dims* dims, int spc, int R, CfScratch* l) {
  if (R < 1) { set_error("n_restarts = %d must be >= 1", R); return -2; }
  RD_TRY(chunk_layout(dims, "samples_per_chunk", spc, R, false, 0, true, l));
  const int64_t rows = (int64_t)spc * R, E = (int64_t)dims->T * dims->N + dims->d_static;
  l->xd = l->a.take(rows * E);
  l->yd = l->a.take(rows * E);
  l->row = l->a.take(2 * rows * CF_ROW);
  l->best = l->a.take(2LL * spc);
  return 0;
}

// Coalition attribution (Shapley-value sampling, ablation, KernelSHAP): chunks of cc coalitions (B*cc rows), the
// endpoint forward on 2B rows, the fp64 running sums [B, P] and the chunk's keep table [cc, P] (uint8, Shapley).
struct CoalScratch : ChunkLayout { int64_t acc, keep; };
int coalition_scratch(const rd_dims* dims, int n_players, int cc, CoalScratch* l) {
  RD_TRY(chunk_layout(dims, "coalitions_per_chunk", cc, dims->B, true, 0, false, l));
  if (n_players < 1) { set_error("n_players = %d must be >= 1", n_players); return -2; }
  l->acc = l->a.take(2LL * dims->B * n_players);
  l->keep = l->a.take(ceil_div((int64_t)cc * n_players, 4));
  return 0;
}

// Monte Carlo dropout: chunks of cc replicates (B*cc rows, training forwards) and the fp64 sums [B, 2*n_classes + 1].
struct McScratch : ChunkLayout { int64_t acc; };
int mc_scratch(const rd_dims* dims, int cc, McScratch* l) {
  RD_TRY(chunk_layout(dims, "replicates_per_chunk", cc, dims->B, false, 1, false, l));
  l->acc = l->a.take(2LL * dims->B * (2 * dims->n_classes + 1));
  return 0;
}

// Y[M,N] = epi(X[M,K] . W[N,K]^T)
GemmP nt(const float* X, int64_t ldx, const float* W, int64_t ldw, float* Y, int64_t ldy, int64_t M, int N, int K) {
  GemmP g;
  g.A = X; g.ta = 0; g.sAi = ldx; g.sAk = 1;
  g.B = W; g.tb = 1; g.sBj = ldw; g.sBk = 1;
  g.C = Y; g.sCi = ldy; g.sCj = 1;
  g.M = (int)M; g.N = N; g.K = K;
  return g;
}
// dX[M,Kin] = epi(dY[M,Nout] . W[Nout,Kin])
GemmP nn(const float* dY, int64_t ldy, const float* W, int64_t ldw, float* dX, int64_t ldx, int64_t M, int Kin, int Nout) {
  GemmP g;
  g.A = dY; g.ta = 0; g.sAi = ldy; g.sAk = 1;
  g.B = W; g.tb = 0; g.sBk = ldw; g.sBj = 1;
  g.C = dX; g.sCi = ldx; g.sCj = 1;
  g.M = (int)M; g.N = Kin; g.K = Nout;
  return g;
}
// dW[Nout,Kin] = sum_r dY[r,Nout]^T X[r,Kin], db = sum_r dY[r,:]: queued for the next grouped tensor-core launch when
// the shape fits, else done right away on the CUDA cores (split over rows, deterministic two-stage reduce).
struct WgradQueue {
  WgradItem it[WG_MAX];
  ColsumItem cs[CS_MAX];
  int n = 0, ncs = 0;
  int flush(cudaStream_t st) {
    if (n == 0 && ncs == 0) return 0;
    int rc = tc_wgrad_group(it, n, cs, ncs, st);
    n = 0; ncs = 0;
    return rc;
  }
  // out[c] = sum over the chunks of partial[chunk*stride + c]: reduced by the group's reduction launch
  int colsum(const float* partial, long long stride, int nsplit, int ncols, float* out, cudaStream_t st) {
    if (ncs == CS_MAX) RD_TRY(flush(st));
    cs[ncs++] = ColsumItem{partial, stride, nsplit, ncols, out};
    return 0;
  }
};

int tn(WgradQueue* q, const float* dY, int64_t ldy, const float* X, int64_t ldx, float* dW, float* db, int Nout, int Kin,
       int64_t rows, float* tc_partial, float* partial, cudaStream_t st) {
  if (rows >= 256 && tc_partial && tc_wgrad_supported(Nout, Kin, ldy, ldx, dY, X)) {
    if (q) {
      if (q->n == WG_MAX) RD_TRY(q->flush(st));
      q->it[q->n++] = WgradItem{dY, ldy, X, ldx, rows, Nout, Kin, dW, db, tc_partial};
      return 0;
    }
    return tc_wgrad(dY, ldy, X, ldx, rows, Nout, Kin, dW, db, tc_partial, st);
  }
  GemmP g;
  g.A = dY; g.ta = 1; g.sAk = ldy; g.sAi = 1;
  g.B = X; g.tb = 0; g.sBk = ldx; g.sBj = 1;
  g.C = dW; g.sCi = Kin; g.sCj = 1;
  g.M = Nout; g.N = Kin; g.K = (int)rows;
  int ns;
  gemm_splitk_plan(Nout, Kin, (int)rows, &ns);
  g.nsplit = ns; g.partial = partial;
  g.asum = db;   // db[n] = sum_r dY[r, n] comes out of the same pass
  return gemm(g, st);
}

}  // namespace

// Y[M,N] = epi(X[M,K] . W[N,K]^T): error-compensated tensor-core GEMM when the shape allows it, else CUDA cores.
static int linear_nt(const GemmP& g, const float* W_lo, cudaStream_t st) {
  TcGemmArgs a;
  a.A = g.A; a.lda = g.sAi; a.B = g.B; a.B_lo = W_lo; a.M = g.M; a.N = g.N; a.K = g.K; a.C = g.C;
  a.bias = g.bias; a.relu = g.relu; a.gate = g.gate; a.gate_ld = g.gate_ld; a.gate_scale = g.gate_scale;
  a.drop_p = g.drop_p; a.rng = g.rng; a.drop_site = g.drop_site; a.resid = g.resid; a.resid_ld = g.resid_ld;
  a.drop_mask = g.drop_mask; a.drop_mask_ld = g.drop_mask_ld; a.rep = g.rep;
  const bool plain = g.ta == 0 && g.tb == 1 && g.sBj == g.K && g.sCi == g.N && g.sCj == 1 && g.nz == 1 && g.nsplit == 1 &&
                     g.alpha == 1.f && !g.rowscale && !g.perm && !g.asum;
  if (plain && W_lo && tc_gemm_supported(a)) return tc_gemm(a, st);
  return gemm(g, st);
}

// The predicate of linear_nt for a plain y = x W^T GEMM: the backward calls it with the forward's operands to know
// whether the forward's epilogue stored the dropout keep bits (only the tensor-core kernel does).
static bool linear_nt_is_tc(const GemmP& g, const float* W_lo) {
  TcGemmArgs a;
  a.A = g.A; a.lda = g.sAi; a.B = g.B; a.B_lo = W_lo; a.M = g.M; a.N = g.N; a.K = g.K; a.C = g.C;
  a.bias = g.bias; a.relu = g.relu; a.gate = g.gate; a.gate_ld = g.gate_ld; a.gate_scale = g.gate_scale;
  a.drop_p = g.drop_p; a.rng = g.rng; a.drop_site = g.drop_site; a.resid = g.resid; a.resid_ld = g.resid_ld;
  return W_lo && tc_gemm_supported(a);
}

// ---- the backward's gradient consumer ------------------------------------------------------------------------------
namespace {
// raindrop_bwd hands each linear's (dY, X) operand pair, each LayerNorm and the head to one consumer, whose mode says
// what becomes of them: NONE nothing (the data-gradient chain alone: frozen parameters); WEIGHTS the weight gradients
// into `grads`, items of one grouped tensor-core launch (tn, WgradQueue; head_bwd writes the head's); SQNORMS DP-SGD's
// per-sample squared norms; ROWS TracIn's per-sample gradient rows into G, times `scale`; ROTATED the EK-FAC rows, each
// linear's operands rotated into the bases first; FACTORS the EK-FAC factor sums (none from LayerNorms and the head).
// The per-sample modes flush a phase's linears as one group launch at the end of every phase, which lays its buffers
// (`partial`, `kws`, `rot`) out from their start again: the previous phase's launches have completed (stream order).
enum GradMode { GRAD_NONE, GRAD_WEIGHTS, GRAD_SQNORMS, GRAD_ROWS, GRAD_ROTATED, GRAD_FACTORS };
struct GradConsumer {
  GradMode mode = GRAD_NONE;
  const rd_grads* grads = nullptr;                                                      // WEIGHTS
  double* sqnorms = nullptr; double* partial = nullptr;                                 // SQNORMS
  float* G = nullptr; float scale = 1.f;                                                // ROWS, ROTATED (ldg = the bucket length)
  const float* bases = nullptr; const float* bases_lo = nullptr; float* rot = nullptr;  // ROTATED
  double* factors = nullptr; float* kws = nullptr; float* kpartial = nullptr;           // FACTORS
  // set by raindrop_bwd: the shape, its trained tensors (built with `grads`) and the backward scratch
  const Shape* s = nullptr; const Trained* t = nullptr; const BwLayout* b = nullptr; float* sc = nullptr;
  WgradQueue wq;
  struct Item { const Linear* o; const float* Y; const float* X; } it[DP_MAX_ITEMS];   // a per-sample mode's phase
  int n = 0;

  int linear(const Linear& o, const float* Y, const float* X, cudaStream_t st) {
    if (mode == GRAD_WEIGHTS)
      return tn(&wq, Y, o.Nout, X, o.Kin, t->grad[o.fw], t->grad[o.fw + 1], o.Nout, o.Kin, o.rows, sc + b->wp[o.ord], sc + b->partial, st);
    if (mode != GRAD_NONE) it[n++] = Item{&o, Y, X};
    return 0;
  }

  // LayerNorm with weight field fw over the T*B rows of its input x, stats {mean, rstd} and output gradient dy; part:
  // layernorm_bwd's deferred per-CTA partial rows [chunks][2][D]
  int ln(int fw, const float* part, int chunks, const float* x, const float* stats, const float* dy, cudaStream_t st) {
    const int D = s->D;
    if (mode == GRAD_WEIGHTS) {
      RD_TRY(wq.colsum(part, 2 * D, chunks, D, t->grad[fw], st));
      return wq.colsum(part + D, 2 * D, chunks, D, t->grad[fw + 1], st);
    }
    if (mode == GRAD_SQNORMS) return dp_ln_sqnorm(x, stats, dy, s->T, s->B, D, sqnorms, t->f.n, fw, fw + 1, st);
    if (mode != GRAD_ROWS && mode != GRAD_ROTATED) return 0;
    return psg_ln(x, stats, dy, s->T, s->B, D, G, t->bucket, t->f.off[fw], t->f.off[fw + 1], scale, st);
  }

  int head(const float* dlogits, const float* hpre, const float* dh, const float* feat, const float* dfeat,
           const float* statics, cudaStream_t st) {
    const Shape& z = *s;
    if (mode == GRAD_SQNORMS)
      return dp_head_sqnorm(z.B, z.D, z.Df, z.ds, z.ncls, dlogits, hpre, dh, feat, dfeat, statics, sqnorms, t->f.n, st);
    if (mode != GRAD_ROWS && mode != GRAD_ROTATED) return 0;
    return psg_head(z.B, z.D, z.Df, z.ds, z.ncls, dlogits, hpre, dh, feat, dfeat, statics, G, t->bucket, t->f.off, scale, st);
  }

  // The end of a backward phase.  Weights mode keeps its items when the ob-prop phase follows, so that the encoder's
  // last items share the ob-prop items' group launch.
  int flush(bool obprop_follows, cudaStream_t st) {
    if (mode == GRAD_WEIGHTS) return obprop_follows ? 0 : wq.flush(st);
    const int rc = n == 0 ? 0 : mode == GRAD_SQNORMS ? sqnorm_group(st) : mode == GRAD_FACTORS ? factor_sums(st) : row_group(st);
    n = 0;
    return rc;
  }

  // every queued linear's per-sample squared norms: one dp_norm_group launch pair (B * ntiles CTAs per item, in order)
  int sqnorm_group(cudaStream_t st) {
    DpNormGroup g;
    long long blk = 0;
    for (g.n = 0; g.n < n; ++g.n) {
      const Linear& o = *it[g.n].o;
      DpNormItem& q = g.it[g.n];
      q.Y = it[g.n].Y; q.X = it[g.n].X; q.ldy = o.Nout; q.ldx = o.Kin; q.sstride = o.sstride; q.rstride = o.rstride; q.blk0 = blk;
      q.Nout = o.Nout; q.Kin = o.Kin; q.R = o.R; q.ghost = dp_ghost(o.R, o.Nout, o.Kin) ? 1 : 0;
      q.ntiles = dp_norm_tiles(o.R, o.Nout, o.Kin, q.ghost != 0, &q.tm, &q.tn);
      q.fw = o.fw; q.fb = o.fw + 1;
      blk += (long long)s->B * q.ntiles;
    }
    return dp_norm_group(g, s->B, partial, sqnorms, t->f.n, st);
  }

  // Every queued linear's per-sample gradient rows: one psg_group launch.  Rotated rows first turn each item into
  // Y^ = dY Q_S and X^ = [X | 1] Q_A on the error-compensated tensor-core GEMM (linear_nt, bias = the last row of Q_A),
  // and psg_group appends no ones column to them.
  int row_group(cudaStream_t st) {
    PsgGroup pg;
    long long blk = 0;
    int64_t off = 0;
    for (pg.n = 0; pg.n < n; ++pg.n) {
      const Linear& o = *it[pg.n].o;
      PsgItem& q = pg.it[pg.n];
      q.Y = it[pg.n].Y; q.X = it[pg.n].X; q.ldy = o.Nout; q.ldx = o.Kin;
      if (mode == GRAD_ROTATED) {
        float* yh = rot + off; off += round_up(o.rows * o.Nout, 64);
        float* xh = rot + off; off += round_up(o.rows * o.Np, 64);
        RD_TRY(linear_nt(nt(q.Y, o.Nout, bases + o.qs, o.Nout, yh, o.Nout, o.rows, o.Nout, o.Nout), bases_lo + o.qs, st));
        GemmP r = nt(q.X, o.Kin, bases + o.qa, o.Kin, xh, o.Np, o.rows, o.Np, o.Kin);
        r.bias = bases + o.qb;
        RD_TRY(linear_nt(r, bases_lo + o.qa, st));
        q.Y = yh; q.X = xh; q.ldx = o.Np;
      }
      q.sstride = o.sstride; q.rstride = o.rstride; q.blk0 = blk; q.gw = t->f.off[o.fw]; q.gb = t->f.off[o.fw + 1];
      q.Nout = o.Nout; q.Kin = o.Kin; q.R = o.R; q.ntiles = psg_tiles(o.Nout, o.Kin, &q.tn);
      blk += (long long)s->B * q.ntiles;
    }
    return psg_group(pg, s->B, G, t->bucket, scale, st, mode == GRAD_ROTATED);
  }

  // EK-FAC factors: per item, dW = X^T X with db = column sums of X, and dW = dY^T dY (tn: queued for one grouped
  // tensor-core launch when the shape fits, else CUDA cores), then each block's sums are added into the fp64 factors
  // (dY carries the gradient of l_b / B, so S is scaled by B^2).
  int factor_sums(cudaStream_t st) {
    int64_t off = 0;
    const float* Aw[DP_MAX_ITEMS]; const float* Ab[DP_MAX_ITEMS]; const float* Sw[DP_MAX_ITEMS];
    for (int i = 0; i < n; ++i) {
      const Linear& o = *it[i].o;
      float* aw = kws + off; off += round_up((int64_t)o.Kin * o.Kin, 64);
      float* ab = kws + off; off += round_up(o.Kin, 64);
      float* sw = kws + off; off += round_up((int64_t)o.Nout * o.Nout, 64);
      float* sb = kws + off; off += round_up(o.Nout, 64);
      float* pa = kws + off; off += round_up(tc_wgrad_partial_floats(o.Kin, o.Kin, o.rows), 64);
      float* ps = kws + off; off += round_up(tc_wgrad_partial_floats(o.Nout, o.Nout, o.rows), 64);
      RD_TRY(tn(&wq, it[i].X, o.Kin, it[i].X, o.Kin, aw, ab, o.Kin, o.Kin, o.rows, pa, kpartial, st));
      RD_TRY(tn(&wq, it[i].Y, o.Nout, it[i].Y, o.Nout, sw, sb, o.Nout, o.Nout, o.rows, ps, kpartial, st));
      Aw[i] = aw; Ab[i] = ab; Sw[i] = sw;
    }
    RD_TRY(wq.flush(st));
    for (int i = 0; i < n; ++i) {
      const Linear& o = *it[i].o;
      RD_TRY(kfac_accumulate(Aw[i], Ab[i], Sw[i], o.Kin, o.Nout, o.rows, (double)s->B * (double)s->B, factors + o.a, factors + o.s, st));
    }
    return 0;
  }
};

// Scratch of the factor pass: the backward scratch, then per block the fp32 sums X^T X, x, dY^T dY, dY colsums and two
// tensor-core partial buffers (factor_sums lays a phase's items out from the start of that region, in queue order), and
// the CUDA-core fallback's split-K partial buffer.
struct KfacLayout { int64_t bw, kws, kpartial, total; };
KfacLayout kfac_layout(const Shape& s) {
  KfacLayout l;
  Arena a;
  l.bw = a.take(bw_layout(s).total);
  const Trained t = trained(s);
  int64_t ws = 0, pf = 0;
  for (int i = 0; i < t.nlin; ++i) {
    const Linear& o = t.lin[i];
    ws += round_up((int64_t)o.Kin * o.Kin, 64) + round_up(o.Kin, 64) + round_up((int64_t)o.Nout * o.Nout, 64) +
          round_up(o.Nout, 64) + round_up(tc_wgrad_partial_floats(o.Kin, o.Kin, o.rows), 64) +
          round_up(tc_wgrad_partial_floats(o.Nout, o.Nout, o.rows), 64);
    const int64_t p1 = splitk_partial_floats(o.Kin, o.Kin, o.rows), p2 = splitk_partial_floats(o.Nout, o.Nout, o.rows);
    if (p1 > pf) pf = p1;
    if (p2 > pf) pf = p2;
  }
  l.kws = a.take(ws);
  l.kpartial = a.take(pf);
  l.total = a.off;
  return l;
}

// Scratch of the rotated rows: the backward scratch, the remainder image of the bases, and the rotated operands of the
// larger phase (every item of a phase is resident until its group launch).
struct EkfacLayout { int64_t bw, lo, rot, total; };
EkfacLayout ekfac_layout(const Shape& s) {
  EkfacLayout l;
  Arena a;
  l.bw = a.take(bw_layout(s).total);
  const Trained t = trained(s);
  l.lo = a.take(t.base_floats);
  l.rot = a.take(phase_max(t, [&](const Linear& o) { return round_up(o.rows * o.Nout, 64) + round_up(o.rows * o.Np, 64); }));
  l.total = a.off;
  return l;
}
}  // namespace

// ---- observation propagation layer (operator level) ---------------------------------------------
// Forward goes to the tensor-core kernel when the shape fits its tiling, otherwise to the generic
// CUDA-core GEMM (same epilogue).
static int obprop_forward(const ObpropTcArgs& a, cudaStream_t st) {
  if (obprop_tc_supported(a.C) && (!a.perm || a.pdob == 4)) return obprop_tc_fwd(a, st);
  GemmP g = nt(a.x, a.C, a.W, a.C, a.out, a.C, a.rows, a.C, a.C);
  g.bias = a.bias; g.relu = a.relu; g.rowscale = a.scale; g.rowscale_mod = a.scale_mod;
  g.gate = a.gate; g.gate_ld = a.C;
  g.perm = a.perm; g.pB = a.pB; g.pN = a.pN; g.pdob = a.pdob; g.pD = a.pD;
  return gemm(g, st);
}

// dX0 = gO1 . W1 [B*N, C]: on the tensor cores "NT" against W1^T (W1t / W1tlo from split_weights), always
// error-compensated since gO1 is not TF32-rounded in either mode; on the CUDA cores straight from W1
static int input_grad_dx0(const Shape& s, const rd_params* P, const float* gO1, const float* W1t, const float* W1tlo,
                          float* dX0, cudaStream_t st) {
  if (s.tc) {
    ObpropTcArgs a;
    a.x = gO1; a.W = W1t; a.W_lo = W1tlo; a.bias = nullptr; a.relu = 0; a.rows = s.M1; a.C = s.C; a.out = dX0;
    return obprop_tc_fwd(a, st);
  }
  return gemm(nn(gO1, s.C, P->ob1_value_weight, s.C, dX0, s.C, s.M1, s.C, s.C), st);
}

// rep_B > 0 (Monte Carlo dropout, training dims): the dims->B rows are replicate-major copies of a rep_B-row batch, row
// j = m*rep_B + b drawing the dropout words of row b of the rep_B-row forward at step (rng_state[1] + rep_step + m)
// (rep_remap); rng_state is read, never advanced.
static int raindrop_fwd(const rd_dims* dims, const rd_params* P, const float* src, const float* statics,
                        const float* times, const int64_t* lengths, const float* nscale, uint64_t* rng_state,
                        float* ws, float* logits, const int64_t* y, float* loss, float* d_logits, int encoder_only,
                        cudaStream_t st, int rep_B = 0, uint64_t rep_step = 0) {
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (!encoder_only) RD_TRY(check_raindrop_v2("rd_raindrop_v2_fwd", s));
  // a training forward is followed by a backward: refuse before any output is written or the rng counter moves.  Monte
  // Carlo replicates (rep_B > 0) are training forwards that no backward follows.
  if (dims->training && rep_B == 0 && !head_bwd_supported(s.Df)) {
    set_error("%s: training needs the head backward, feature width %d > 722", encoder_only ? "rd_encoder_head_fwd" : "rd_raindrop_v2_fwd",
              s.Df);
    return -2;
  }
  if (s.ds > 0 && (!statics || !P->emb_weight || !P->emb_bias)) { set_error("static branch needs statics/emb"); return -2; }
  WsLayout w = ws_layout(s);
  uint64_t* rng = reinterpret_cast<uint64_t*>(ws + w.rng);
  if (s.p > 0.f && !rng_state) { set_error("training with dropout needs rng_state"); return -2; }
  if (y && (!loss || !d_logits)) { set_error("labels given without loss / d_logits outputs"); return -2; }
  // rides along with the first weight-prep launch: dropout-stream capture (+ advance) and the loss ticket reset
  StepPrologue pro;
  if (s.p > 0.f) { pro.rng_state = rng_state; pro.rng_captured = rng; pro.advance = rep_B ? 0 : 1; pro.step_offset = rep_step; }
  DropRep rep;
  if (rep_B > 0 && s.B > rep_B && s.p > 0.f) { rep.B = rep_B; rep.Bc = s.B; }   // one replicate: the remap is the identity
  pro.zero_counter = reinterpret_cast<unsigned*>(ws + w.cnt);
  float* X0 = ws + w.X0; float* H1 = ws + w.H1;
  // Fast mode: tensor-core operands are kept exactly TF32-representable by their producers (lift, layer-1 epilogue,
  // rounded weight copies) so the MMA's operand truncation is exact.  Error-compensated mode (latency-bound row
  // counts): operands stay fp32, the weights come with their remainders, nothing is rounded.
  // No observation propagation on the encoder-only entry: no lin_value copies.  The workspace layout still follows the
  // shape's own tc / exact, as rd_workspace_bytes / rd_workspace_offset and the backward compute it.
  const int tc = encoder_only ? 0 : s.tc, exact = encoder_only ? 0 : s.exact;
  const float* W1 = P->ob1_value_weight; const float* W2 = P->ob2_value_weight;
  if (tc && !exact) { W1 = ws + w.W1r; W2 = ws + w.W2r; }   // rounded copies, produced by the weight-prep launch just below
  for (int l0 = 0; l0 < s.L; l0 += 3) {   // every derived weight tensor of the step in one launch (<= 16 tensors each)
    WeightSplit items[16];
    int n = 0;
    if (l0 == 0 && tc && !exact) {
      items[n] = {P->ob1_value_weight, s.C, s.C, nullptr, nullptr, nullptr}; items[n++].rn = ws + w.W1r;
      items[n] = {P->ob2_value_weight, s.C, s.C, nullptr, nullptr, nullptr}; items[n].rn = ws + w.W2r; items[n++].rn_t = ws + w.W2t;
    }
    if (l0 == 0 && exact) {
      items[n++] = {P->ob1_value_weight, s.C, s.C, ws + w.W1lo, nullptr, nullptr};
      items[n++] = {P->ob2_value_weight, s.C, s.C, ws + w.W2lo, ws + w.W2t, ws + w.W2tlo};
    }
    for (int l = l0; l < s.L && l < l0 + 3; ++l) {
      const rd_encoder_layer_params& E = P->layer[l];
      items[n++] = {E.in_proj_weight, 3 * s.D, s.D, ws + w.wsp[l].in_lo, ws + w.wsp[l].in_t, ws + w.wsp[l].in_tlo};
      items[n++] = {E.out_proj_weight, s.D, s.D, ws + w.wsp[l].out_lo, ws + w.wsp[l].out_t, ws + w.wsp[l].out_tlo};
      items[n++] = {E.linear1_weight, s.nhid, s.D, ws + w.wsp[l].l1_lo, ws + w.wsp[l].l1_t, ws + w.wsp[l].l1_tlo};
      items[n++] = {E.linear2_weight, s.D, s.nhid, ws + w.wsp[l].l2_lo, ws + w.wsp[l].l2_t, ws + w.wsp[l].l2_tlo};
    }
    RD_TRY(split_weights(items, n, st, l0 == 0 ? &pro : nullptr));
  }
  float* Z0 = ws + w.Z[0];
  if (!encoder_only) {
  // lift of the raw observations and the positional encoding (written into Z0[..., 4N:]) in one launch
  RD_TRY(lift_posenc(src, P->R_u, s.B, s.T, s.N, s.dob, s.p, rng, tc && !exact, X0, times, s.M2, dims->pe_timescales, RD_D_PE, Z0,
                     s.D, s.Dm, st, rep));
  {
    ObpropTcArgs a;
    a.x = X0; a.W = W1; a.bias = P->ob1_value_bias; a.scale = nscale; a.scale_mod = s.N;
    a.rows = s.M1; a.C = s.C; a.out = H1; a.round_out = tc && !exact;
    a.W_lo = exact ? ws + w.W1lo : nullptr;
    RD_TRY(obprop_forward(a, st));
    a.x = H1; a.W = W2; a.bias = P->ob2_value_bias; a.out = Z0; a.round_out = 0;
    a.W_lo = exact ? ws + w.W2lo : nullptr;
    a.perm = 1; a.pB = s.B; a.pN = s.N; a.pdob = s.dob; a.pD = s.D;
    RD_TRY(obprop_forward(a, st));
  }
  }

  const float scale = 1.f / sqrtf((float)s.hd);
  const int64_t row3 = (int64_t)s.B * 3 * s.D;
  const int64_t TT = (int64_t)s.T * s.T;
  for (int l = 0; l < s.L; ++l) {
    const rd_encoder_layer_params& E = P->layer[l];
    float* x = ws + w.Z[l];
    float* qkv = ws + w.l[l].qkv;
    float* Pm = ws + w.l[l].P;
    float* Pd = s.p > 0.f ? ws + w.l[l].Pd : nullptr;
    {
      GemmP g = nt(x, s.D, E.in_proj_weight, s.D, qkv, 3 * s.D, s.M2, 3 * s.D, s.D);
      g.bias = E.in_proj_bias;
      RD_TRY(linear_nt(g, ws + w.wsp[l].in_lo, st));
    }
    float* ctx = ws + w.l[l].ctx;
    if (attn_tc_supported(s.T, s.hd)) {
      RD_TRY(attn_tc_fwd(qkv, lengths, s.B, s.H, s.T, s.hd, s.p, rng, SITE_ATTN + l, ctx, st, rep));
    } else if (attn_small_supported(s.T, s.hd)) {
      RD_TRY(attn_small_fwd(qkv, lengths, s.B, s.H, s.T, s.hd, s.p, rng, SITE_ATTN + l, ctx, st, rep));
    } else {
      {  // S[b,h] = scale * Q K^T
        GemmP g;
        g.A = qkv; g.ta = 0; g.sAi = row3; g.sAk = 1; g.sAzo = 3 * s.D; g.sAzi = s.hd;
        g.B = qkv + s.D; g.tb = 1; g.sBj = row3; g.sBk = 1; g.sBzo = 3 * s.D; g.sBzi = s.hd;
        g.C = Pm; g.sCi = s.T; g.sCj = 1; g.sCzo = s.H * TT; g.sCzi = TT;
        g.M = s.T; g.N = s.T; g.K = s.hd; g.nz = s.B * s.H; g.nz_inner = s.H; g.alpha = scale;
        RD_TRY(gemm(g, st));
      }
      RD_TRY(attn_softmax_fwd(Pm, lengths, s.B, s.H, s.T, s.p, rng, SITE_ATTN + l, Pd, st, rep));
      {  // ctx[b,h] = P V
        GemmP g;
        g.A = Pd ? Pd : Pm; g.ta = 0; g.sAi = s.T; g.sAk = 1; g.sAzo = s.H * TT; g.sAzi = TT;
        g.B = qkv + 2 * s.D; g.tb = 0; g.sBk = row3; g.sBj = 1; g.sBzo = 3 * s.D; g.sBzi = s.hd;
        g.C = ctx; g.sCi = (int64_t)s.B * s.D; g.sCj = 1; g.sCzo = s.D; g.sCzi = s.hd;
        g.M = s.T; g.N = s.hd; g.K = s.T; g.nz = s.B * s.H; g.nz_inner = s.H;
        RD_TRY(gemm(g, st));
      }
    }
    float* r1 = ws + w.l[l].r1; float* x1 = ws + w.l[l].x1;
    {
      GemmP g = nt(ctx, s.D, E.out_proj_weight, s.D, r1, s.D, s.M2, s.D, s.D);
      g.bias = E.out_proj_bias; g.drop_p = s.p; g.rng = rng; g.drop_site = SITE_RESID1 + l; g.rep = rep;
      g.resid = x; g.resid_ld = s.D;
      if (s.p > 0.f) { g.drop_mask = reinterpret_cast<uint32_t*>(ws + w.l[l].m1); g.drop_mask_ld = (s.D + 31) / 32; }
      RD_TRY(linear_nt(g, ws + w.wsp[l].out_lo, st));
    }
    RD_TRY(layernorm_fwd(r1, E.norm1_weight, E.norm1_bias, s.M2, s.D, dims->ln_eps, x1, ws + w.l[l].st1, st));
    float* f = ws + w.l[l].f; float* r2 = ws + w.l[l].r2;
    {
      GemmP g = nt(x1, s.D, E.linear1_weight, s.D, f, s.nhid, s.M2, s.nhid, s.D);
      g.bias = E.linear1_bias; g.relu = 1; g.drop_p = s.p; g.rng = rng; g.drop_site = SITE_FFN + l; g.rep = rep;
      RD_TRY(linear_nt(g, ws + w.wsp[l].l1_lo, st));
    }
    {
      GemmP g = nt(f, s.nhid, E.linear2_weight, s.nhid, r2, s.D, s.M2, s.D, s.nhid);
      g.bias = E.linear2_bias; g.drop_p = s.p; g.rng = rng; g.drop_site = SITE_RESID2 + l; g.rep = rep;
      g.resid = x1; g.resid_ld = s.D;
      if (s.p > 0.f) { g.drop_mask = reinterpret_cast<uint32_t*>(ws + w.l[l].m2); g.drop_mask_ld = (s.D + 31) / 32; }
      RD_TRY(linear_nt(g, ws + w.wsp[l].l2_lo, st));
    }
    RD_TRY(layernorm_fwd(r2, E.norm2_weight, E.norm2_bias, s.M2, s.D, dims->ln_eps, ws + w.Z[l + 1], ws + w.l[l].st2, st));
  }
  float* feat = ws + w.feat; float* hpre = ws + w.hpre;
  RD_TRY(head_fwd(s.B, s.T, s.D, s.emb, s.ds, s.ncls, ws + w.Z[s.L], lengths, statics, P->emb_weight, P->emb_bias,
                  P->mlp0_weight, P->mlp0_bias, P->mlp2_weight, P->mlp2_bias, feat, hpre, logits, y, ws + w.loss_ps, d_logits,
                  loss, reinterpret_cast<unsigned*>(ws + w.cnt), st));
  return 0;
}

static int raindrop_bwd(const rd_dims* dims, const rd_params* P, const float* statics, const int64_t* lengths,
                        const float* nscale, const float* ws, const float* dlogits, float* sc, int phases,
                        float* d_z0_out, cudaStream_t st, GradConsumer& c) {
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if ((phases & ~3) || phases == 0) { set_error("rd_raindrop_v2_bwd: phases must be 1, 2 or 3"); return -2; }
  WsLayout w = ws_layout(s);
  BwLayout b = bw_layout(s);
  const Trained t = trained(s, c.grads);
  c.s = &s; c.t = &t; c.b = &b; c.sc = sc;
  const rd_grads& G = c.mode == GRAD_WEIGHTS ? *c.grads : kNoGrads;   // the head's outer products: weights mode only
  const uint64_t* rng = reinterpret_cast<const uint64_t*>(ws + w.rng);
  const float ik = s.p > 0.f ? 1.f / (1.f - s.p) : 1.f;
  float* gA = sc + b.gA; float* gB = sc + b.gB; float* gD = sc + b.gD; float* dP = sc + b.dP;

  if (phases & RD_BWD_ENCODER) {
  // ---- head: logits = mlp2(relu(mlp0(feat))), pooled = masked mean          code/models_rd.py:366-385
  const float* feat = ws + w.feat; const float* hpre = ws + w.hpre;
  float* dfeat = sc + b.dfeat; float* dhpre = sc + b.dhpre;
  RD_TRY(head_bwd(s.B, s.T, s.D, s.emb, s.ds, s.ncls, lengths, statics, P->mlp0_weight, P->mlp2_weight, feat, hpre, dlogits,
                  dhpre, dfeat, gA, G.mlp0_weight, G.mlp0_bias, G.mlp2_weight, G.mlp2_bias, G.emb_weight, G.emb_bias, st));
  RD_TRY(c.head(dlogits, hpre, dhpre, feat, dfeat, statics, st));

  const float scale = 1.f / sqrtf((float)s.hd);
  const int64_t row3 = (int64_t)s.B * 3 * s.D;
  const int64_t TT = (int64_t)s.T * s.T;
  for (int l = s.L - 1; l >= 0; --l) {
    const rd_encoder_layer_params& E = P->layer[l];
    const float* x = ws + w.Z[l];
    const float* qkv = ws + w.l[l].qkv; const float* Pm = ws + w.l[l].P;
    const float* Pd = s.p > 0.f ? ws + w.l[l].Pd : Pm;
    const float* ctx = ws + w.l[l].ctx; const float* r1 = ws + w.l[l].r1; const float* x1 = ws + w.l[l].x1;
    const float* f = ws + w.l[l].f; const float* r2 = ws + w.l[l].r2;
    float* K2 = sc + b.l[l].K2; float* gF = sc + b.l[l].gF; float* K1 = sc + b.l[l].K1; float* dqkv = sc + b.l[l].dqkv;
    // norm2 + feed-forward block.  K2 = gradient w.r.t. the (dropped) linear2 output: operand of its weight
    // gradient, kept until the grouped launch; res = the undropped residual-path gradient
    float* res = s.p > 0.f ? gB : K2;
    int chunks = 0;
    // did the forward GEMMs of this layer store their dropout keep bits (tensor-core epilogue)?  Same predicate, same operands.
    const uint32_t* m2 = nullptr; const uint32_t* m1 = nullptr;
    const int mld = (s.D + 31) / 32;
    if (s.p > 0.f) {
      GemmP g2 = nt(f, s.nhid, E.linear2_weight, s.nhid, const_cast<float*>(r2), s.D, s.M2, s.D, s.nhid);
      g2.bias = E.linear2_bias; g2.drop_p = s.p; g2.rng = rng; g2.resid = x1; g2.resid_ld = s.D;
      if (linear_nt_is_tc(g2, ws + w.wsp[l].l2_lo)) m2 = reinterpret_cast<const uint32_t*>(ws + w.l[l].m2);
      GemmP g1 = nt(ctx, s.D, E.out_proj_weight, s.D, const_cast<float*>(r1), s.D, s.M2, s.D, s.D);
      g1.bias = E.out_proj_bias; g1.drop_p = s.p; g1.rng = rng; g1.resid = x; g1.resid_ld = s.D;
      if (linear_nt_is_tc(g1, ws + w.wsp[l].out_lo)) m1 = reinterpret_cast<const uint32_t*>(ws + w.l[l].m1);
    }
    RD_TRY(layernorm_bwd(r2, ws + w.l[l].st2, E.norm2_weight, gA, s.M2, s.D, res, sc + b.l[l].ln[0], K2, s.p, rng,
                         SITE_RESID2 + l, &chunks, st, m2, mld));
    RD_TRY(c.ln(t.norm2[l], sc + b.l[l].ln[0], chunks, r2, ws + w.l[l].st2, gA, st));
    RD_TRY(c.linear(t.layer(l, LINEAR2), K2, f, st));
    {   // gF = (K2 . W2) * [f > 0] / (1-p)   ("NT" against W2^T so that the tensor-core kernel applies)
      GemmP g = nt(K2, s.D, ws + w.wsp[l].l2_t, s.D, gF, s.nhid, s.M2, s.nhid, s.D);
      g.gate = f; g.gate_ld = s.nhid; g.gate_scale = ik;  // relu' and the FFN dropout mask in one
      RD_TRY(linear_nt(g, ws + w.wsp[l].l2_tlo, st));
    }
    RD_TRY(c.linear(t.layer(l, LINEAR1), gF, x1, st));
    {
      GemmP g = nt(gF, s.nhid, ws + w.wsp[l].l1_t, s.nhid, gA, s.D, s.M2, s.D, s.nhid);
      g.resid = res; g.resid_ld = s.D;
      RD_TRY(linear_nt(g, ws + w.wsp[l].l1_tlo, st));
    }
    // norm1 + self-attention block
    res = s.p > 0.f ? gB : K1;
    RD_TRY(layernorm_bwd(r1, ws + w.l[l].st1, E.norm1_weight, gA, s.M2, s.D, res, sc + b.l[l].ln[1], K1, s.p, rng,
                         SITE_RESID1 + l, &chunks, st, m1, mld));
    RD_TRY(c.ln(t.norm1[l], sc + b.l[l].ln[1], chunks, r1, ws + w.l[l].st1, gA, st));
    RD_TRY(c.linear(t.layer(l, OUT_PROJ), K1, ctx, st));
    RD_TRY(linear_nt(nt(K1, s.D, ws + w.wsp[l].out_t, s.D, gD, s.D, s.M2, s.D, s.D), ws + w.wsp[l].out_tlo, st));
    if (attn_tc_supported(s.T, s.hd)) {
      RD_TRY(attn_tc_bwd(qkv, gD, lengths, s.B, s.H, s.T, s.hd, s.p, rng, SITE_ATTN + l, dqkv, st));
    } else if (attn_small_supported(s.T, s.hd)) {
      RD_TRY(attn_small_bwd(qkv, gD, lengths, s.B, s.H, s.T, s.hd, s.p, rng, SITE_ATTN + l, dqkv, st));
    } else {
      {  // dPd[b,h] = dctx V^T
        GemmP g;
        g.A = gD; g.ta = 0; g.sAi = (int64_t)s.B * s.D; g.sAk = 1; g.sAzo = s.D; g.sAzi = s.hd;
        g.B = qkv + 2 * s.D; g.tb = 1; g.sBj = row3; g.sBk = 1; g.sBzo = 3 * s.D; g.sBzi = s.hd;
        g.C = dP; g.sCi = s.T; g.sCj = 1; g.sCzo = s.H * TT; g.sCzi = TT;
        g.M = s.T; g.N = s.T; g.K = s.hd; g.nz = s.B * s.H; g.nz_inner = s.H;
        RD_TRY(gemm(g, st));
      }
      {  // dV[b,h] = Pd^T dctx
        GemmP g;
        g.A = Pd; g.ta = 1; g.sAk = s.T; g.sAi = 1; g.sAzo = s.H * TT; g.sAzi = TT;
        g.B = gD; g.tb = 0; g.sBk = (int64_t)s.B * s.D; g.sBj = 1; g.sBzo = s.D; g.sBzi = s.hd;
        g.C = dqkv + 2 * s.D; g.sCi = row3; g.sCj = 1; g.sCzo = 3 * s.D; g.sCzi = s.hd;
        g.M = s.T; g.N = s.hd; g.K = s.T; g.nz = s.B * s.H; g.nz_inner = s.H;
        RD_TRY(gemm(g, st));
      }
      RD_TRY(attn_softmax_bwd(Pm, dP, s.B, s.H, s.T, s.p, rng, SITE_ATTN + l, st));
      {  // dQ[b,h] = scale * dS K
        GemmP g;
        g.A = dP; g.ta = 0; g.sAi = s.T; g.sAk = 1; g.sAzo = s.H * TT; g.sAzi = TT;
        g.B = qkv + s.D; g.tb = 0; g.sBk = row3; g.sBj = 1; g.sBzo = 3 * s.D; g.sBzi = s.hd;
        g.C = dqkv; g.sCi = row3; g.sCj = 1; g.sCzo = 3 * s.D; g.sCzi = s.hd;
        g.M = s.T; g.N = s.hd; g.K = s.T; g.nz = s.B * s.H; g.nz_inner = s.H; g.alpha = scale;
        RD_TRY(gemm(g, st));
      }
      {  // dK[b,h] = scale * dS^T Q
        GemmP g;
        g.A = dP; g.ta = 1; g.sAk = s.T; g.sAi = 1; g.sAzo = s.H * TT; g.sAzi = TT;
        g.B = qkv; g.tb = 0; g.sBk = row3; g.sBj = 1; g.sBzo = 3 * s.D; g.sBzi = s.hd;
        g.C = dqkv + s.D; g.sCi = row3; g.sCj = 1; g.sCzo = 3 * s.D; g.sCzi = s.hd;
        g.M = s.T; g.N = s.hd; g.K = s.T; g.nz = s.B * s.H; g.nz_inner = s.H; g.alpha = scale;
        RD_TRY(gemm(g, st));
      }
    }
    RD_TRY(c.linear(t.layer(l, IN_PROJ), dqkv, x, st));
    {
      // the first layer's input gradient is d(loss)/d(encoder input): optionally delivered straight to the caller
      GemmP g = nt(dqkv, 3 * s.D, ws + w.wsp[l].in_t, 3 * s.D, (l == 0 && d_z0_out) ? d_z0_out : gA, s.D, s.M2, s.D, 3 * s.D);
      g.resid = res; g.resid_ld = s.D;
      RD_TRY(linear_nt(g, ws + w.wsp[l].in_tlo, st));
    }
  }
  RD_TRY(c.flush(phases & RD_BWD_OBPROP, st));   // without the ob-prop phase the caller may reduce the gradients now
  }

  if (phases & RD_BWD_OBPROP) {
  // ---- observation propagation: gA = d(loss)/d(Z0) [T,B,D]          code/models_rd.py:322-343
  float* gO2 = sc + b.gO2; float* gO1 = sc + b.gO1;
  const float* X0 = ws + w.X0; const float* H1 = ws + w.H1;
  const int tc = s.tc;
  RD_TRY(obprop_out_grad(gA, ws + w.Z[0], nscale, s.B, s.T, s.N, s.dob, s.D, tc && !s.exact, gO2, st));
  RD_TRY(c.linear(t.obprop(2), gO2, H1, st));
  if (tc) {
    // dZ1 = (dZ2 . W2) * s * [H1 > 0] on the tensor cores: "NT" form against a transposed, TF32-rounded W2
    const float* W2t = ws + w.W2t;      // written by the forward's weight-prep launch
    ObpropTcArgs a;
    a.x = gO2; a.W = W2t; a.bias = nullptr; a.relu = 0; a.scale = nscale; a.scale_mod = s.N; a.gate = H1;
    a.W_lo = s.exact ? ws + w.W2tlo : nullptr;
    a.rows = s.M1; a.C = s.C; a.out = gO1;
    RD_TRY(obprop_tc_fwd(a, st));
  } else {
    GemmP g = nn(gO2, s.C, P->ob2_value_weight, s.C, gO1, s.C, s.M1, s.C, s.C);
    g.rowscale = nscale; g.rowscale_mod = s.N; g.gate = H1; g.gate_ld = s.C;
    RD_TRY(gemm(g, st));
  }
  RD_TRY(c.linear(t.obprop(1), gO1, X0, st));
  RD_TRY(c.flush(false, st));
  }
  return 0;
}

// W1^T with its error-compensation remainder, which input_grad_dx0 reads on the tensor cores (nothing on the CUDA cores)
static int prepare_w1t(const Shape& s, const rd_params* P, float* W1t, float* W1tlo, cudaStream_t st) {
  if (!s.tc) return 0;
  const WeightSplit it = {P->ob1_value_weight, s.C, s.C, nullptr, W1t, W1tlo};
  return split_weights(&it, 1, st);
}

// The input gradient of a chunk of a chunked driver (rows dc, shape s) after its forward: the backward from the chunk's
// d_logits into its backward scratch, then dX0.
static int chunk_input_grad(const rd_dims* dc, const Shape& s, const rd_params* P, const Expanded& x,
                            const float* node_scale, float* S, const ChunkLayout& l, cudaStream_t st) {
  GradConsumer none;
  RD_TRY(raindrop_bwd(dc, P, x.statics, x.lengths, node_scale, S + l.ws, S + l.dlogits, S + l.sc, RD_BWD_ALL, nullptr, st, none));
  return input_grad_dx0(s, P, S + l.sc + bw_layout(s).gO1, S + l.W1t, S + l.W1tlo, S + l.dX0, st);
}

}  // namespace rd

// =================================================================================================
// C ABI
// =================================================================================================
using namespace rd;

extern "C" {

int rd_abi_version(void) { return RD_ABI_VERSION; }
const char* rd_last_error_string(void) { return last_error(); }
uint64_t rd_launch_count(void) { return launch_count(); }

int rd_node_scale(const int64_t* edge_tgt, const float* edge_w, int32_t E, int32_t N, float* out, void* stream) {
  if ((E > 0 && (!edge_tgt || !edge_w)) || !out || E < 0 || N < 1) { set_error("rd_node_scale: bad arguments"); return -2; }
  return node_scale(edge_tgt, edge_w, E, N, out, (cudaStream_t)stream);
}

size_t rd_obprop_fwd_scratch_bytes(int64_t rows, int32_t C) {
  return (size_t)(round_up(rows * C, 64) + round_up((int64_t)C * C, 64)) * sizeof(float);
}

int rd_obprop_fwd(const float* x, const float* weight, const float* bias, const float* nscale, int32_t mod,
                  int64_t rows, int32_t C, float* out, void* scratch, void* stream) {
  if (!x || !weight || !bias || !nscale || !out || rows < 0 || C < 1 || mod < 1) {
    set_error("rd_obprop_fwd: bad arguments");
    return -2;
  }
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  ObpropTcArgs a;
  a.x = x; a.W = weight; a.bias = bias; a.scale = nscale; a.scale_mod = mod; a.rows = rows; a.C = C; a.out = out;
  if (obprop_tc_supported(C) && scratch) {   // arbitrary caller data
    float* xr = (float*)scratch;
    float* wr = xr + round_up(rows * C, 64);
    if (obprop_tc_exact(rows, C, 0)) {        // latency-bound size: error-compensated kernel, operands as they are
      WeightSplit it = {weight, C, C, wr, nullptr, nullptr};
      RD_TRY(split_weights(&it, 1, st));
      a.W_lo = wr;
    } else {                                  // streaming size: round both operands to TF32 first, single pass
      RD_TRY(round_tf32(x, rows * C, xr, st));
      RD_TRY(round_tf32(weight, (int64_t)C * C, wr, st));
      a.x = xr; a.W = wr;
    }
  }
  return obprop_forward(a, st);
}

size_t rd_obprop_bwd_scratch_bytes(int64_t rows, int32_t C) {
  int64_t tcp = tc_wgrad_partial_floats(C, C, rows), skp = splitk_partial_floats(C, C, rows);
  int64_t a = round_up(rows * C, 64) + round_up(tcp > skp ? tcp : skp, 64);
  return (size_t)a * sizeof(float);
}

int rd_obprop_bwd(const float* x, const float* out, const float* d_out, const float* weight, const float* nscale,
                  int32_t mod, int64_t rows, int32_t C, float* d_x, float* d_weight, float* d_bias, void* scratch,
                  void* stream) {
  if (!x || !out || !d_out || !weight || !nscale || !d_weight || !d_bias || !scratch || rows < 1 || C < 1) {
    set_error("rd_obprop_bwd: bad arguments");
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* dpre = (float*)scratch;
  float* partial = dpre + round_up(rows * C, 64);
  RD_TRY(relu_scale_bwd(d_out, out, nscale, mod, rows, C, dpre, st));
  RD_TRY(tn(nullptr, dpre, C, x, C, d_weight, d_bias, C, C, rows, partial, partial, st));
  if (d_x) RD_TRY(gemm(nn(dpre, C, weight, C, d_x, C, rows, C, C), st));
  return 0;
}

size_t rd_linear_scratch_bytes(int32_t in_features, int32_t out_features) {
  return (size_t)round_up((int64_t)in_features * out_features, 64) * sizeof(float);
}

int rd_linear_fwd(const float* x, const float* weight, const float* bias, int64_t rows, int32_t in_features,
                  int32_t out_features, int32_t relu, float* out, void* scratch, void* stream) {
  if (!x || !weight || !out || !scratch || rows < 0 || in_features < 1 || out_features < 1) {
    set_error("rd_linear_fwd: bad arguments");
    return -2;
  }
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  WeightSplit it = {weight, out_features, in_features, (float*)scratch, nullptr, nullptr};
  RD_TRY(split_weights(&it, 1, st));
  GemmP g = nt(x, in_features, weight, in_features, out, out_features, rows, out_features, in_features);
  g.bias = bias; g.relu = relu;
  return linear_nt(g, (const float*)scratch, st);
}

int rd_debug_attention_timing(uint64_t* buffer) { attn_tc_set_debug((unsigned long long*)buffer); return 0; }
int rd_debug_gemm_timing(uint64_t* buffer) { tc_gemm_set_debug((unsigned long long*)buffer); return 0; }
int rd_debug_wgrad_timing(uint64_t* buffer) { tc_wgrad_set_debug((unsigned long long*)buffer); return 0; }

int rd_temporal_attention_fwd(const float* qkv, const int64_t* lengths, int32_t B, int32_t H, int32_t T, int32_t hd,
                              float drop_p, const uint64_t* rng_captured, uint32_t site, int32_t impl, float* ctx,
                              void* stream) {
  if (!qkv || !lengths || !ctx || B < 1 || H < 1 || T < 1 || hd < 1 || drop_p < 0.f || drop_p >= 1.f || (drop_p > 0.f && !rng_captured)) {
    set_error("rd_temporal_attention_fwd: bad arguments");
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if ((impl == 0 || impl == 1) && attn_tc_supported(T, hd)) return attn_tc_fwd(qkv, lengths, B, H, T, hd, drop_p, rng_captured, site, ctx, st);
  if ((impl == 0 || impl == 2) && attn_small_supported(T, hd)) return attn_small_fwd(qkv, lengths, B, H, T, hd, drop_p, rng_captured, site, ctx, st);
  set_error("rd_temporal_attention_fwd: T=%d hd=%d not supported by implementation %d", T, hd, impl);
  return -2;
}

int rd_temporal_attention_bwd(const float* qkv, const float* d_ctx, const int64_t* lengths, int32_t B, int32_t H,
                              int32_t T, int32_t hd, float drop_p, const uint64_t* rng_captured, uint32_t site,
                              int32_t impl, float* d_qkv, void* stream) {
  if (!qkv || !d_ctx || !lengths || !d_qkv || B < 1 || H < 1 || T < 1 || hd < 1 || drop_p < 0.f || drop_p >= 1.f ||
      (drop_p > 0.f && !rng_captured)) {
    set_error("rd_temporal_attention_bwd: bad arguments");
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if ((impl == 0 || impl == 1) && attn_tc_supported(T, hd)) return attn_tc_bwd(qkv, d_ctx, lengths, B, H, T, hd, drop_p, rng_captured, site, d_qkv, st);
  if ((impl == 0 || impl == 2) && attn_small_supported(T, hd)) return attn_small_bwd(qkv, d_ctx, lengths, B, H, T, hd, drop_p, rng_captured, site, d_qkv, st);
  set_error("rd_temporal_attention_bwd: T=%d hd=%d not supported by implementation %d", T, hd, impl);
  return -2;
}

size_t rd_linear_wgrad_partial_bytes(int64_t rows, int32_t out_features, int32_t in_features) {
  if (rows < 1 || out_features < 1 || in_features < 1) return 0;
  int64_t a = tc_wgrad_partial_floats(out_features, in_features, rows), b = splitk_partial_floats(out_features, in_features, rows);
  return (size_t)round_up(a > b ? a : b, 64) * sizeof(float);
}

int rd_linear_wgrad_group(const rd_wgrad_item* items, int32_t n, void* stream) {
  if (!items || n < 0) { set_error("rd_linear_wgrad_group: bad arguments"); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  WgradQueue wq;
  for (int i = 0; i < n; ++i) {
    const rd_wgrad_item& it = items[i];
    if (!it.d_out || !it.x || !it.d_weight || !it.d_bias || !it.partial || it.rows < 1 || it.out_features < 1 || it.in_features < 1) {
      set_error("rd_linear_wgrad_group: problem %d has a NULL pointer or an empty shape", i);
      return -2;
    }
    RD_TRY(tn(&wq, it.d_out, it.out_features, it.x, it.in_features, it.d_weight, it.d_bias, it.out_features, it.in_features,
              it.rows, (float*)it.partial, (float*)it.partial, st));
  }
  return wq.flush(st);
}

size_t rd_workspace_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)ws_layout(s).total * sizeof(float);
}

size_t rd_backward_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)bw_layout(s).total * sizeof(float);
}

int64_t rd_workspace_offset(const rd_dims* dims, int32_t which, int64_t* n_floats) {
  Shape s;
  if (make_shape(dims, &s) != 0) return -1;
  WsLayout w = ws_layout(s);
  int64_t off = -1, n = 0;
  switch (which) {
    case RD_WS_X0: off = w.X0; n = s.M1 * s.C; break;
    case RD_WS_H1: off = w.H1; n = s.M1 * s.C; break;
    case RD_WS_ENC_IN: off = w.Z[0]; n = s.M2 * s.D; break;
    case RD_WS_ENC_OUT: off = w.Z[s.L]; n = s.M2 * s.D; break;
    case RD_WS_FEAT: off = w.feat; n = (int64_t)s.B * s.Df; break;
    case RD_WS_RNG: off = w.rng; n = 4; break;
    case RD_WS_HEAD_HIDDEN: off = w.hpre; n = (int64_t)s.B * s.Df; break;
    default:
      if (which >= RD_WS_FFN && which < RD_WS_FFN + s.L) { off = w.l[which - RD_WS_FFN].f; n = s.M2 * s.nhid; break; }
      set_error("rd_workspace_offset: unknown buffer %d", which); return -1;
  }
  if (n_floats) *n_floats = n;
  return off * (int64_t)sizeof(float);
}

int rd_raindrop_v2_fwd(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                       const float* times, const int64_t* lengths, const float* node_scale, uint64_t* rng_state,
                       void* workspace, float* logits, const int64_t* y, float* loss, float* d_logits, void* stream) {
  if (!dims || !params || !src || !times || !lengths || !node_scale || !workspace || !logits) {
    set_error("rd_raindrop_v2_fwd: NULL argument");
    return -2;
  }
  return raindrop_fwd(dims, params, src, statics, times, lengths, node_scale, rng_state, (float*)workspace, logits,
                      y, loss, d_logits, 0, (cudaStream_t)stream);
}

int rd_raindrop_v2_bwd(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                       const float* node_scale, const void* workspace, const float* d_logits, const rd_grads* grads,
                       void* scratch, int32_t phases, void* stream) {
  if (!dims || !params || !lengths || !node_scale || !workspace || !d_logits || !scratch) {
    set_error("rd_raindrop_v2_bwd: NULL argument");
    return -2;
  }
  GradConsumer c{grads ? GRAD_WEIGHTS : GRAD_NONE, grads};
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, (float*)scratch,
                      phases, nullptr, (cudaStream_t)stream, c);
}

size_t rd_input_grad_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)input_grad_layout(s).total * sizeof(float);
}

int rd_raindrop_v2_input_grad(const rd_dims* dims, const rd_params* params, const float* src, const float* times,
                              const int64_t* lengths, const void* workspace, const void* bwd_scratch, void* scratch,
                              float* d_src, float* d_times, float* d_statics, void* stream) {
  if (!dims || !params || !workspace || !bwd_scratch) { set_error("rd_raindrop_v2_input_grad: NULL argument"); return -2; }
  if (d_src && (!src || !scratch || !params->R_u || !params->ob1_value_weight)) {
    set_error("rd_raindrop_v2_input_grad: d_src needs src, scratch, R_u and ob1_value_weight");
    return -2;
  }
  if (d_times && !times) { set_error("rd_raindrop_v2_input_grad: d_times needs times"); return -2; }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if ((d_src || d_times) && (s.dpe != RD_D_PE || s.emb != s.N)) {
    set_error("rd_raindrop_v2_input_grad: d_src / d_times need the Raindrop_v2 workspace (d_pe = 16, emb_dim = d_inp)");
    return -2;
  }
  if (d_statics && (s.ds == 0 || !params->emb_weight)) { set_error("rd_raindrop_v2_input_grad: no static branch"); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  const WsLayout w = ws_layout(s);
  const BwLayout b = bw_layout(s);
  const float* ws = (const float*)workspace;
  const float* sc = (const float*)bwd_scratch;
  float* dX0 = nullptr;
  if (d_src) {
    const IgLayout il = input_grad_layout(s);
    float* W1t = (float*)scratch + il.W1t; float* W1tlo = (float*)scratch + il.W1tlo;
    dX0 = (float*)scratch + il.dX0;
    RD_TRY(prepare_w1t(s, params, W1t, W1tlo, st));
    RD_TRY(input_grad_dx0(s, params, sc + b.gO1, W1t, W1tlo, dX0, st));
  }
  return input_grad(src, params->R_u, dX0, s.B, s.T, s.N, s.dob, s.p, reinterpret_cast<const uint64_t*>(ws + w.rng), d_src,
                    times, sc + b.gA, s.M2, s.D, s.Dm, dims->pe_timescales, s.dpe, lengths, d_times, sc + b.dfeat, s.Df, s.D,
                    params->emb_weight, s.emb, s.ds, d_statics, st);
}

size_t rd_integrated_gradients_scratch_bytes(const rd_dims* dims, int32_t steps_per_chunk) {
  IgScratch l;
  if (!dims || ig_scratch(dims, steps_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

int rd_raindrop_v2_integrated_gradients(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                        const float* times, const int64_t* lengths, const float* node_scale,
                                        const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                        const float* alphas, const float* weights, int32_t n_steps, int32_t steps_per_chunk,
                                        void* scratch, float* attr_src, float* attr_statics, float* endpoint_logits,
                                        void* stream) {
  const char* fn = "rd_raindrop_v2_integrated_gradients";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !baseline_src || !alphas || !weights || !scratch || !attr_src || !endpoint_logits || !params->R_u ||
      !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (s0.ds > 0 && !baseline_statics) { set_error("%s: d_static > 0 needs baseline_statics", fn); return -2; }
  if (n_steps < 1 || steps_per_chunk < 1) { set_error("%s: n_steps and steps_per_chunk must be >= 1", fn); return -2; }
  IgScratch l;
  RD_TRY(ig_scratch(dims, steps_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, mc = steps_per_chunk;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  float* attr_st = s0.ds > 0 ? attr_statics : nullptr;

  // 1. the endpoints: one forward on 2B rows (baseline rows, then input rows) -> endpoint_logits [2, B, ncls]
  const rd_dims de = chunk_dims(dims, 2 * B, (int64_t)B * mc, 0);
  RD_TRY(ig_expand(src, baseline_src, statics, baseline_statics, times, lengths, nullptr, 2, B, s0.T, s0.N, s0.ds, s0.ncls,
                   nullptr, nullptr, x.src, x.statics, x.times, x.lengths, nullptr, st));
  RD_TRY(raindrop_fwd(&de, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, endpoint_logits,
                      nullptr, nullptr, nullptr, 0, st));
  // 2. W1^T with its remainder, once per call
  RD_TRY(prepare_w1t(s0, params, S + l.W1t, S + l.W1tlo, st));
  // 3. chunks of mc steps (the last one possibly shorter, same scratch, same arithmetic mode)
  for (int c0 = 0; c0 < n_steps; c0 += mc) {
    const int m = n_steps - c0 < mc ? n_steps - c0 : mc;
    const rd_dims dc = chunk_dims(dims, B * m, (int64_t)B * mc, 0);
    Shape s;
    RD_TRY(make_shape(&dc, &s));
    RD_TRY(ig_expand(src, baseline_src, statics, baseline_statics, times, lengths, alphas + c0, m, B, s.T, s.N, s.ds, s.ncls,
                     target, endpoint_logits + (int64_t)B * s.ncls, x.src, x.statics, x.times, x.lengths, S + l.dlogits, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, S + l.logits,
                        nullptr, nullptr, nullptr, 0, st));
    RD_TRY(chunk_input_grad(&dc, s, params, x, node_scale, S, l, st));
    RD_TRY(ig_accumulate(src, baseline_src, alphas + c0, weights + c0, m, B, s.T, s.N, s.dob, params->R_u, S + l.dX0,
                         S + l.acc_src, attr_src, statics, baseline_statics, S + l.sc + bw_layout(s).dfeat, s.Df, s.D,
                         params->emb_weight, s.emb, s.ds, S + l.acc_static, attr_st, c0 == 0, c0 + m >= n_steps, st));
  }
  return 0;
}

size_t rd_pgd_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk) {
  PgdScratch l;
  if (!dims || pgd_scratch(dims, samples_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

int rd_raindrop_v2_pgd(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                       const float* times, const int64_t* lengths, const float* node_scale, const int64_t* y,
                       const uint8_t* sensor_perturbable, const uint8_t* sample_attacked, int32_t perturb_static,
                       int32_t norm, float eps, float alpha, int32_t n_steps, int32_t random_start, const uint64_t* rng,
                       int32_t samples_per_chunk, void* scratch, float* src_adv, float* statics_adv, float* logits_adv,
                       float* logits_clean, float* loss_adv, void* stream) {
  const char* fn = "rd_raindrop_v2_pgd";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !scratch || !src_adv || !logits_adv || !logits_clean || !loss_adv || !params->R_u ||
      !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (norm != RD_PGD_LINF && norm != RD_PGD_L2) { set_error("%s: norm must be RD_PGD_LINF or RD_PGD_L2, got %d", fn, norm); return -2; }
  if (!(eps >= 0.f) || !(alpha >= 0.f) || isinf(eps) || isinf(alpha) || n_steps < 0) {
    set_error("%s: eps and alpha must be finite and >= 0, n_steps >= 0 (eps = %g, alpha = %g, n_steps = %d)", fn, eps,
              alpha, n_steps);
    return -2;
  }
  if (random_start && !rng) { set_error("%s: random_start needs rng", fn); return -2; }
  if (perturb_static && s0.ds == 0) { set_error("%s: perturb_static needs a static branch (d_static > 0)", fn); return -2; }
  const int B = s0.B, spc = samples_per_chunk;
  PgdScratch l;
  RD_TRY(pgd_scratch(dims, spc, &l));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = (float*)scratch;
  float* lg = S + l.logits;
  double* best = reinterpret_cast<double*>(S + l.best);
  const Expanded x = l.inputs(S, s0.ds);
  PgdArgs a;
  a.src = src; a.statics = s0.ds > 0 ? statics : nullptr; a.times = times; a.lengths = lengths;
  a.sens = sensor_perturbable; a.attacked = sample_attacked;
  a.x_e = x.src; a.st_e = x.statics; a.times_e = x.times; a.len_e = x.lengths; a.delta = S + l.delta; a.grad = S + l.grad;
  a.B = B; a.T = s0.T; a.N = s0.N; a.ds = s0.ds; a.pst = perturb_static ? 1 : 0;
  // W1^T with its remainder, once per call
  if (n_steps > 0) RD_TRY(prepare_w1t(s0, params, S + l.W1t, S + l.W1tlo, st));
  for (int c0 = 0; c0 < B; c0 += spc) {
    const int m = B - c0 < spc ? B - c0 : spc;
    const rd_dims dc = chunk_dims(dims, m, spc, 0);
    Shape s;
    RD_TRY(make_shape(&dc, &s));
    const float* dfeat = S + l.sc + bw_layout(s).dfeat;
    a.m = m; a.c0 = c0;
    float* clean = logits_clean + (int64_t)c0 * s.ncls;
    RD_TRY(pgd_expand(a, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, clean, nullptr,
                        nullptr, nullptr, 0, st));
    const float* cur = clean;
    if (random_start) {
      RD_TRY(pgd_start(a, norm, eps, rng, st));
      RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, lg, nullptr,
                          nullptr, nullptr, 0, st));
      cur = lg;
    }
    for (int k = 0;; ++k) {
      RD_TRY(pgd_track(a, s.ncls, cur, logits_clean, y, best, k == 0, S + l.dlogits, src_adv, statics_adv, logits_adv,
                       loss_adv, st));
      if (k == n_steps) break;
      RD_TRY(chunk_input_grad(&dc, s, params, x, node_scale, S, l, st));
      RD_TRY(pgd_step(a, norm, eps, alpha, params->R_u, s.dob, S + l.dX0, dfeat, s.Df, s.D, params->emb_weight, s.emb,
                      st));
      RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, lg, nullptr,
                          nullptr, nullptr, 0, st));
      cur = lg;
    }
  }
  return 0;
}

size_t rd_counterfactual_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk, int32_t n_restarts) {
  CfScratch l;
  if (!dims || cf_scratch(dims, samples_per_chunk, n_restarts, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

int rd_raindrop_v2_counterfactual(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                  const float* times, const int64_t* lengths, const float* node_scale,
                                  const int64_t* target, const uint8_t* sensor_mutable, const float* weights,
                                  const float* lower, const float* upper, const rd_cf_options* opt, const uint64_t* rng,
                                  int32_t samples_per_chunk, void* scratch, float* src_cf, float* statics_cf,
                                  float* logits_cf, float* logits_clean, int64_t* target_out, uint8_t* valid,
                                  double* distance, double* c_final, uint8_t* round_valid, void* stream) {
  const char* fn = "rd_raindrop_v2_counterfactual";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !opt || !scratch || !src_cf || !logits_cf || !logits_clean || !target_out || !valid || !distance ||
      !c_final || !round_valid || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  const rd_cf_options o = *opt;
  if (o.n_search < 1 || o.n_steps < 0 || o.n_restarts < 1) {
    set_error("%s: n_search and n_restarts must be >= 1, n_steps >= 0 (%d, %d, %d)", fn, o.n_search, o.n_restarts,
              o.n_steps);
    return -2;
  }
  if (!(o.kappa >= 0.0) || isinf(o.kappa) || !(o.c_init > 0.0) || isinf(o.c_init) || !(o.beta >= 0.f) || isinf(o.beta) ||
      !(o.step_size > 0.f) || isinf(o.step_size) || !(o.init_scale >= 0.f) || isinf(o.init_scale)) {
    set_error("%s: kappa, beta and init_scale must be finite and >= 0, c_init and step_size finite and > 0 (kappa = %g, "
              "c_init = %g, beta = %g, step_size = %g, init_scale = %g)", fn, o.kappa, o.c_init, o.beta, o.step_size,
              o.init_scale);
    return -2;
  }
  if (s0.ncls < 2) { set_error("%s: a counterfactual needs n_classes >= 2", fn); return -2; }
  if (o.n_restarts > 1 && !rng) { set_error("%s: n_restarts > 1 needs rng", fn); return -2; }
  if (o.perturb_static && s0.ds == 0) { set_error("%s: perturb_static needs a static branch (d_static > 0)", fn); return -2; }
  const int B = s0.B, spc = samples_per_chunk, R = o.n_restarts;
  CfScratch l;
  RD_TRY(cf_scratch(dims, spc, R, &l));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = (float*)scratch;
  float* lg = S + l.logits;
  const Expanded x = l.inputs(S, s0.ds);
  CfArgs a;
  a.src = src; a.statics = s0.ds > 0 ? statics : nullptr; a.times = times; a.lengths = lengths;
  a.sens = sensor_mutable; a.w = weights; a.lo = lower; a.hi = upper;
  a.x_e = x.src; a.st_e = x.statics; a.times_e = x.times; a.len_e = x.lengths; a.xd = S + l.xd; a.yd = S + l.yd;
  a.row = reinterpret_cast<double*>(S + l.row); a.best = reinterpret_cast<double*>(S + l.best);
  a.B = B; a.T = s0.T; a.N = s0.N; a.ds = s0.ds; a.R = R; a.pst = o.perturb_static ? 1 : 0;
  CfOut k;
  k.logits = lg; k.logits_clean = logits_clean; k.logits_cf = logits_cf; k.src_cf = src_cf;
  k.st_cf = s0.ds > 0 ? statics_cf : nullptr; k.target_out = target_out; k.valid = valid; k.distance = distance;
  k.ncls = s0.ncls;
  // W1^T with its remainder, once per call
  if (o.n_steps > 0) RD_TRY(prepare_w1t(s0, params, S + l.W1t, S + l.W1tlo, st));
  for (int c0 = 0; c0 < B; c0 += spc) {
    const int m = B - c0 < spc ? B - c0 : spc;
    const rd_dims dc = chunk_dims(dims, m * R, (int64_t)spc * R, 0);
    Shape s;
    RD_TRY(make_shape(&dc, &s));
    const float* dfeat = S + l.sc + bw_layout(s).dfeat;
    a.m = m; a.c0 = c0;
    RD_TRY(cf_expand(a, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, lg, nullptr,
                        nullptr, nullptr, 0, st));
    RD_TRY(cf_init(a, k, target, o.c_init, st));
    for (int round = 0; round < o.n_search; ++round) {
      RD_TRY(cf_start(a, o.init_scale, o.beta, rng, st));
      for (int step = 0;; ++step) {
        RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, lg, nullptr,
                            nullptr, nullptr, 0, st));
        RD_TRY(cf_track(a, k, o.kappa, S + l.dlogits, st));
        if (step == o.n_steps) break;
        RD_TRY(chunk_input_grad(&dc, s, params, x, node_scale, S, l, st));
        RD_TRY(cf_step(a, step, o.step_size, o.beta, params->R_u, s.dob, S + l.dX0, dfeat, s.Df, s.D, params->emb_weight,
                       s.emb, st));
      }
      RD_TRY(cf_round(a, round, o.n_search, round_valid, c_final, st));
    }
  }
  return 0;
}

size_t rd_coalition_attribution_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t coalitions_per_chunk) {
  CoalScratch l;
  if (!dims || coalition_scratch(dims, n_players, coalitions_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// What every coalition entry point (Shapley sampling and ablation, KernelSHAP) shares: the argument checks, the scratch
// carved by coalition_scratch and the endpoint forward.  `fn` names the caller in error messages.
struct CoalRun {
  Shape s0;
  int P, G, B, cc;
  Expanded x;
  float* ws; float* logits; double* acc; uint8_t* keep;
};
static int coalition_setup(const char* fn, const rd_dims* dims, const rd_params* params, const float* src,
                           const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                           const float* baseline_src, const float* baseline_statics, const int32_t* cell_player,
                           int64_t stride_t, int64_t stride_b, int32_t n_players, int32_t coalitions_per_chunk, void* scratch,
                           const float* attr, const float* endpoint_logits, CoalRun* r) {
  Shape& s0 = r->s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !baseline_src || !cell_player || !scratch || !attr || !endpoint_logits || !params->R_u ||
      !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (s0.ds > 0 && !baseline_statics) { set_error("%s: d_static > 0 needs baseline_statics", fn); return -2; }
  const int P = n_players, G = P - (s0.ds > 0 ? 1 : 0);
  if (G < 1) { set_error("%s: n_players = %d gives %d players of the value cells, need >= 1", fn, P, G); return -2; }
  if (stride_t < 0 || stride_b < 0) {
    set_error("%s: player strides must be >= 0, got (%lld, %lld)", fn, (long long)stride_t, (long long)stride_b);
    return -2;
  }
  CoalScratch l;
  RD_TRY(coalition_scratch(dims, P, coalitions_per_chunk, &l));
  r->P = P; r->G = G; r->B = s0.B; r->cc = coalitions_per_chunk;
  float* S = (float*)scratch;
  r->x = l.inputs(S, s0.ds);
  r->ws = S + l.ws; r->logits = S + l.logits;
  r->acc = reinterpret_cast<double*>(S + l.acc);
  r->keep = reinterpret_cast<uint8_t*>(S + l.keep);
  return 0;
}

// The endpoints: one forward on 2B rows (x' rows: every player removed, cells of no player keep x; then x rows)
// -> endpoint_logits [2, B, ncls], in the arithmetic mode pinned from B*cc rows.
static int coalition_endpoints(const CoalRun& r, const rd_dims* dims, const rd_params* params, const float* src,
                               const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                               const float* baseline_src, const float* baseline_statics, const int32_t* cell_player,
                               int64_t stride_t, int64_t stride_b, float* endpoint_logits, cudaStream_t st) {
  const rd_dims de = chunk_dims(dims, 2 * r.B, (int64_t)r.B * r.cc, 0);
  RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, stride_t, stride_b,
                          nullptr, r.P, r.G, COALITION_ENDPOINTS, 0, 2, r.B, r.s0.T, r.s0.N, r.s0.ds, nullptr, r.x.src,
                          r.x.statics, r.x.times, r.x.lengths, st));
  return raindrop_fwd(&de, params, r.x.src, r.x.statics, r.x.times, r.x.lengths, node_scale, nullptr, r.ws, endpoint_logits,
                      nullptr, nullptr, nullptr, 0, st);
}

// The one implementation behind both Shapley-sampling / ablation entry points.
static int coalition_attribution(const char* fn, const rd_dims* dims, const rd_params* params, const float* src,
                                 const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                                 const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                 const int32_t* cell_player, int64_t stride_t, int64_t stride_b, int32_t n_players,
                                 const int32_t* orders, int32_t m, int32_t method, int32_t coalitions_per_chunk, void* scratch,
                                 float* attr, float* endpoint_logits, void* stream) {
  if (method != RD_ATTR_SHAPLEY && method != RD_ATTR_ABLATION) {
    set_error("%s: method must be RD_ATTR_SHAPLEY or RD_ATTR_ABLATION, got %d", fn, method);
    return -2;
  }
  CoalRun r;
  RD_TRY(coalition_setup(fn, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                         cell_player, stride_t, stride_b, n_players, coalitions_per_chunk, scratch, attr, endpoint_logits, &r));
  const int P = r.P, G = r.G, B = r.B, cc = r.cc;
  if (method == RD_ATTR_SHAPLEY && (!orders || m < 1 || (int64_t)m * (P - 1) > (1LL << 30))) {
    set_error("%s: Shapley sampling needs orders and 1 <= m, m*(P-1) <= 2^30 (m = %d)", fn, m);
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int n_coal = method == RD_ATTR_SHAPLEY ? m * (P - 1) : P;

  // 1. the endpoints
  RD_TRY(coalition_endpoints(r, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                             cell_player, stride_t, stride_b, endpoint_logits, st));
  // 2. chunks of cc coalitions (the last one possibly shorter, same scratch, same arithmetic mode); with no coalition
  //    (Shapley over one player) a single accumulation turns the endpoints into the result
  int c0 = 0;
  do {
    const int nc = n_coal - c0 < cc ? n_coal - c0 : cc;
    if (nc > 0) {
      const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
      RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, stride_t, stride_b,
                              orders, P, G, method, c0, nc, B, r.s0.T, r.s0.N, r.s0.ds, r.keep, r.x.src, r.x.statics,
                              r.x.times, r.x.lengths, st));
      RD_TRY(raindrop_fwd(&dc, params, r.x.src, r.x.statics, r.x.times, r.x.lengths, node_scale, nullptr, r.ws, r.logits,
                          nullptr, nullptr, nullptr, 0, st));
    }
    RD_TRY(coalition_accumulate(r.logits, endpoint_logits, target, orders, P, method, m, c0, nc, B, r.s0.ncls, r.acc, attr,
                                c0 == 0, c0 + nc >= n_coal, st));
    c0 += cc;
  } while (c0 < n_coal);
  return 0;
}

int rd_raindrop_v2_coalition_attribution(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                         const float* times, const int64_t* lengths, const float* node_scale,
                                         const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                         const int32_t* sensor_player, int32_t n_players, const int32_t* orders, int32_t m,
                                         int32_t method, int32_t coalitions_per_chunk, void* scratch, float* attr,
                                         float* endpoint_logits, void* stream) {
  const char* fn = "rd_raindrop_v2_coalition_attribution";
  if (!dims || !sensor_player) { set_error("%s: NULL argument", fn); return -2; }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  const int P = n_players, G = P - (s0.ds > 0 ? 1 : 0);
  if (G < 1 || G > s0.N) { set_error("%s: n_players = %d gives %d sensor groups for N = %d", fn, P, G, s0.N); return -2; }
  return coalition_attribution(fn, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                               target, sensor_player, 0, 0, n_players, orders, m, method, coalitions_per_chunk, scratch, attr,
                               endpoint_logits, stream);
}

int rd_raindrop_v2_cell_coalition_attribution(const rd_dims* dims, const rd_params* params, const float* src,
                                              const float* statics, const float* times, const int64_t* lengths,
                                              const float* node_scale, const float* baseline_src,
                                              const float* baseline_statics, const int64_t* target,
                                              const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                              int32_t n_players, const int32_t* orders, int32_t m, int32_t method,
                                              int32_t coalitions_per_chunk, void* scratch, float* attr,
                                              float* endpoint_logits, void* stream) {
  return coalition_attribution("rd_raindrop_v2_cell_coalition_attribution", dims, params, src, statics, times, lengths,
                               node_scale, baseline_src, baseline_statics, target, cell_player, player_stride_t,
                               player_stride_b, n_players, orders, m, method, coalitions_per_chunk, scratch, attr,
                               endpoint_logits, stream);
}

// KernelSHAP: the checks, scratch and endpoint forward of coalition_attribution (coalition_setup, coalition_endpoints;
// the layout's keep table is not used), then the chunked coalition forwards with the caller's coalition table as the
// keep table, the regression right-hand side accumulated in the fp64 running sums (acc) and one solve launch at the end.
int rd_raindrop_v2_kernel_shap(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                               const float* times, const int64_t* lengths, const float* node_scale, const float* baseline_src,
                               const float* baseline_statics, const int64_t* target, const int32_t* cell_player,
                               int64_t player_stride_t, int64_t player_stride_b, int32_t n_players, const uint8_t* coalitions,
                               const double* weights, int32_t n_coalitions, const double* solve, int32_t coalitions_per_chunk,
                               void* scratch, float* attr, float* endpoint_logits, void* stream) {
  const char* fn = "rd_raindrop_v2_kernel_shap";
  if (!solve) { set_error("%s: NULL argument", fn); return -2; }
  if (n_coalitions < 0 || (n_coalitions > 0 && (!coalitions || !weights))) {
    set_error("%s: n_coalitions = %d must be >= 0, and > 0 needs coalitions and weights", fn, n_coalitions);
    return -2;
  }
  if (n_players > RD_KERNEL_SHAP_MAX_PLAYERS) {
    set_error("%s: n_players = %d, at most %d", fn, n_players, RD_KERNEL_SHAP_MAX_PLAYERS);
    return -2;
  }
  CoalRun r;
  RD_TRY(coalition_setup(fn, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                         cell_player, player_stride_t, player_stride_b, n_players, coalitions_per_chunk, scratch, attr,
                         endpoint_logits, &r));
  cudaStream_t st = (cudaStream_t)stream;
  const int P = r.P, G = r.G, B = r.B, cc = r.cc;
  const int64_t M = n_coalitions;

  // 1. the endpoints
  RD_TRY(coalition_endpoints(r, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                             cell_player, player_stride_t, player_stride_b, endpoint_logits, st));
  // 2. chunks of cc coalitions (the last one possibly shorter, same scratch, same arithmetic mode); with no coalition a
  //    single accumulation zeroes the sums and the solve returns k (F(x) - F(x')).  c0 runs in 64 bits: M may be up to
  //    INT32_MAX, and c0 + cc past it must not wrap (inside the loop c0 < M fits an int).
  int64_t c0 = 0;
  do {
    const int nc = (int)(M - c0 < cc ? M - c0 : cc);
    if (nc > 0) {
      const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
      RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, player_stride_t,
                              player_stride_b, nullptr, P, G, COALITION_TABLE, (int)c0, nc, B, r.s0.T, r.s0.N, r.s0.ds,
                              const_cast<uint8_t*>(coalitions + c0 * P), r.x.src, r.x.statics, r.x.times, r.x.lengths,
                              st));
      RD_TRY(raindrop_fwd(&dc, params, r.x.src, r.x.statics, r.x.times, r.x.lengths, node_scale, nullptr, r.ws, r.logits,
                          nullptr, nullptr, nullptr, 0, st));
    }
    RD_TRY(kernel_shap_accumulate(r.logits, endpoint_logits, target, coalitions, weights, P, (int)c0, nc, B, r.s0.ncls, r.acc,
                                  c0 == 0, st));
    c0 += cc;
  } while (c0 < M);
  // 3. attr = acc . K^T + (F(x) - F(x')) k^T
  return kernel_shap_solve(r.acc, solve, endpoint_logits, target, P, B, r.s0.ncls, attr, st);
}

// ---- faithfulness of attributions by removal -------------------------------------------------------------------------
// Chunks of cc (curve, count) pairs or replicates (B*cc rows; curves also run the 2B-row endpoint forward) and the
// chunk's per-row keep table [cc*B, P] (uint8) at the arena's tail.
struct RemovalScratch : ChunkLayout { int64_t keep; };
static int removal_scratch(const rd_dims* dims, int n_players, int cc, bool curves, RemovalScratch* l) {
  RD_TRY(chunk_layout(dims, curves ? "pairs_per_chunk" : "replicates_per_chunk", cc, dims->B, curves, 0, false, l));
  if (n_players < 1 || n_players > RD_REMOVAL_MAX_PLAYERS) {
    set_error("n_players = %d must be in [1, %d]", n_players, RD_REMOVAL_MAX_PLAYERS);
    return -2;
  }
  l->keep = l->a.take(ceil_div((int64_t)cc * dims->B * n_players, 4));
  return 0;
}

size_t rd_removal_curves_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t pairs_per_chunk) {
  RemovalScratch l;
  if (!dims || removal_scratch(dims, n_players, pairs_per_chunk, true, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

size_t rd_removal_infidelity_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t replicates_per_chunk) {
  RemovalScratch l;
  if (!dims || removal_scratch(dims, n_players, replicates_per_chunk, false, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// The player checks both removal calls and the debug entry share, after the shape's.
static int removal_players(const char* fn, const Shape& s0, const int32_t* cell_player, int64_t stride_t, int64_t stride_b,
                           int32_t n_players, int* G) {
  if (!cell_player) { set_error("%s: NULL argument", fn); return -2; }
  *G = n_players - (s0.ds > 0 ? 1 : 0);
  if (n_players > RD_REMOVAL_MAX_PLAYERS || *G < 1) {
    set_error("%s: n_players = %d must be in [1 + (d_static > 0), %d]", fn, n_players, RD_REMOVAL_MAX_PLAYERS);
    return -2;
  }
  if (stride_t < 0 || stride_b < 0) {
    set_error("%s: player strides must be >= 0, got (%lld, %lld)", fn, (long long)stride_t, (long long)stride_b);
    return -2;
  }
  return 0;
}

// floor(p_remove 2^32): a word below it removes its player (p_remove = 1: every word)
static int removal_threshold(const char* fn, double p_remove, uint64_t* below) {
  if (!(p_remove > 0.0 && p_remove <= 1.0)) { set_error("%s: p_remove = %g must lie in (0, 1]", fn, p_remove); return -2; }
  *below = (uint64_t)floor(p_remove * 4294967296.0);
  return 0;
}

// What both removal calls share: the checks, the scratch carved by removal_scratch, in the CoalRun the coalition calls'
// endpoint forward reads.
static int removal_setup(const char* fn, const rd_dims* dims, const rd_params* params, const float* src,
                         const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                         const float* baseline_src, const float* baseline_statics, const int32_t* cell_player,
                         int64_t stride_t, int64_t stride_b, int32_t n_players, const float* attributions, int32_t cc,
                         bool curves, void* scratch, CoalRun* r) {
  Shape& s0 = r->s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !baseline_src || !attributions || !scratch || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (s0.ds > 0 && !baseline_statics) { set_error("%s: d_static > 0 needs baseline_statics", fn); return -2; }
  RD_TRY(removal_players(fn, s0, cell_player, stride_t, stride_b, n_players, &r->G));
  RemovalScratch l;
  RD_TRY(removal_scratch(dims, n_players, cc, curves, &l));
  r->P = n_players; r->B = s0.B; r->cc = cc;
  float* S = (float*)scratch;
  r->x = l.inputs(S, s0.ds);
  r->ws = S + l.ws; r->logits = S + l.logits;
  r->acc = nullptr;
  r->keep = reinterpret_cast<uint8_t*>(S + l.keep);
  return 0;
}

// The endpoints, the rank launch, then per chunk of pairs the keep table, the expansion and one eval forward into
// curve_logits; the summaries after the last chunk.
int rd_raindrop_v2_removal_curves(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                  const float* times, const int64_t* lengths, const float* node_scale,
                                  const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                  const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                  int32_t n_players, const float* attributions, int32_t order, const int32_t* counts,
                                  int32_t n_counts, int32_t pairs_per_chunk, void* scratch, int32_t* rank,
                                  float* curve_logits, float* endpoint_logits, float* values, double* summaries,
                                  int64_t* target_out, void* stream) {
  const char* fn = "rd_raindrop_v2_removal_curves";
  if (!counts || !rank || !curve_logits || !endpoint_logits || !values || !summaries || !target_out) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (order != RD_REMOVAL_DESCENDING && order != RD_REMOVAL_ASCENDING && order != RD_REMOVAL_ABSOLUTE) {
    set_error("%s: order = %d is not an RD_REMOVAL_* order", fn, order);
    return -2;
  }
  CoalRun r;
  RD_TRY(removal_setup(fn, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                       cell_player, player_stride_t, player_stride_b, n_players, attributions, pairs_per_chunk, true,
                       scratch, &r));
  const int P = r.P, G = r.G, B = r.B, cc = r.cc, K = n_counts;
  if (K < 1 || K > P + 1) { set_error("%s: n_counts = %d must be in [1, n_players + 1 = %d]", fn, K, P + 1); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(coalition_endpoints(r, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                             cell_player, player_stride_t, player_stride_b, endpoint_logits, st));
  RD_TRY(removal_rank(attributions, B, P, order, rank, st));
  const int n_pairs = 2 * K;
  for (int q0 = 0; q0 < n_pairs; q0 += cc) {
    const int nc = n_pairs - q0 < cc ? n_pairs - q0 : cc;
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
    RD_TRY(removal_curve_keep(rank, counts, K, q0, nc, B, P, r.keep, st));
    RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, player_stride_t,
                            player_stride_b, nullptr, P, G, COALITION_ROWS, 0, nc, B, r.s0.T, r.s0.N, r.s0.ds, r.keep,
                            r.x.src, r.x.statics, r.x.times, r.x.lengths, st));
    RD_TRY(raindrop_fwd(&dc, params, r.x.src, r.x.statics, r.x.times, r.x.lengths, node_scale, nullptr, r.ws,
                        curve_logits + (int64_t)q0 * B * r.s0.ncls, nullptr, nullptr, nullptr, 0, st));
  }
  return removal_curve_summary(curve_logits, endpoint_logits, target, counts, K, B, P, r.s0.ncls, values, summaries,
                               target_out, st);
}

// One forward on the B rows of x, then per chunk of replicates the keep table, the expansion, one eval forward and the
// moment launch.
int rd_raindrop_v2_removal_infidelity(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                      const float* times, const int64_t* lengths, const float* node_scale,
                                      const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                      const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                      int32_t n_players, const float* attributions, const uint64_t* rng, double p_remove,
                                      int32_t n_samples, int32_t replicates_per_chunk, void* scratch, float* clean_logits,
                                      double* moments, int64_t* target_out, void* stream) {
  const char* fn = "rd_raindrop_v2_removal_infidelity";
  if (!rng || !clean_logits || !moments) { set_error("%s: NULL argument", fn); return -2; }
  if (n_samples < 1) { set_error("%s: n_samples = %d must be >= 1", fn, n_samples); return -2; }
  uint64_t below;
  RD_TRY(removal_threshold(fn, p_remove, &below));
  CoalRun r;
  RD_TRY(removal_setup(fn, dims, params, src, statics, times, lengths, node_scale, baseline_src, baseline_statics,
                       cell_player, player_stride_t, player_stride_b, n_players, attributions, replicates_per_chunk, false,
                       scratch, &r));
  const int P = r.P, G = r.G, B = r.B, cc = r.cc;
  cudaStream_t st = (cudaStream_t)stream;
  const rd_dims de = chunk_dims(dims, B, (int64_t)B * cc, 0);
  RD_TRY(raindrop_fwd(&de, params, src, r.s0.ds > 0 ? statics : nullptr, times, lengths, node_scale, nullptr, r.ws,
                      clean_logits, nullptr, nullptr, nullptr, 0, st));
  for (int m0 = 0; m0 < n_samples; m0 += cc) {
    const int nc = n_samples - m0 < cc ? n_samples - m0 : cc;
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
    RD_TRY(removal_sample_keep(rng, below, m0, nc, B, P, r.keep, st));
    RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, player_stride_t,
                            player_stride_b, nullptr, P, G, COALITION_ROWS, 0, nc, B, r.s0.T, r.s0.N, r.s0.ds, r.keep,
                            r.x.src, r.x.statics, r.x.times, r.x.lengths, st));
    RD_TRY(raindrop_fwd(&dc, params, r.x.src, r.x.statics, r.x.times, r.x.lengths, node_scale, nullptr, r.ws, r.logits,
                        nullptr, nullptr, nullptr, 0, st));
    RD_TRY(removal_moments(r.logits, clean_logits, target, attributions, r.keep, nc, B, P, r.s0.ncls, m0 == 0, moments,
                           target_out, st));
    if (n_samples - m0 <= cc) break;
  }
  return 0;
}

int rd_debug_removal_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                            const int64_t* lengths, const float* baseline_src, const float* baseline_statics,
                            const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                            int32_t n_players, const int32_t* rank, const int32_t* counts, int32_t n_counts,
                            const uint64_t* rng, double p_remove, int64_t q0, int32_t nc, uint8_t* keep_table,
                            float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, void* stream) {
  const char* fn = "rd_debug_removal_inputs";
  if (!dims || !src || !times || !lengths || !baseline_src || !keep_table || !src_e || !times_e || !lengths_e) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.ds > 0 && (!statics || !baseline_statics || !statics_e)) {
    set_error("%s: d_static > 0 needs statics, baseline_statics and statics_e", fn);
    return -2;
  }
  int G;
  RD_TRY(removal_players(fn, s0, cell_player, player_stride_t, player_stride_b, n_players, &G));
  if (nc < 1 || q0 < 0 || (int64_t)s0.B * nc > (1LL << 30)) {
    set_error("%s: nc = %d must be >= 1 with B * nc <= 2^30, and q0 = %lld >= 0", fn, nc, (long long)q0);
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int P = n_players, B = s0.B;
  if (rank) {
    if (!counts || n_counts < 1 || n_counts > P + 1 || q0 + nc > 2LL * n_counts) {
      set_error("%s: curve pairs need counts, 1 <= n_counts <= n_players + 1 and q0 + nc <= 2 n_counts", fn);
      return -2;
    }
    RD_TRY(removal_curve_keep(rank, counts, n_counts, q0, nc, B, P, keep_table, st));
  } else {
    if (!rng) { set_error("%s: give rank (curves) or rng (infidelity)", fn); return -2; }
    uint64_t below;
    RD_TRY(removal_threshold(fn, p_remove, &below));
    RD_TRY(removal_sample_keep(rng, below, q0, nc, B, P, keep_table, st));
  }
  return coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, player_stride_t,
                          player_stride_b, nullptr, P, G, COALITION_ROWS, 0, nc, B, s0.T, s0.N, s0.ds, keep_table, src_e,
                          s0.ds > 0 ? statics_e : nullptr, times_e, lengths_e, st);
}

size_t rd_mc_dropout_scratch_bytes(const rd_dims* dims, int32_t replicates_per_chunk) {
  McScratch l;
  if (!dims || mc_scratch(dims, replicates_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// Chunks of cc replicates: the inputs expanded when the chunk size changes (the first and a ragged last chunk), one
// training forward whose dropout draws replicate m0 + m at step rng[1] + m0 + m (the prologue captures {seed, step + m0},
// rep_remap adds m), and one launch that adds the chunk to the fp64 sums and, after the last chunk, writes the statistics.
int rd_raindrop_v2_mc_dropout(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                              const float* times, const int64_t* lengths, const float* node_scale, const uint64_t* rng,
                              int32_t n_samples, int32_t replicates_per_chunk, void* scratch, float* mean_probs,
                              float* variance, float* entropies, float* samples, void* stream) {
  const char* fn = "rd_raindrop_v2_mc_dropout";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s0));
  if (!src || !times || !rng || !scratch || !mean_probs || !variance || !entropies || !params->R_u ||
      !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (n_samples < 1 || replicates_per_chunk < 1) { set_error("%s: n_samples and replicates_per_chunk must be >= 1", fn); return -2; }
  McScratch l;
  RD_TRY(mc_scratch(dims, replicates_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, cc = replicates_per_chunk;
  const int64_t M = n_samples;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  double* acc = reinterpret_cast<double*>(S + l.acc);
  int expanded = 0;
  for (int64_t c0 = 0; c0 < M; c0 += cc) {
    const int nc = (int)(M - c0 < cc ? M - c0 : cc);
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 1);
    if (nc != expanded) {
      RD_TRY(mc_expand(src, statics, times, lengths, B, nc, s0.T, s0.N, s0.ds, x.src, x.statics, x.times, x.lengths, st));
      expanded = nc;
    }
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, const_cast<uint64_t*>(rng), S + l.ws,
                        S + l.logits, nullptr, nullptr, nullptr, 0, st, B, (uint64_t)c0));
    RD_TRY(mc_accumulate(S + l.logits, nc, B, s0.ncls, c0, M, acc, samples, mean_probs, variance, entropies, c0 == 0,
                         c0 + nc >= M, st));
  }
  return 0;
}

size_t rd_smooth_scratch_bytes(const rd_dims* dims, int32_t replicates_per_chunk) {
  ChunkLayout l;
  if (!dims || chunk_layout(dims, "replicates_per_chunk", replicates_per_chunk, dims->B, false, 0, false, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// The checks rd_raindrop_v2_smooth_counts and rd_debug_smoothing_inputs share, after the shape's.
static int smooth_check(const char* fn, const Shape& s0, int32_t perturb_static, float sigma) {
  if (!(sigma >= 0.f) || isinf(sigma)) { set_error("%s: sigma must be finite and >= 0, got %g", fn, sigma); return -2; }
  if (perturb_static && s0.ds == 0) { set_error("%s: perturb_static needs a static branch (d_static > 0)", fn); return -2; }
  return 0;
}

// Chunks of cc replicates: one launch expanding the chunk's noisy inputs, one eval forward on B*cc replicate-major rows
// and one launch adding each row's vote to counts.
int rd_raindrop_v2_smooth_counts(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const uint8_t* sensor_perturbable, int32_t perturb_static, float sigma,
                                 const uint64_t* rng, int32_t n_samples, int32_t replicates_per_chunk, void* scratch,
                                 int64_t* counts, void* stream) {
  const char* fn = "rd_raindrop_v2_smooth_counts";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !rng || !scratch || !counts || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (n_samples < 1 || replicates_per_chunk < 1) { set_error("%s: n_samples and replicates_per_chunk must be >= 1", fn); return -2; }
  RD_TRY(smooth_check(fn, s0, perturb_static, sigma));
  ChunkLayout l;
  RD_TRY(chunk_layout(dims, "replicates_per_chunk", replicates_per_chunk, dims->B, false, 0, false, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, cc = replicates_per_chunk;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  for (int c0 = 0; c0 < n_samples; c0 += cc) {
    const int nc = n_samples - c0 < cc ? n_samples - c0 : cc;
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
    RD_TRY(smooth_expand(src, statics, times, lengths, sensor_perturbable, perturb_static, sigma, rng, c0, B, nc, s0.T, s0.N,
                         s0.ds, x.src, x.statics, x.times, x.lengths, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, S + l.logits,
                        nullptr, nullptr, nullptr, 0, st));
    RD_TRY(smooth_vote(S + l.logits, B, nc, s0.ncls, c0 == 0, counts, st));
    if (n_samples - c0 <= cc) break;
  }
  return 0;
}

int rd_debug_smoothing_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                              const int64_t* lengths, const uint8_t* sensor_perturbable, int32_t perturb_static,
                              float sigma, const uint64_t* rng, int64_t m0, int32_t nc, float* src_e, float* statics_e,
                              float* times_e, int64_t* lengths_e, void* stream) {
  const char* fn = "rd_debug_smoothing_inputs";
  if (!dims || !src || !times || !lengths || !rng || !src_e) { set_error("%s: NULL argument", fn); return -2; }
  if (nc < 1 || m0 < 0) { set_error("%s: nc must be >= 1 and m0 >= 0 (nc = %d, m0 = %lld)", fn, nc, (long long)m0); return -2; }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.ds > 0 && (!statics || !statics_e)) { set_error("%s: d_static > 0 needs statics and statics_e", fn); return -2; }
  RD_TRY(smooth_check(fn, s0, perturb_static, sigma));
  if ((int64_t)s0.B * nc > (1LL << 30)) { set_error("%s: B * nc = %lld rows are too many", fn, (long long)s0.B * nc); return -2; }
  return smooth_expand(src, statics, times, lengths, sensor_perturbable, perturb_static, sigma, rng, m0, s0.B, nc, s0.T,
                       s0.N, s0.ds, src_e, statics_e, times_e, lengths_e, (cudaStream_t)stream);
}

// Randomized ablation: the smoothing layout plus the chunk's keep table [cc*B, P] (uint8).
struct AblationScratch : ChunkLayout { int64_t keep; };
static int ablation_scratch(const rd_dims* dims, int n_players, int cc, AblationScratch* l) {
  RD_TRY(chunk_layout(dims, "replicates_per_chunk", cc, dims->B, false, 0, false, l));
  if (n_players < 1 || n_players > RD_ABLATION_MAX_PLAYERS) {
    set_error("n_players = %d must be in [1, %d]", n_players, RD_ABLATION_MAX_PLAYERS);
    return -2;
  }
  l->keep = l->a.take(ceil_div((int64_t)cc * dims->B * n_players, 4));
  return 0;
}

size_t rd_ablation_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t replicates_per_chunk) {
  AblationScratch l;
  if (!dims || ablation_scratch(dims, n_players, replicates_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// The checks rd_raindrop_v2_ablation_counts and rd_debug_ablation_inputs share, after the shape's.  *J: C(P, keep) in
// exhaustive mode, 0 in sampled mode (the keep kernel's mode switch).
static int ablation_check(const char* fn, const Shape& s0, int32_t n_players, int32_t ablate_static, int32_t ablate_mask,
                          int32_t keep, int32_t exhaustive, int64_t* J) {
  const int P = n_players, st = ablate_static ? 1 : 0;
  if (ablate_static && s0.ds == 0) { set_error("%s: ablate_static needs a static branch (d_static > 0)", fn); return -2; }
  if (P < 1 || P > RD_ABLATION_MAX_PLAYERS || P - st > s0.N) {
    set_error("%s: n_players = %d must be in [1, %d] and at most d_inp%s = %d", fn, P, RD_ABLATION_MAX_PLAYERS,
              st ? " + 1" : "", s0.N + st);
    return -2;
  }
  if (keep < 1 || keep > P) { set_error("%s: keep = %d must be in [1, n_players = %d]", fn, keep, P); return -2; }
  if ((ablate_mask != 0 && ablate_mask != 1) || (exhaustive != 0 && exhaustive != 1)) {
    set_error("%s: ablate_mask and exhaustive must be 0 or 1 (got %d, %d)", fn, ablate_mask, exhaustive);
    return -2;
  }
  *J = 0;
  if (exhaustive) {
    // C(P, keep) = prod_{i < m} (P - i) / (i + 1) with m = min(keep, P - keep); every partial product is a binomial
    int64_t c = 1;
    const int m = keep < P - keep ? keep : P - keep;
    for (int i = 0; i < m && c <= 0x7fffffffLL; ++i) c = c * (P - i) / (i + 1);
    if (c > 0x7fffffffLL) {
      set_error("%s: exhaustive mode needs C(n_players, keep) <= 2^31 - 1 (n_players = %d, keep = %d)", fn, P, keep);
      return -2;
    }
    *J = c;
  }
  return 0;
}

// Chunks of cc replicates: the keep-table and expansion launches (ablate_inputs), one eval forward on B*cc
// replicate-major rows and one launch adding each row's vote to counts.
int rd_raindrop_v2_ablation_counts(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                   const float* times, const int64_t* lengths, const float* node_scale,
                                   const uint8_t* sensor_player, int32_t n_players, int32_t ablate_static,
                                   int32_t ablate_mask, int32_t keep, int32_t exhaustive, const uint64_t* rng,
                                   int32_t n_samples, int32_t replicates_per_chunk, void* scratch, int64_t* counts,
                                   void* stream) {
  const char* fn = "rd_raindrop_v2_ablation_counts";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !rng || !scratch || !counts || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (n_samples < 1 || replicates_per_chunk < 1) { set_error("%s: n_samples and replicates_per_chunk must be >= 1", fn); return -2; }
  int64_t J;
  RD_TRY(ablation_check(fn, s0, n_players, ablate_static, ablate_mask, keep, exhaustive, &J));
  AblationScratch l;
  RD_TRY(ablation_scratch(dims, n_players, replicates_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, cc = replicates_per_chunk;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  uint8_t* table = reinterpret_cast<uint8_t*>(S + l.keep);
  for (int c0 = 0; c0 < n_samples; c0 += cc) {
    const int nc = n_samples - c0 < cc ? n_samples - c0 : cc;
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
    RD_TRY(ablate_inputs(src, statics, times, lengths, sensor_player, n_players, ablate_static, ablate_mask, keep, J, rng, c0,
                         B, nc, s0.T, s0.N, s0.ds, table, x.src, x.statics, x.times, x.lengths, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, S + l.logits,
                        nullptr, nullptr, nullptr, 0, st));
    RD_TRY(smooth_vote(S + l.logits, B, nc, s0.ncls, c0 == 0, counts, st));
    if (n_samples - c0 <= cc) break;
  }
  return 0;
}

int rd_debug_ablation_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                             const int64_t* lengths, const uint8_t* sensor_player, int32_t n_players, int32_t ablate_static,
                             int32_t ablate_mask, int32_t keep, int32_t exhaustive, const uint64_t* rng, int64_t m0,
                             int32_t nc, uint8_t* keep_table, float* src_e, float* statics_e, float* times_e,
                             int64_t* lengths_e, void* stream) {
  const char* fn = "rd_debug_ablation_inputs";
  if (!dims || !src || !times || !lengths || !rng || !keep_table || !src_e) { set_error("%s: NULL argument", fn); return -2; }
  if (nc < 1 || m0 < 0) { set_error("%s: nc must be >= 1 and m0 >= 0 (nc = %d, m0 = %lld)", fn, nc, (long long)m0); return -2; }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.ds > 0 && (!statics || !statics_e)) { set_error("%s: d_static > 0 needs statics and statics_e", fn); return -2; }
  int64_t J;
  RD_TRY(ablation_check(fn, s0, n_players, ablate_static, ablate_mask, keep, exhaustive, &J));
  if ((int64_t)s0.B * nc > (1LL << 30)) { set_error("%s: B * nc = %lld rows are too many", fn, (long long)s0.B * nc); return -2; }
  return ablate_inputs(src, statics, times, lengths, sensor_player, n_players, ablate_static, ablate_mask, keep, J, rng, m0,
                       s0.B, nc, s0.T, s0.N, s0.ds, keep_table, src_e, statics_e, times_e, lengths_e, (cudaStream_t)stream);
}

// ---- early prediction -------------------------------------------------------------------------------------------------
// Chunks of kc prefixes: the smoothing layout plus the chunk's cutoff table [kc, B] (int32).
struct PrefixScratch : ChunkLayout { int64_t table; };
static int prefix_scratch(const rd_dims* dims, int kc, PrefixScratch* l) {
  RD_TRY(chunk_layout(dims, "prefixes_per_chunk", kc, dims->B, false, 0, false, l));
  l->table = l->a.take((int64_t)kc * dims->B);
  return 0;
}

size_t rd_prefix_scratch_bytes(const rd_dims* dims, int32_t prefixes_per_chunk) {
  PrefixScratch l;
  if (!dims || prefix_scratch(dims, prefixes_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// The checks of the prefixes given by horizon or by row count, after the shape's.
static int prefix_check(const char* fn, const float* horizons, const int32_t* rows, int32_t K) {
  if ((horizons != nullptr) == (rows != nullptr)) { set_error("%s: give exactly one of horizons and rows", fn); return -2; }
  if (K < 1) { set_error("%s: n_prefixes = %d must be >= 1", fn, K); return -2; }
  return 0;
}

static PrefixArgs prefix_args(const Shape& s0, const float* src, const float* statics, const float* times,
                              const int64_t* lengths, const float* horizons, const int32_t* rows) {
  PrefixArgs a{};
  a.src = src; a.statics = s0.ds > 0 ? statics : nullptr; a.times = times; a.lengths = lengths;
  a.horizons = horizons; a.rows = rows;
  a.B = s0.B; a.T = s0.T; a.N = s0.N; a.ds = s0.ds;
  return a;
}

// Chunks of kc prefixes: the cutoff and expansion launches (prefix_inputs), then ONE eval forward on B*kc prefix-major
// rows that writes its logits straight into rows k0*B .. of the output.
int rd_raindrop_v2_prefix_logits(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const float* horizons, const int32_t* rows, int32_t n_prefixes,
                                 int32_t prefixes_per_chunk, void* scratch, float* logits, int32_t* cutoffs,
                                 int64_t* prefix_lengths, void* stream) {
  const char* fn = "rd_raindrop_v2_prefix_logits";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !scratch || !logits || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  RD_TRY(prefix_check(fn, horizons, rows, n_prefixes));
  if (prefixes_per_chunk < 1) { set_error("%s: prefixes_per_chunk must be >= 1", fn); return -2; }
  PrefixScratch l;
  RD_TRY(prefix_scratch(dims, prefixes_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, kc = prefixes_per_chunk;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  PrefixArgs a = prefix_args(s0, src, statics, times, lengths, horizons, rows);
  a.table = reinterpret_cast<int32_t*>(S + l.table);
  a.cutoffs = cutoffs;
  a.lengths_out = prefix_lengths;
  a.src_e = x.src; a.statics_e = x.statics; a.times_e = x.times; a.lengths_e = x.lengths;
  for (int k0 = 0; k0 < n_prefixes; k0 += kc) {
    const int nc = n_prefixes - k0 < kc ? n_prefixes - k0 : kc;
    const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * kc, 0);
    a.k0 = k0; a.nc = nc;
    RD_TRY(prefix_inputs(a, st));
    RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws,
                        logits + (int64_t)k0 * B * s0.ncls, nullptr, nullptr, nullptr, 0, st));
    if (n_prefixes - k0 <= kc) break;
  }
  return 0;
}

int rd_debug_prefix_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                           const int64_t* lengths, const float* horizons, const int32_t* rows, int32_t n_prefixes,
                           const uint64_t* rng, double p_full, double min_fraction, int32_t* cutoffs, float* src_e,
                           float* statics_e, float* times_e, int64_t* lengths_e, void* stream) {
  const char* fn = "rd_debug_prefix_inputs";
  if (!dims || !src || !times || !lengths || !cutoffs || !src_e || !times_e || !lengths_e) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  if (rng) {
    if (horizons || n_prefixes != 1) { set_error("%s: drawn cutoffs take no horizons and n_prefixes = 1", fn); return -2; }
    if (!(p_full >= 0.0 && p_full <= 1.0) || !(min_fraction >= 0.0 && min_fraction <= 1.0)) {
      set_error("%s: p_full and min_fraction must lie in [0, 1] (got %g, %g)", fn, p_full, min_fraction);
      return -2;
    }
  } else {
    RD_TRY(prefix_check(fn, horizons, rows, n_prefixes));
  }
  if ((int64_t)s0.B * n_prefixes > (1LL << 30)) {
    set_error("%s: B * n_prefixes = %lld rows are too many", fn, (long long)s0.B * n_prefixes);
    return -2;
  }
  PrefixArgs a = prefix_args(s0, src, statics, times, lengths, horizons, rows);
  a.rng = rng;
  a.full_below = (uint64_t)floor(p_full * 4294967296.0);
  a.min_fraction = min_fraction;
  a.table = cutoffs;
  a.src_e = src_e; a.statics_e = s0.ds > 0 ? statics_e : nullptr; a.times_e = times_e; a.lengths_e = lengths_e;
  a.k0 = 0; a.nc = n_prefixes;
  return prefix_inputs(a, (cudaStream_t)stream);
}

// ---- worst-case sensor removal ----------------------------------------------------------------------------------------
// Chunks of cc candidates: the smoothing layout plus the chunk's keep table [cc*B, P] (uint8), validity [cc*B] and
// per-candidate score and success [B, cc]; per sample the reference class, the zero rank key of the exhaustive
// unranking, the beam [B, W, R] (int16) and its size, the list (ping-pong: scores [2][B, W], keep rows [2][B, W, P],
// sizes [2][B]), the best and best successful candidate of the round (scores [2][B], keep rows [2][B, P], logits
// [2][B, n_classes], flags [2][B]) and the done flags [B].
struct SensorAttackScratch : ChunkLayout {
  int64_t keep, valid, cscore, csucc, yref, key, beam, beam_n, top_score, top_keep, top_n, trk_score, trk_keep,
      trk_logits, trk_ok, done;
};
static int sensor_attack_scratch(const rd_dims* dims, int P, int W, int R, int cc, SensorAttackScratch* l) {
  if (P < 1 || P > RD_ABLATION_MAX_PLAYERS) { set_error("n_players = %d must be in [1, %d]", P, RD_ABLATION_MAX_PLAYERS); return -2; }
  if (W < 1 || W > RD_SENSOR_ATTACK_MAX_BEAM) {
    set_error("beam_width = %d must be in [1, %d]", W, RD_SENSOR_ATTACK_MAX_BEAM);
    return -2;
  }
  if (R < 1 || R > P || R > RD_SENSOR_ATTACK_MAX_REMOVED) {
    set_error("max_removed = %d must be in [1, min(n_players = %d, %d)]", R, P, RD_SENSOR_ATTACK_MAX_REMOVED);
    return -2;
  }
  RD_TRY(chunk_layout(dims, "candidates_per_chunk", cc, dims->B, false, 0, false, l));
  const int64_t B = dims->B, rows = (int64_t)cc * B;
  Arena& a = l->a;
  l->keep = a.take(ceil_div(rows * P, 4));
  l->valid = a.take(ceil_div(rows, 4));
  l->cscore = a.take(rows);
  l->csucc = a.take(ceil_div(rows, 4));
  l->yref = a.take(B);
  l->key = a.take(4);
  l->beam = a.take(ceil_div(B * W * R, 2));
  l->beam_n = a.take(B);
  l->top_score = a.take(2 * B * W);
  l->top_keep = a.take(ceil_div(2 * B * W * P, 4));
  l->top_n = a.take(2 * B);
  l->trk_score = a.take(2 * B);
  l->trk_keep = a.take(ceil_div(2 * B * P, 4));
  l->trk_logits = a.take(2 * B * dims->n_classes);
  l->trk_ok = a.take(2 * B);
  l->done = a.take(B);
  return 0;
}

size_t rd_sensor_attack_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t beam_width, int32_t max_removed,
                                      int32_t candidates_per_chunk) {
  SensorAttackScratch l;
  if (!dims || sensor_attack_scratch(dims, n_players, beam_width, max_removed, candidates_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// C(n, k) saturated at cap + 1
static int64_t binom_capped(int n, int k, int64_t cap) {
  if (k < 0 || k > n) return 0;
  if (k > n - k) k = n - k;
  int64_t c = 1;
  for (int i = 0; i < k; ++i) {
    c = c * (n - i) / (i + 1);       // a binomial at every step
    if (c > cap) return cap + 1;
  }
  return c;
}

// Round 0 evaluates the empty set.  Round r = 1 .. R evaluates W_r * P slots (w, p) of the beam, W_r = min(W, C(P, r-1))
// (beam mode), or the C(P, r) sets of r players (exhaustive).  Per chunk of cc candidates: the keep table (sa_keep, or
// ablate_inputs' unranking of the kept (P - r)-subsets in exhaustive mode and in round 0), the expansion
// (ablate_expand), ONE eval forward on B*cc rows and the selection (sa_select).
int rd_raindrop_v2_sensor_attack(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const uint8_t* sensor_player, int32_t n_players, int32_t remove_static,
                                 int32_t remove_mask, const int64_t* y, const int64_t* target, int32_t beam_width,
                                 int32_t max_removed, int32_t exhaustive, int32_t candidates_per_chunk, void* scratch,
                                 uint8_t* removed, int64_t* n_removed, float* logits, float* clean_logits, float* score,
                                 float* best_score, void* stream) {
  const char* fn = "rd_raindrop_v2_sensor_attack";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !scratch || !removed || !n_removed || !logits || !clean_logits || !score || !best_score ||
      !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (y && target) { set_error("%s: give y or target, not both", fn); return -2; }
  int64_t J;
  RD_TRY(ablation_check(fn, s0, n_players, remove_static, remove_mask, 1, exhaustive, &J));
  const int P = n_players, W = beam_width, R = max_removed, cc = candidates_per_chunk;
  SensorAttackScratch l;
  RD_TRY(sensor_attack_scratch(dims, P, W, R, cc, &l));
  const int64_t cap = 0x7fffffffLL;
  if (exhaustive) {
    int64_t total = 0;
    for (int r = 0; r <= R && total <= cap; ++r) total += binom_capped(P, r, cap);
    if (total > cap) {
      set_error("%s: exhaustive mode needs sum_{r <= max_removed} C(n_players, r) <= 2^31 - 1 (n_players = %d, "
                "max_removed = %d)", fn, P, R);
      return -2;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B;
  float* S = (float*)scratch;
  const Expanded x = l.inputs(S, s0.ds);
  uint8_t* keep = reinterpret_cast<uint8_t*>(S + l.keep);
  uint64_t* key = reinterpret_cast<uint64_t*>(S + l.key);
  if (cudaMemsetAsync(key, 0, 2 * sizeof(uint64_t), st) != cudaSuccess) {
    set_error("%s: cudaMemsetAsync failed", fn);
    return -1;
  }
  SaKeepArgs ka{};
  ka.beam = reinterpret_cast<int16_t*>(S + l.beam); ka.beam_n = reinterpret_cast<int32_t*>(S + l.beam_n);
  ka.keep = keep; ka.valid = reinterpret_cast<uint8_t*>(S + l.valid);
  ka.B = B; ka.P = P; ka.W = W; ka.R = R;
  SaSelectArgs sa{};
  sa.logits = S + l.logits; sa.keep = keep;
  sa.cls = target ? target : y;
  sa.cscore = S + l.cscore; sa.csucc = reinterpret_cast<uint8_t*>(S + l.csucc);
  sa.yref = reinterpret_cast<int32_t*>(S + l.yref); sa.done = reinterpret_cast<int32_t*>(S + l.done);
  sa.top_score = S + l.top_score; sa.top_keep = reinterpret_cast<uint8_t*>(S + l.top_keep);
  sa.top_n = reinterpret_cast<int32_t*>(S + l.top_n);
  sa.trk_score = S + l.trk_score; sa.trk_keep = reinterpret_cast<uint8_t*>(S + l.trk_keep);
  sa.trk_logits = S + l.trk_logits; sa.trk_ok = reinterpret_cast<int32_t*>(S + l.trk_ok);
  sa.beam = reinterpret_cast<int16_t*>(S + l.beam); sa.beam_n = reinterpret_cast<int32_t*>(S + l.beam_n);
  sa.removed = removed; sa.n_removed = n_removed; sa.logits_out = logits; sa.clean_logits = clean_logits;
  sa.score = score; sa.best_score = best_score;
  sa.B = B; sa.C = s0.ncls; sa.P = P; sa.W = W; sa.R = R; sa.cc = cc; sa.targeted = target ? 1 : 0;
  int cur = 0;
  for (int r = 0; r <= R; ++r) {
    const bool unrank = exhaustive || r == 0;
    const int64_t wr = r > 0 ? binom_capped(P, r - 1, W) : 1;
    const int64_t n_r = unrank ? binom_capped(P, r, cap) : (wr < W ? wr : W) * P;
    sa.r = r;
    sa.wsel = exhaustive || r == R ? 0 : (r == 0 ? 1 : W);
    sa.valid = unrank ? nullptr : ka.valid;
    for (int64_t c0 = 0; c0 < n_r; c0 += cc) {
      const int nc = (int)(n_r - c0 < cc ? n_r - c0 : cc);
      const rd_dims dc = chunk_dims(dims, B * nc, (int64_t)B * cc, 0);
      if (unrank) {
        RD_TRY(ablate_inputs(src, statics, times, lengths, sensor_player, P, remove_static, remove_mask, P - r,
                             binom_capped(P, r, cap), key, c0, B, nc, s0.T, s0.N, s0.ds, keep, x.src, x.statics, x.times,
                             x.lengths, st));
      } else {
        ka.r = r; ka.s0 = c0; ka.nc = nc;
        RD_TRY(sa_keep(ka, st));
        RD_TRY(ablate_expand(src, statics, times, lengths, sensor_player, P, remove_static, remove_mask, B, nc, s0.T,
                             s0.N, s0.ds, keep, x.src, x.statics, x.times, x.lengths, st));
      }
      RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, S + l.logits,
                          nullptr, nullptr, nullptr, 0, st));
      sa.nc = nc; sa.cur = cur; sa.first = c0 == 0; sa.last = c0 + nc >= n_r;
      RD_TRY(sa_select(sa, st));
      cur ^= 1;
    }
  }
  return 0;
}

// ---- out-of-distribution scores ---------------------------------------------------------------------------------------
// Bank columns per similarity GEMM: as many as keep a chunk's [spc, slice] similarities within 64 MiB, a multiple of 4,
// at most the whole (padded) bank.  Slicing does not change a similarity: every one is a full-K dot of the same rows.
static int64_t ood_slice(int64_t n_bank, int spc) {
  const int64_t cap = ((1LL << 24) / spc) / 4 * 4, all = round_up(n_bank, 4);
  return cap < 4 ? 4 : (cap < all ? cap : all);
}

// Candidates the kNN selection keeps per query row: k plus RD_OOD_SEL_EXTRA, at most the bank.
static int ood_selected(int k, int64_t n_bank) {
  return (int)(k + RD_OOD_SEL_EXTRA < n_bank ? k + RD_OOD_SEL_EXTRA : n_bank);
}

// A chunk of spc samples (ChunkLayout), then the centred or normalised query rows q [spc, Fp], Z [spc, rp], the
// remainder of W^T [rp, Fp], the similarities of one bank slice [spc, slice] and the running candidates [spc, ks] (uint64).
struct OodScratch : ChunkLayout { int64_t q, Z, Wlo, sim, run; };
static int ood_scratch(const rd_dims* dims, int r, int64_t n_bank, int k, int spc, OodScratch* l) {
  RD_TRY(chunk_layout(dims, "samples_per_chunk", spc, 1, false, 0, false, l));
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (r < 0 || r > s.Df || n_bank < 0 || n_bank > 0x7fffffffLL) {
    set_error("rank r = %d must be in [0, %d] and n_bank = %lld in [0, 2^31)", r, s.Df, (long long)n_bank);
    return -2;
  }
  if (n_bank > 0 && (k < 1 || k > RD_OOD_MAX_K || k > n_bank)) {
    set_error("k = %d must be in [1, min(%d, n_bank = %lld)]", k, RD_OOD_MAX_K, (long long)n_bank);
    return -2;
  }
  const int64_t Fp = round_up(s.Df, 4), rp = round_up(r, 4);
  l->q = l->a.take(spc * Fp);
  l->Z = l->a.take(spc * rp);
  l->Wlo = l->a.take(rp * Fp);
  l->sim = l->a.take(n_bank > 0 ? spc * ood_slice(n_bank, spc) : 0);
  l->run = l->a.take(n_bank > 0 ? 2LL * spc * ood_selected(k, n_bank) : 0);
  return 0;
}

// Samples b0 .. b0+m-1 of the batch into the chunk's input buffers (src [T, m, 2N], times [T, m], statics, lengths).
static int ood_slice_inputs(const Shape& s0, const float* src, const float* statics, const float* times,
                            const int64_t* lengths, int b0, int m, const Expanded& x, cudaStream_t st) {
  const size_t w = (size_t)2 * s0.N * sizeof(float);
  cudaError_t e = cudaMemcpy2DAsync(x.src, m * w, src + (int64_t)b0 * 2 * s0.N, s0.B * w, m * w, s0.T,
                                    cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpy2DAsync(x.times, m * sizeof(float), times + b0, s0.B * sizeof(float), m * sizeof(float), s0.T,
                          cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && s0.ds > 0)
    e = cudaMemcpyAsync(x.statics, statics + (int64_t)b0 * s0.ds, (size_t)m * s0.ds * sizeof(float),
                        cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(x.lengths, lengths + b0, (size_t)m * sizeof(int64_t), cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) { set_error("ood: chunk copy: %s", cudaGetErrorString(e)); return -1; }
  return 0;
}

// The eval forward of samples b0 .. b0+m-1 (the inputs themselves when one chunk covers the batch); returns the chunk's
// shape and, through feat, the chosen layer's rows [m, Df] in the workspace.  The logits land at S + l.logits.
static int ood_chunk_forward(const rd_dims* dims, const rd_params* params, const Shape& s0, const float* src,
                             const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                             int layer, int spc, int b0, int m, float* S, const ChunkLayout& l, const float** feat,
                             cudaStream_t st) {
  const rd_dims dc = chunk_dims(dims, m, spc, 0);
  Shape s;
  RD_TRY(make_shape(&dc, &s));
  Expanded x{const_cast<float*>(src), const_cast<float*>(statics), const_cast<float*>(times),
             const_cast<int64_t*>(lengths)};
  if (m < s0.B) {
    x = l.inputs(S, s0.ds);
    RD_TRY(ood_slice_inputs(s0, src, statics, times, lengths, b0, m, x, st));
  }
  RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws, S + l.logits,
                      nullptr, nullptr, nullptr, 0, st));
  const WsLayout w = ws_layout(s);
  *feat = S + l.ws + (layer == RD_OOD_HIDDEN ? w.hpre : w.feat);
  return 0;
}

static int ood_model_check(const char* fn, const rd_params* params, const float* src, const float* times, int layer,
                           int spc, const void* scratch) {
  if (!src || !times || !scratch || !params->R_u || !params->ob1_value_weight) { set_error("%s: NULL argument", fn); return -2; }
  if (layer != RD_OOD_POOLED && layer != RD_OOD_HIDDEN) { set_error("%s: layer must be RD_OOD_POOLED or RD_OOD_HIDDEN", fn); return -2; }
  if (spc < 1) { set_error("%s: samples_per_chunk must be >= 1", fn); return -2; }
  return 0;
}

static int ood_copy(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) { set_error("ood: copy: %s", cudaGetErrorString(e)); return -1; }
  return 0;
}

size_t rd_ood_features_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk) {
  ChunkLayout l;
  if (!dims || chunk_layout(dims, "samples_per_chunk", samples_per_chunk, 1, false, 0, false, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

int rd_raindrop_v2_features(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                            const float* times, const int64_t* lengths, const float* node_scale, int32_t layer,
                            int32_t samples_per_chunk, void* scratch, float* feats, float* logits, void* stream) {
  const char* fn = "rd_raindrop_v2_features";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  RD_TRY(ood_model_check(fn, params, src, times, layer, samples_per_chunk, scratch));
  ChunkLayout l;
  RD_TRY(chunk_layout(dims, "samples_per_chunk", samples_per_chunk, 1, false, 0, false, &l));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = (float*)scratch;
  for (int b0 = 0; b0 < s0.B; b0 += samples_per_chunk) {
    const int m = s0.B - b0 < samples_per_chunk ? s0.B - b0 : samples_per_chunk;
    const float* f;
    RD_TRY(ood_chunk_forward(dims, params, s0, src, statics, times, lengths, node_scale, layer, samples_per_chunk, b0, m, S,
                             l, &f, st));
    if (feats) RD_TRY(ood_copy(feats + (int64_t)b0 * s0.Df, f, (size_t)m * s0.Df * sizeof(float), st));
    if (logits) RD_TRY(ood_copy(logits + (int64_t)b0 * s0.ncls, S + l.logits, (size_t)m * s0.ncls * sizeof(float), st));
  }
  return 0;
}

int rd_feature_moments(const float* feats, const int64_t* labels, int64_t n, int32_t F, int32_t n_classes,
                       int32_t accumulate, double* class_sums, int64_t* class_counts, double* gram, void* stream) {
  const char* fn = "rd_feature_moments";
  if (!feats || (class_sums && (!labels || !class_counts))) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 0 || F < 1 || n_classes < 1) { set_error("%s: n = %lld must be >= 0, F = %d and n_classes = %d >= 1", fn, (long long)n, F, n_classes); return -2; }
  if (n == 0 && accumulate) return 0;
  return ood_moments(feats, labels, n, F, n_classes, accumulate, class_sums, class_counts, gram, (cudaStream_t)stream);
}

int rd_ood_prepare_bank(const float* feats, int64_t n, int32_t F, int32_t ld, float* bank, float* bank_lo, void* stream) {
  const char* fn = "rd_ood_prepare_bank";
  if (!feats || !bank || !bank_lo) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 1 || n > 0x7fffffffLL || F < 1 || ld < F || ld % 4) {
    set_error("%s: n = %lld must be in [1, 2^31), F >= 1 and ld >= F a multiple of 4 (F = %d, ld = %d)", fn, (long long)n, F, ld);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(bank) | reinterpret_cast<uintptr_t>(bank_lo)) & 15) {
    set_error("%s: bank and bank_lo must be 16-byte aligned", fn);
    return -2;
  }
  cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(ood_rows(feats, F, n, F, nullptr, ld, bank, st));
  return grad_lo_image(bank, n * ld, bank_lo, st);
}

size_t rd_ood_scores_scratch_bytes(const rd_dims* dims, int32_t r, int64_t n_bank, int32_t k, int32_t samples_per_chunk) {
  OodScratch l;
  if (!dims || ood_scratch(dims, r, n_bank, k, samples_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// Per chunk: one eval forward; msp / energy from its logits; Z = (f - mean) W (tc_nt, 3xTF32) and the class distances;
// the normalised rows against each bank slice (tc_nt, 3xTF32) merged into the running top-k.
int rd_raindrop_v2_ood_scores(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                              const float* times, const int64_t* lengths, const float* node_scale, int32_t layer,
                              const double* mean, const float* w_t, const float* class_proj, int32_t r, const float* bank,
                              const float* bank_lo, int64_t n_bank, int32_t k, float temperature,
                              int32_t samples_per_chunk, void* scratch, float* logits, float* msp, float* energy,
                              float* mahalanobis, int64_t* mahalanobis_class, float* mahalanobis_per_class, float* knn,
                              int64_t* knn_index, void* stream) {
  const char* fn = "rd_raindrop_v2_ood_scores";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  RD_TRY(ood_model_check(fn, params, src, times, layer, samples_per_chunk, scratch));
  const bool do_maha = mahalanobis || mahalanobis_class || mahalanobis_per_class, do_knn = knn || knn_index;
  if (do_maha && (!mean || !w_t || !class_proj || r < 1)) { set_error("%s: Mahalanobis outputs need mean, w_t, class_proj and r >= 1", fn); return -2; }
  if (do_knn && (!bank || !bank_lo || n_bank < 1)) { set_error("%s: kNN outputs need bank, bank_lo and n_bank >= 1", fn); return -2; }
  if ((msp || energy) && !(temperature > 0.f && isfinite(temperature))) {
    set_error("%s: temperature must be finite and > 0, got %g", fn, temperature);
    return -2;
  }
  OodScratch l;
  RD_TRY(ood_scratch(dims, do_maha ? r : 0, do_knn ? n_bank : 0, k, samples_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = (float*)scratch;
  const int spc = samples_per_chunk, Fp = (int)round_up(s0.Df, 4), rp = (int)round_up(r, 4);
  if (do_maha) RD_TRY(grad_lo_image(w_t, (long long)rp * Fp, S + l.Wlo, st));
  const int64_t slice = do_knn ? ood_slice(n_bank, spc) : 0;
  for (int b0 = 0; b0 < s0.B; b0 += spc) {
    const int m = s0.B - b0 < spc ? s0.B - b0 : spc;
    const float* f;
    RD_TRY(ood_chunk_forward(dims, params, s0, src, statics, times, lengths, node_scale, layer, spc, b0, m, S, l, &f, st));
    const float* lg = S + l.logits;
    if (logits) RD_TRY(ood_copy(logits + (int64_t)b0 * s0.ncls, lg, (size_t)m * s0.ncls * sizeof(float), st));
    if (msp || energy) RD_TRY(ood_logit_scores(lg, m, s0.ncls, temperature, msp ? msp + b0 : nullptr, energy ? energy + b0 : nullptr, st));
    if (do_maha) {
      RD_TRY(ood_rows(f, s0.Df, m, s0.Df, mean, Fp, S + l.q, st));
      TcNtArgs g;
      g.A = S + l.q; g.lda = Fp; g.B = w_t; g.B_lo = S + l.Wlo; g.M = m; g.N = rp; g.K = Fp; g.C = S + l.Z;
      tc_nt_plan(m, rp, true, &g.BN, &g.n_tiles);
      RD_TRY(tc_nt(g, st));
      RD_TRY(ood_class_dist(S + l.Z, class_proj, m, s0.ncls, rp,
                            mahalanobis_per_class ? mahalanobis_per_class + (int64_t)b0 * s0.ncls : nullptr,
                            mahalanobis ? mahalanobis + b0 : nullptr, mahalanobis_class ? mahalanobis_class + b0 : nullptr, st));
    }
    if (do_knn) {
      RD_TRY(ood_rows(f, s0.Df, m, s0.Df, nullptr, Fp, S + l.q, st));
      for (int64_t c0 = 0; c0 < n_bank; c0 += slice) {
        const int nc = (int)(n_bank - c0 < slice ? n_bank - c0 : slice), ncp = (int)round_up(nc, 4);
        TcNtArgs g;
        g.A = S + l.q; g.lda = Fp; g.B = bank + c0 * Fp; g.B_lo = bank_lo + c0 * Fp; g.M = m; g.N = ncp; g.K = Fp;
        g.C = S + l.sim;
        tc_nt_plan(m, ncp, true, &g.BN, &g.n_tiles);
        RD_TRY(tc_nt(g, st));
        RD_TRY(ood_topk(S + l.sim, ncp, m, nc, c0, k, ood_selected(k, n_bank), c0 == 0, c0 + slice >= n_bank,
                        reinterpret_cast<uint64_t*>(S + l.run),
                        S + l.q, bank, Fp, knn ? knn + b0 : nullptr, knn_index ? knn_index + (int64_t)b0 * k : nullptr, st));
      }
    }
  }
  return 0;
}

// SWAG predictive: a chunk of rpc samples (ChunkLayout), then the fp64 sums of mc_accumulate [B, 2*n_classes + 1] and
// one replicate's logits [B, n_classes].
struct SwagScratch : ChunkLayout { int64_t acc, rep; };
static int swag_scratch(const rd_dims* dims, int rpc, SwagScratch* l) {
  RD_TRY(chunk_layout(dims, "rows_per_chunk", rpc, 1, false, 0, false, l));
  l->acc = l->a.take(2LL * dims->B * (2 * dims->n_classes + 1));
  l->rep = l->a.take((int64_t)dims->B * dims->n_classes);
  return 0;
}

size_t rd_swag_predictive_scratch_bytes(const rd_dims* dims, int32_t rows_per_chunk) {
  SwagScratch l;
  if (!dims || swag_scratch(dims, rows_per_chunk, &l) != 0) return 0;
  return (size_t)l.a.off * sizeof(float);
}

// Per replicate: one sample launch into theta_s (the weights are drawn once per replicate), the eval forward of every
// chunk of rpc samples into the replicate's logits, and one mc_accumulate launch.
int rd_raindrop_v2_swag_predictive(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                   const float* times, const int64_t* lengths, const float* node_scale,
                                   const rd_swag_member* members, int32_t n_members, double scale, const uint64_t* rng,
                                   int32_t n_samples, float* theta_s, int64_t n, int32_t rows_per_chunk, void* scratch,
                                   float* mean_probs, float* variance, float* entropies, float* samples, void* stream) {
  const char* fn = "rd_raindrop_v2_swag_predictive";
  Shape s0;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, true, &s0));
  if (!src || !times || !members || !rng || !theta_s || !scratch || !mean_probs || !variance || !entropies ||
      !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (n_members < 1 || n_samples < 1 || rows_per_chunk < 1 || (int64_t)n_members * n_samples > 0x7fffffffLL) {
    set_error("%s: n_members = %d, n_samples = %d and rows_per_chunk = %d must be >= 1 with n_members * n_samples < 2^31",
              fn, n_members, n_samples, rows_per_chunk);
    return -2;
  }
  for (int i = 0; i < n_members; ++i)
    RD_TRY(swag_sample_check(fn, members[i].mean, members[i].sq_mean, members[i].dev, n, members[i].k, scale));
  if (reinterpret_cast<uintptr_t>(theta_s) & 15) { set_error("%s: theta_s must be 16-byte aligned", fn); return -2; }
  SwagScratch l;
  RD_TRY(swag_scratch(dims, rows_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, rpc = rows_per_chunk;
  const int64_t M = (int64_t)n_members * n_samples;
  float* S = (float*)scratch;
  double* acc = reinterpret_cast<double*>(S + l.acc);
  float* rep = S + l.rep;
  for (int64_t r = 0; r < M; ++r) {
    const rd_swag_member& mb = members[r / n_samples];
    RD_TRY(swag_sample(mb.mean, mb.sq_mean, mb.dev, n, mb.k, scale, rng, r, theta_s, st));
    for (int b0 = 0; b0 < B; b0 += rpc) {
      const int m = B - b0 < rpc ? B - b0 : rpc;
      const rd_dims dc = chunk_dims(dims, m, rpc, 0);
      Expanded x{const_cast<float*>(src), const_cast<float*>(statics), const_cast<float*>(times),
                 const_cast<int64_t*>(lengths)};
      if (m < B) {
        x = l.inputs(S, s0.ds);
        RD_TRY(ood_slice_inputs(s0, src, statics, times, lengths, b0, m, x, st));
      }
      RD_TRY(raindrop_fwd(&dc, params, x.src, x.statics, x.times, x.lengths, node_scale, nullptr, S + l.ws,
                          rep + (int64_t)b0 * s0.ncls, nullptr, nullptr, nullptr, 0, st));
    }
    RD_TRY(mc_accumulate(rep, 1, B, s0.ncls, r, M, acc, samples, mean_probs, variance, entropies, r == 0, r == M - 1, st));
  }
  return 0;
}

size_t rd_dp_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)dp_layout(s).total * sizeof(float);
}

int rd_raindrop_v2_per_sample_grad_sqnorms(const rd_dims* dims, const rd_params* params, const float* statics,
                                           const int64_t* lengths, const float* node_scale, const void* workspace,
                                           const float* d_logits, void* scratch, double* sqnorms, void* stream) {
  const char* fn = "rd_raindrop_v2_per_sample_grad_sqnorms";
  Shape s;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s));
  if (!workspace || !d_logits || !scratch || !sqnorms) { set_error("%s: NULL argument", fn); return -2; }
  const DpLayout l = dp_layout(s);
  GradConsumer c;
  c.mode = GRAD_SQNORMS; c.sqnorms = sqnorms; c.partial = reinterpret_cast<double*>((float*)scratch + l.partial);
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits,
                      (float*)scratch + l.bw, RD_BWD_ALL, nullptr, (cudaStream_t)stream, c);
}

size_t rd_per_sample_grads_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)bw_layout(s).total * sizeof(float);
}

int rd_raindrop_v2_per_sample_grads(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                                    const float* node_scale, const void* workspace, const float* d_logits, void* scratch,
                                    float* G, int64_t ldg, void* stream) {
  const char* fn = "rd_raindrop_v2_per_sample_grads";
  Shape s;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s));
  if (!workspace || !d_logits || !scratch || !G) { set_error("%s: NULL argument", fn); return -2; }
  const Trained t = trained(s);
  if (ldg != t.bucket) { set_error("%s: ldg = %lld must be the bucket length %lld", fn, (long long)ldg, (long long)t.bucket); return -2; }
  if (reinterpret_cast<uintptr_t>(G) & 15) { set_error("%s: G must be 16-byte aligned", fn); return -2; }
  GradConsumer c;
  c.mode = GRAD_ROWS; c.G = G;
  c.scale = (float)s.B;      // d_logits holds the gradient of l_b / B (the forward's batch mean): rows are of l_b
  cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(psg_pad(t.f, s.B, G, ldg, st));
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, (float*)scratch,
                      RD_BWD_ALL, nullptr, st, c);
}

int64_t rd_kfac_factors_doubles(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return trained(s).factor_doubles;
}

int64_t rd_ekfac_bases_floats(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return trained(s).base_floats;
}

size_t rd_kfac_factors_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)kfac_layout(s).total * sizeof(float);
}

int rd_raindrop_v2_kfac_factors(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                                const float* node_scale, const void* workspace, const float* d_logits, void* scratch,
                                double* factors, void* stream) {
  const char* fn = "rd_raindrop_v2_kfac_factors";
  Shape s;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s));
  if (!workspace || !d_logits || !scratch || !factors) { set_error("%s: NULL argument", fn); return -2; }
  if (reinterpret_cast<uintptr_t>(scratch) & 15) { set_error("%s: scratch must be 16-byte aligned", fn); return -2; }
  const KfacLayout l = kfac_layout(s);
  GradConsumer c;
  c.mode = GRAD_FACTORS; c.factors = factors; c.kws = (float*)scratch + l.kws; c.kpartial = (float*)scratch + l.kpartial;
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits,
                      (float*)scratch + l.bw, RD_BWD_ALL, nullptr, (cudaStream_t)stream, c);
}

size_t rd_ekfac_rows_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)ekfac_layout(s).total * sizeof(float);
}

// The rotated rows on checked arguments (ldg = the bucket length; G, bases and scratch 16-byte aligned), scratch laid
// out as ekfac_layout(s): the bases' remainder image, the padding columns, then the backward in rotated-rows mode.
static int ekfac_rows(const Shape& s, const rd_dims* dims, const rd_params* params, const float* statics,
                      const int64_t* lengths, const float* node_scale, const void* workspace, const float* d_logits,
                      const float* bases, float* S, float* G, cudaStream_t st) {
  const Trained t = trained(s);
  const EkfacLayout l = ekfac_layout(s);
  GradConsumer c;
  c.mode = GRAD_ROTATED; c.G = G; c.bases = bases; c.bases_lo = S + l.lo; c.rot = S + l.rot;
  c.scale = (float)s.B;      // as rd_raindrop_v2_per_sample_grads: rows are of l_b
  RD_TRY(grad_lo_image(bases, t.base_floats, S + l.lo, st));
  RD_TRY(psg_pad(t.f, s.B, G, t.bucket, st));
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, S + l.bw, RD_BWD_ALL,
                      nullptr, st, c);
}

int rd_raindrop_v2_ekfac_rows(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                              const float* node_scale, const void* workspace, const float* d_logits, const float* bases,
                              void* scratch, float* G, int64_t ldg, void* stream) {
  const char* fn = "rd_raindrop_v2_ekfac_rows";
  Shape s;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s));
  if (!workspace || !d_logits || !bases || !scratch || !G) { set_error("%s: NULL argument", fn); return -2; }
  const int64_t bucket = trained(s).bucket;
  if (ldg != bucket) { set_error("%s: ldg = %lld must be the bucket length %lld", fn, (long long)ldg, (long long)bucket); return -2; }
  if ((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(bases) | reinterpret_cast<uintptr_t>(scratch)) & 15) {
    set_error("%s: G, bases and scratch must be 16-byte aligned", fn);
    return -2;
  }
  return ekfac_rows(s, dims, params, statics, lengths, node_scale, workspace, d_logits, bases, (float*)scratch, G,
                    (cudaStream_t)stream);
}

// Scratch of the logit covariance: the rows scratch, the seed d_logits, the rows of every class and the Gram partials.
struct LaplaceLayout { int64_t rows_scratch, dlog, G, partial, total; };
static LaplaceLayout laplace_layout(const Shape& s, int64_t ldg) {
  LaplaceLayout l;
  Arena a;
  l.rows_scratch = a.take(ekfac_layout(s).total);
  l.dlog = a.take((int64_t)s.B * s.ncls);
  l.G = a.take((int64_t)s.ncls * s.B * ldg);
  l.partial = a.take(2 * laplace_gram_partial_doubles(s.B, s.ncls, ldg));
  l.total = a.off;
  return l;
}

size_t rd_laplace_logit_cov_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0 || s.ncls > RD_LAPLACE_MAX_CLASSES) return 0;
  return (size_t)laplace_layout(s, trained(s).bucket).total * sizeof(float);
}

int rd_raindrop_v2_laplace_logit_cov(const rd_dims* dims, const rd_params* params, const float* statics,
                                     const int64_t* lengths, const float* node_scale, const void* workspace,
                                     const float* bases, const float* w, void* scratch, double* cov, void* stream) {
  const char* fn = "rd_raindrop_v2_laplace_logit_cov";
  Shape s;
  RD_TRY(check_model_call(fn, dims, params, lengths, node_scale, statics, false, &s));
  if (!workspace || !bases || !w || !scratch || !cov) { set_error("%s: NULL argument", fn); return -2; }
  if (s.ncls > RD_LAPLACE_MAX_CLASSES) { set_error("%s: n_classes = %d, at most %d", fn, s.ncls, RD_LAPLACE_MAX_CLASSES); return -2; }
  if ((reinterpret_cast<uintptr_t>(bases) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(scratch)) & 15) {
    set_error("%s: bases, w and scratch must be 16-byte aligned", fn);
    return -2;
  }
  const int64_t ldg = trained(s).bucket;
  const LaplaceLayout l = laplace_layout(s, ldg);
  float* S = (float*)scratch;
  cudaStream_t st = (cudaStream_t)stream;
  for (int c = 0; c < s.ncls; ++c) {
    RD_TRY(laplace_seed(S + l.dlog, s.B, s.ncls, c, st));
    RD_TRY(ekfac_rows(s, dims, params, statics, lengths, node_scale, workspace, S + l.dlog, bases, S + l.rows_scratch,
                      S + l.G + (int64_t)c * s.B * ldg, st));
  }
  return laplace_gram(S + l.G, s.B, s.ncls, ldg, w, reinterpret_cast<double*>(S + l.partial), cov, st);
}

int rd_dp_clip_scale(const rd_dims* dims, const void* workspace, const double* sqnorms, const float* weight,
                     float max_grad_norm, float expected_batch_size, float* d_logits, float* clip_factors, float* loss,
                     void* stream) {
  if (!dims || !workspace || !sqnorms || !weight || !d_logits || !clip_factors || !loss) {
    set_error("rd_dp_clip_scale: NULL argument");
    return -2;
  }
  if (!(max_grad_norm > 0.f) || !(expected_batch_size > 0.f)) {
    set_error("rd_dp_clip_scale: max_grad_norm and expected_batch_size must be > 0");
    return -2;
  }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  const WsLayout w = ws_layout(s);
  return dp_clip(sqnorms, s.B, trained(s).f.n, s.ncls, weight, (double)max_grad_norm, (double)expected_batch_size,
                 (const float*)workspace + w.loss_ps, d_logits, clip_factors, loss, (cudaStream_t)stream);
}

int rd_dp_add_noise(float* grad, int64_t n, const int64_t* field_offsets, const int64_t* field_numel, int32_t n_fields,
                    float noise_std, uint64_t* key, void* stream) {
  if (!grad || !field_offsets || !field_numel || !key || n < 0 || (n & 3) || n_fields < 1 || n_fields > DP_MAX_FIELDS ||
      !(noise_std >= 0.f)) {
    set_error("rd_dp_add_noise: bad arguments");
    return -2;
  }
  DpFields f;
  f.n = n_fields;
  int64_t prev_end = 0;
  for (int i = 0; i < n_fields; ++i) {
    f.off[i] = field_offsets[i]; f.numel[i] = field_numel[i];
    if (f.off[i] < prev_end || (f.off[i] & 3) || f.numel[i] < 0 || f.off[i] + f.numel[i] > n) {
      set_error("rd_dp_add_noise: field %d [%lld, +%lld) is not ascending, 4-aligned and inside the bucket", i,
                (long long)f.off[i], (long long)f.numel[i]);
      return -2;
    }
    prev_end = f.off[i] + f.numel[i];
  }
  if (n == 0) return 0;
  return dp_noise(grad, n, f, noise_std, key, (cudaStream_t)stream);
}

int rd_positional_encoding_bwd(const float* times, const float* d_pe, int64_t n_tokens, const float* timescales_host,
                               int32_t d_pe_width, int64_t ld, int32_t col0, float* d_times, void* stream) {
  if (!times || !d_pe || !timescales_host || !d_times || n_tokens < 0) { set_error("rd_positional_encoding_bwd: bad arguments"); return -2; }
  if (n_tokens == 0) return 0;
  return input_grad(nullptr, nullptr, nullptr, 1, 0, 0, 0, 0.f, nullptr, nullptr, times, d_pe, n_tokens, ld, col0, timescales_host,
                    d_pe_width, nullptr, d_times, nullptr, 0, 0, nullptr, 0, 0, nullptr, (cudaStream_t)stream);
}

int rd_positional_encoding(const float* times, int64_t n_tokens, const float* timescales_host, int32_t d_pe, float* out,
                           int64_t ld, int32_t col0, void* stream) {
  if (!times || !timescales_host || !out || n_tokens < 0) { set_error("rd_positional_encoding: bad arguments"); return -2; }
  if (n_tokens == 0) return 0;
  return posenc(times, n_tokens, timescales_host, d_pe, out, ld, col0, (cudaStream_t)stream);
}

int rd_encoder_head_fwd(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                        uint64_t* rng_state, void* workspace, float* logits, const int64_t* y, float* loss, float* d_logits,
                        void* stream) {
  if (!dims || !params || !lengths || !workspace || !logits) { set_error("rd_encoder_head_fwd: NULL argument"); return -2; }
  return raindrop_fwd(dims, params, nullptr, statics, nullptr, lengths, nullptr, rng_state, (float*)workspace, logits, y, loss,
                      d_logits, 1, (cudaStream_t)stream);
}

int rd_encoder_head_bwd(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                        const void* workspace, const float* d_logits, const rd_grads* grads, void* scratch, float* d_enc_in,
                        void* stream) {
  if (!dims || !params || !lengths || !workspace || !d_logits || !scratch || !d_enc_in) {
    set_error("rd_encoder_head_bwd: NULL argument");
    return -2;
  }
  GradConsumer c{grads ? GRAD_WEIGHTS : GRAD_NONE, grads};
  return raindrop_bwd(dims, params, statics, lengths, nullptr, (const float*)workspace, d_logits, (float*)scratch,
                      RD_BWD_ENCODER, d_enc_in, (cudaStream_t)stream, c);
}

int rd_dropout(const float* x, int64_t n, float p, const uint64_t* rng_captured, uint32_t site, float* y, void* stream) {
  if (!x || !y || !rng_captured || n < 0 || p < 0.f || p >= 1.f) { set_error("rd_dropout: bad arguments"); return -2; }
  if (n == 0) return 0;
  return apply_dropout(x, n, p, rng_captured, site, y, (cudaStream_t)stream);
}

int rd_gather_batch(const float* src, const int64_t* idx, int64_t T, int64_t n_total, int32_t width, int32_t B, float* out,
                    void* stream) {
  if (!src || !idx || !out || T < 0 || n_total < 1 || width < 1 || B < 0) { set_error("rd_gather_batch: bad arguments"); return -2; }
  return gather_batch(src, idx, T, n_total, width, B, out, (cudaStream_t)stream);
}

int rd_assemble_batch(const float* P, const float* Ptime, const float* Pstatic, const int64_t* y, const int64_t* idx,
                      int32_t T, int64_t n_total, int32_t width, int32_t d_static, int32_t B, float* src, float* times,
                      float* statics, int64_t* y_out, int64_t* lengths, void* stream) {
  if (!P || !Ptime || !idx || !src || !times || !lengths || T < 1 || n_total < 1 || width < 1 || B < 0 || (Pstatic && (!statics || d_static < 1)) ||
      (y && !y_out)) {
    set_error("rd_assemble_batch: bad arguments");
    return -2;
  }
  return assemble_batch(P, Ptime, Pstatic, y, idx, T, n_total, width, d_static, B, src, times, statics, y_out, lengths,
                        (cudaStream_t)stream);
}

size_t rd_feature_stats_scratch_bytes(int64_t n, int32_t T, int32_t F) {
  if (n < 1 || T < 1 || F < 1) return 0;
  return (size_t)feature_stats_scratch_bytes(n, T, F);
}

int rd_feature_stats(const float* raw, int64_t n, int32_t T, int32_t F, float* mean, float* stdv, void* scratch, void* stream) {
  if (!raw || !mean || !stdv || !scratch || n < 1 || T < 1 || F < 1) { set_error("rd_feature_stats: bad arguments"); return -2; }
  return feature_stats(raw, n, T, F, mean, stdv, scratch, (cudaStream_t)stream);
}

int rd_mask_normalize(const float* raw, const float* mean, const float* stdv, int64_t n, int32_t T, int32_t F, float* out,
                      const float* minutes, float* times_out, void* stream) {
  if (!raw || !mean || !stdv || !out || n < 1 || T < 1 || F < 1 || (minutes && !times_out)) {
    set_error("rd_mask_normalize: bad arguments");
    return -2;
  }
  return mask_normalize(raw, mean, stdv, n, T, F, out, minutes, times_out, (cudaStream_t)stream);
}

int rd_zero_features(float* P, int64_t T, int32_t B, int32_t width, const int64_t* idx, int32_t K, int32_t per_sample,
                     void* stream) {
  if (!P || !idx || T < 0 || B < 0 || width < 2 || K < 0) { set_error("rd_zero_features: bad arguments"); return -2; }
  return zero_features(P, T, B, width, idx, K, per_sample, (cudaStream_t)stream);
}

int rd_cross_entropy_fwd_bwd(const float* logits, const int64_t* y, int32_t B, int32_t ncls, float* loss,
                             float* d_logits, void* stream) {
  if (!logits || !y || !loss || B < 1 || ncls < 1) { set_error("rd_cross_entropy_fwd_bwd: bad arguments"); return -2; }
  return cross_entropy(logits, y, B, ncls, loss, d_logits, (cudaStream_t)stream);
}

int rd_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                 const float* lr_dev, float beta1, float beta2, float eps, float grad_scale, int64_t* step, void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || !step || n < 0) { set_error("rd_adam_step: bad arguments"); return -2; }
  if (n == 0) return 0;
  return adam(param, grad, exp_avg, exp_avg_sq, n, lr, lr_dev, beta1, beta2, eps, grad_scale, step, (cudaStream_t)stream);
}

int rd_debug_dropout_mask(const uint64_t* rng_captured, uint32_t site, int64_t n, float p, float* out, void* stream) {
  if (!rng_captured || !out || n < 0 || p < 0.f || p >= 1.f) { set_error("rd_debug_dropout_mask: bad arguments"); return -2; }
  if (n == 0) return 0;
  return apply_dropout(nullptr, n, p, rng_captured, site, out, (cudaStream_t)stream);
}

int rd_debug_tc_nt(rd_debug_tc_nt_args* a, void* stream) {
  if (!a) { set_error("rd_debug_tc_nt: bad arguments"); return -2; }
  if (a->BN == 0 || a->n_tiles == 0) tc_nt_plan(a->M, a->N, a->B_lo != nullptr, &a->BN, &a->n_tiles);
  TcNtArgs n;
  n.A = a->A; n.lda = a->lda; n.B = a->B; n.B_lo = a->B_lo;
  n.M = a->M; n.N = a->N; n.K = a->K; n.BN = a->BN; n.n_tiles = a->n_tiles;
  n.C = a->C;
  n.bias = a->bias; n.relu = a->relu;
  n.scale = a->scale; n.scale_mod = a->scale_mod;
  n.gate = a->gate; n.gate_ld = a->gate_ld; n.gate_scale = a->gate_scale;
  n.drop_p = a->drop_p; n.rng = a->rng; n.drop_site = a->drop_site; n.rep.B = a->rep_B; n.rep.Bc = a->rep_Bc;
  n.drop_mask = a->drop_mask; n.drop_mask_ld = a->drop_mask_ld;
  n.resid = a->resid; n.resid_ld = a->resid_ld;
  n.round_out = a->round_out;
  n.perm = a->perm; n.pB = a->pB; n.pN = a->pN; n.pD = a->pD;
  return tc_nt(n, (cudaStream_t)stream);
}

int rd_debug_gemm_f32(rd_debug_gemm_args* a, float* partial, void* stream) {
  if (!a) { set_error("rd_debug_gemm_f32: bad arguments"); return -2; }
  GemmP g;
  g.A = a->A; g.B = a->B; g.C = a->C;
  g.M = a->M; g.N = a->N; g.K = a->K; g.ta = a->ta; g.tb = a->tb;
  g.sAi = a->sAi; g.sAk = a->sAk; g.sBk = a->sBk; g.sBj = a->sBj; g.sCi = a->sCi; g.sCj = a->sCj;
  g.nz = a->nz; g.nz_inner = a->nz_inner;
  g.sAzo = a->sAzo; g.sAzi = a->sAzi; g.sBzo = a->sBzo; g.sBzi = a->sBzi; g.sCzo = a->sCzo; g.sCzi = a->sCzi;
  if (a->nsplit == 0) {
    a->partial_floats = gemm_splitk_plan(a->M, a->N, a->K, &a->nsplit);
    if (a->partial_floats > 0 && !partial) {
      set_error("rd_debug_gemm_f32: the split-K plan (%d splits) needs a partial buffer of %lld floats", a->nsplit,
                (long long)a->partial_floats);
      return -2;
    }
  }
  g.nsplit = a->nsplit; g.partial = partial; g.asum = a->asum;
  g.alpha = a->alpha; g.bias = a->bias; g.relu = a->relu;
  g.rowscale = a->rowscale; g.rowscale_mod = a->rowscale_mod;
  g.gate = a->gate; g.gate_ld = a->gate_ld; g.gate_scale = a->gate_scale;
  g.drop_p = a->drop_p; g.rng = a->rng; g.drop_site = a->drop_site; g.rep.B = a->rep_B; g.rep.Bc = a->rep_Bc;
  g.resid = a->resid; g.resid_ld = a->resid_ld;
  g.perm = a->perm; g.pB = a->pB; g.pN = a->pN; g.pdob = a->pdob; g.pD = a->pD;
  return gemm(g, (cudaStream_t)stream);
}

int rd_debug_split_weights(const float* w, int32_t rows, int32_t cols, float* lo, float* t, float* t_lo, float* rn,
                           float* rn_t, void* stream) {
  if (!w || rows < 1 || cols < 1 || (t == nullptr) != (t_lo == nullptr)) {
    set_error("rd_debug_split_weights: bad arguments");
    return -2;
  }
  WeightSplit it{w, rows, cols, lo, t, t_lo, rn, rn_t};
  return split_weights(&it, 1, (cudaStream_t)stream);
}

int rd_debug_colsum(const float* x, int64_t rows, int32_t cols, int64_t ld, float* out, float* scratch, void* stream) {
  if (!x || !out || !scratch || rows < 1 || cols < 0 || ld < cols) { set_error("rd_debug_colsum: bad arguments"); return -2; }
  return colsum(x, rows, cols, ld, out, scratch, (cudaStream_t)stream);
}

int rd_debug_wgrad_group(const rd_wgrad_item* items, const uint64_t* partial_bytes, int32_t n,
                         const rd_debug_colsum_item* cs, int32_t ncs, rd_debug_wgrad_plan* plan, void* stream) {
  if (n < 0 || ncs < 0 || n > WG_MAX || ncs > CS_MAX) {
    set_error("rd_debug_wgrad_group: at most %d problems and %d column sums per launch", WG_MAX, CS_MAX);
    return -2;
  }
  if (!plan || (n > 0 && (!items || !partial_bytes)) || (ncs > 0 && !cs)) { set_error("rd_debug_wgrad_group: bad arguments"); return -2; }
  WgradItem it[WG_MAX];
  ColsumItem c[CS_MAX];
  for (int i = 0; i < n; ++i) {
    const rd_wgrad_item& a = items[i];
    if (!a.d_out || !a.x || !a.d_weight || !a.partial || a.rows < 1) {
      set_error("rd_debug_wgrad_group: problem %d has a NULL pointer or no rows", i);
      return -2;
    }
    if (!tc_wgrad_supported(a.out_features, a.in_features, a.out_features, a.in_features, a.d_out, a.x) ||
        (reinterpret_cast<uintptr_t>(a.partial) & 15)) {
      set_error("rd_debug_wgrad_group: problem %d is not one the tensor-core kernel takes (out / in features multiples "
                "of 4 and >= 16, d_out, x and partial 16-byte aligned)", i);
      return -2;
    }
    const size_t need = rd_linear_wgrad_partial_bytes(a.rows, a.out_features, a.in_features);
    if (partial_bytes[i] < need) {
      set_error("rd_debug_wgrad_group: problem %d has a partial buffer of %llu bytes, it needs %llu", i,
                (unsigned long long)partial_bytes[i], (unsigned long long)need);
      return -2;
    }
    it[i] = WgradItem{a.d_out, a.out_features, a.x, a.in_features, a.rows, a.out_features, a.in_features, a.d_weight,
                      a.d_bias, (float*)a.partial};
  }
  for (int i = 0; i < ncs; ++i) {
    const rd_debug_colsum_item& s = cs[i];
    if (!s.partial || !s.out || s.nsplit < 1 || s.ncols < 1 || (s.nsplit > 1 && s.stride < s.ncols)) {
      set_error("rd_debug_wgrad_group: bad column sum %d", i);
      return -2;
    }
    c[i] = ColsumItem{s.partial, s.stride, s.nsplit, s.ncols, s.out};
  }
  static_assert(WG_MAX == 12 && CS_MAX == 36, "the limits rd_debug_wgrad_group and its plan are declared with");
  WgradPlan pl{};
  RD_TRY(tc_wgrad_group(it, n, c, ncs, (cudaStream_t)stream, &pl));
  plan->BN = pl.BN;
  plan->rows_target = pl.rows_target;
  for (int i = 0; i < n; ++i) { plan->nsplit[i] = pl.sp[i].nsplit; plan->rows_per_split[i] = pl.sp[i].rows_per_split; }
  return 0;
}

int rd_debug_per_sample_linear(const rd_debug_per_sample_item* items, int32_t n, int32_t B, int32_t mode, double* sqnorms,
                               int32_t nf, double* partial, uint64_t partial_bytes, float* G, int64_t ldg, float scale,
                               rd_debug_per_sample_plan* plan, void* stream) {
  const char* fn = "rd_debug_per_sample_linear";
  static_assert(DP_MAX_ITEMS == 32, "the item limit rd_debug_per_sample_linear is declared with");
  if (n < 1 || n > DP_MAX_ITEMS) { set_error("%s: %d items, it takes 1 to %d", fn, n, DP_MAX_ITEMS); return -2; }
  if (mode != RD_PS_SQNORMS && mode != RD_PS_ROWS && mode != RD_PS_ROTATED) {
    set_error("%s: unknown mode %d", fn, mode);
    return -2;
  }
  const bool sq = mode == RD_PS_SQNORMS;
  if (!items || !plan || (sq && (!sqnorms || !partial)) || (!sq && !G)) { set_error("%s: NULL argument", fn); return -2; }
  if (B < 1 || (sq && nf < 1) || (!sq && ldg < 1)) {
    set_error("%s: bad sizes (B=%d nf=%d ldg=%lld)", fn, B, nf, (long long)ldg);
    return -2;
  }
  DpNormGroup g;
  PsgGroup pg;
  long long blk = 0;
  for (int i = 0; i < n; ++i) {
    const rd_debug_per_sample_item& a = items[i];
    const int xw = a.in_features + (mode == RD_PS_ROTATED ? 1 : 0);     // the columns of x the kernel reads
    if (!a.d_out || !a.x) { set_error("%s: item %d has a NULL pointer", fn, i); return -2; }
    if (a.R < 1 || a.out_features < 1 || a.in_features < 1 || a.sstride < 1 || a.rstride < 1 || a.ld_out < a.out_features ||
        a.ld_x < xw) {
      set_error("%s: item %d has bad sizes (R=%d out=%d in=%d sstride=%lld rstride=%lld ld_out=%lld ld_x=%lld)", fn, i, a.R,
                a.out_features, a.in_features, (long long)a.sstride, (long long)a.rstride, (long long)a.ld_out,
                (long long)a.ld_x);
      return -2;
    }
    plan[i].ghost = 0;
    plan[i].tm = (int32_t)ceil_div(a.out_features, 64);
    if (sq) {
      if (a.form < -1 || a.form > 1) { set_error("%s: item %d has unknown form %d", fn, i, a.form); return -2; }
      if (a.fw < 0 || a.fw >= nf || a.fb < 0 || a.fb >= nf) {
        set_error("%s: item %d has fields (%d, %d) outside nf=%d", fn, i, a.fw, a.fb, nf);
        return -2;
      }
      DpNormItem& q = g.it[i];
      q.Y = a.d_out; q.X = a.x; q.ldy = a.ld_out; q.ldx = a.ld_x; q.sstride = a.sstride; q.rstride = a.rstride; q.blk0 = blk;
      q.Nout = a.out_features; q.Kin = a.in_features; q.R = a.R;
      q.ghost = (a.form < 0 ? dp_ghost(a.R, a.out_features, a.in_features) : a.form == 1) ? 1 : 0;
      q.ntiles = dp_norm_tiles(q.R, q.Nout, q.Kin, q.ghost != 0, &q.tm, &q.tn);
      q.fw = a.fw; q.fb = a.fb;
      plan[i].ghost = q.ghost; plan[i].tm = q.tm; plan[i].tn = q.tn; plan[i].ntiles = q.ntiles;
    } else {
      const long long wn = (long long)a.out_features * a.in_features;
      if (a.gw < 0 || a.gw + wn > ldg || a.gb < 0 || a.gb + a.out_features > ldg) {
        set_error("%s: item %d has fields at (%lld, %lld) that leave the row of %lld", fn, i, (long long)a.gw,
                  (long long)a.gb, (long long)ldg);
        return -2;
      }
      PsgItem& q = pg.it[i];
      q.Y = a.d_out; q.X = a.x; q.ldy = a.ld_out; q.ldx = a.ld_x; q.sstride = a.sstride; q.rstride = a.rstride; q.blk0 = blk;
      q.gw = a.gw; q.gb = a.gb; q.Nout = a.out_features; q.Kin = a.in_features; q.R = a.R;
      q.ntiles = psg_tiles(q.Nout, q.Kin, &q.tn);
      plan[i].tn = q.tn; plan[i].ntiles = q.ntiles;
    }
    blk += (long long)B * plan[i].ntiles;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (!sq) {
    pg.n = n;
    return psg_group(pg, B, G, ldg, scale, st, mode == RD_PS_ROTATED);
  }
  if (partial_bytes < 16ull * (unsigned long long)blk) {
    set_error("%s: a partial buffer of %llu bytes, it needs %llu", fn, (unsigned long long)partial_bytes,
              16ull * (unsigned long long)blk);
    return -2;
  }
  g.n = n;
  return dp_norm_group(g, B, partial, sqnorms, nf, st);
}

int64_t rd_debug_layernorm_scratch_floats(int64_t rows, int32_t D) {
  return rows < 1 || D < 1 ? 0 : ln_bwd_scratch_floats(rows, D);
}

int rd_debug_layernorm(rd_debug_layernorm_args* a, void* stream) {
  const char* fn = "rd_debug_layernorm";
  if (!a) { set_error("%s: NULL argument", fn); return -2; }
  if (!a->forward && !a->backward) { set_error("%s: neither half requested", fn); return -2; }
  if (a->rows < 1 || a->D < 1) { set_error("%s: bad sizes (rows=%lld D=%d)", fn, (long long)a->rows, a->D); return -2; }
  if (!a->x || !a->gamma || !a->stats || (a->forward && (!a->beta || !a->y)) ||
      (a->backward && (!a->dy || !a->dx || !a->scratch || !a->dgamma || !a->dbeta))) {
    set_error("%s: NULL pointer", fn);
    return -2;
  }
  if (a->backward) {
    if (!(a->drop_p >= 0.f && a->drop_p < 1.f)) { set_error("%s: drop_p %g outside [0, 1)", fn, (double)a->drop_p); return -2; }
    if (a->drop_p > 0.f && (!a->rng || !a->dx_drop)) { set_error("%s: drop_p > 0 needs rng and dx_drop", fn); return -2; }
    if (a->keep_bits && a->keep_ld < (a->D + 31) / 32) {
      set_error("%s: keep_ld %d below ceil(D / 32) = %d", fn, a->keep_ld, (a->D + 31) / 32);
      return -2;
    }
    const int64_t need = ln_bwd_scratch_floats(a->rows, a->D);
    if (a->scratch_floats < need) {
      set_error("%s: a scratch buffer of %lld floats, it needs %lld", fn, (long long)a->scratch_floats, (long long)need);
      return -2;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  a->fwd_class = a->bwd_class = -1;
  a->chunks = 0;
  a->keep_source = RD_LN_KEEP_NONE;
  if (a->forward) {
    a->fwd_class = layernorm_fwd_class(a->x, a->gamma, a->beta, a->y, a->D);
    RD_TRY(layernorm_fwd(a->x, a->gamma, a->beta, a->rows, a->D, a->eps, a->y, a->stats, st));
  }
  if (!a->backward) return 0;
  a->bwd_class = layernorm_bwd_class(a->x, a->gamma, a->dy, a->dx, a->dx_drop, a->drop_p, a->D);
  const bool fused = a->bwd_class != LN_SPLIT_VEC && a->bwd_class != LN_SPLIT_SCALAR;
  if (a->drop_p > 0.f) a->keep_source = fused && a->keep_bits ? RD_LN_KEEP_BITS : RD_LN_KEEP_PHILOX;
  int chunks = 0;
  RD_TRY(layernorm_bwd(a->x, a->stats, a->gamma, a->dy, a->rows, a->D, a->dx, a->scratch, a->dx_drop, a->drop_p, a->rng,
                       a->site, &chunks, st, a->keep_bits, a->keep_ld));
  a->chunks = chunks;
  // GradConsumer::ln in weights mode: the two column sums of the partial rows, items of one grouped reduction launch
  WgradQueue q;
  RD_TRY(q.colsum(a->scratch, 2LL * a->D, chunks, a->D, a->dgamma, st));
  RD_TRY(q.colsum(a->scratch + a->D, 2LL * a->D, chunks, a->D, a->dbeta, st));
  return q.flush(st);
}

int rd_debug_per_sample_layernorm(int32_t mode, const float* x, const float* stats, const float* dy, int32_t T, int32_t B,
                                  int32_t D, double* sqnorms, int32_t nf, int32_t fw, int32_t fb, float* G, int64_t ldg,
                                  int64_t gw, int64_t gb, float scale, void* stream) {
  const char* fn = "rd_debug_per_sample_layernorm";
  if (mode != RD_PS_SQNORMS && mode != RD_PS_ROWS) { set_error("%s: unknown mode %d", fn, mode); return -2; }
  const bool sq = mode == RD_PS_SQNORMS;
  if (!x || !stats || !dy || (sq && !sqnorms) || (!sq && !G)) { set_error("%s: NULL argument", fn); return -2; }
  if (T < 1 || B < 1 || D < 1) { set_error("%s: bad sizes (T=%d B=%d D=%d)", fn, T, B, D); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  if (sq) {
    if (fw < 0 || fw >= nf || fb < 0 || fb >= nf) { set_error("%s: fields (%d, %d) outside nf=%d", fn, fw, fb, nf); return -2; }
    return dp_ln_sqnorm(x, stats, dy, T, B, D, sqnorms, nf, fw, fb, st);
  }
  if (gw < 0 || gw + D > ldg || gb < 0 || gb + D > ldg) {
    set_error("%s: fields at (%lld, %lld) that leave the row of %lld", fn, (long long)gw, (long long)gb, (long long)ldg);
    return -2;
  }
  return psg_ln(x, stats, dy, T, B, D, G, ldg, gw, gb, scale, st);
}

}  // extern "C"
