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

// Backward scratch.  The weight gradients are DEFERRED: every linear layer's (dY, X) operand pair stays alive in
// its own buffer until one grouped tensor-core launch (tc_wgrad_group) reduces them all, so dY buffers and the
// split-K partial buffers are per layer / per problem instead of ping-pong.
struct BwLayout {
  int64_t dfeat, dhpre, gA, gB, gD, dP, gO2, gO1, partial, total;
  struct { int64_t K2, gF, K1, dqkv, wp[4], ln[2]; } l[RD_MAX_LAYERS];   // wp: linear2, linear1, out_proj, in_proj partials; ln: norm2, norm1
  int64_t wp_ob[2];
  int64_t partial_floats;
};

int64_t splitk_partial_floats(int Nout, int Kin, int64_t rows) {
  int ns;
  return gemm_splitk_plan(Nout, Kin, (int)rows, &ns);
}

BwLayout bw_layout(const Shape& s) {
  BwLayout b;
  Arena a;
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
    b.l[l].wp[0] = a.take(tc_wgrad_partial_floats(s.D, s.nhid, s.M2));
    b.l[l].wp[1] = a.take(tc_wgrad_partial_floats(s.nhid, s.D, s.M2));
    b.l[l].wp[2] = a.take(tc_wgrad_partial_floats(s.D, s.D, s.M2));
    b.l[l].wp[3] = a.take(tc_wgrad_partial_floats(3 * s.D, s.D, s.M2));
    b.l[l].ln[0] = a.take(ln_bwd_scratch_floats(s.M2, s.D));      // per-CTA dgamma/dbeta partial rows, reduced with the group
    b.l[l].ln[1] = a.take(ln_bwd_scratch_floats(s.M2, s.D));
  }
  b.gO2 = a.take(s.M1 * s.C);
  b.gO1 = a.take(s.M1 * s.C);
  b.wp_ob[0] = a.take(tc_wgrad_partial_floats(s.C, s.C, s.M1));
  b.wp_ob[1] = a.take(tc_wgrad_partial_floats(s.C, s.C, s.M1));
  // shared split-K scratch of the CUDA-core fallback (shapes the tensor-core kernel does not take)
  int64_t pf = 0;
  auto upd = [&](int no, int ki, int64_t rows) { int64_t v = splitk_partial_floats(no, ki, rows); if (v > pf) pf = v; };
  upd(s.C, s.C, s.M1);
  upd(3 * s.D, s.D, s.M2); upd(s.D, s.D, s.M2); upd(s.nhid, s.D, s.M2); upd(s.D, s.nhid, s.M2);
  b.partial_floats = pf;
  b.partial = a.take(pf);
  b.total = a.off;
  return b;
}

// ---- DP-SGD per-sample norm pass -----------------------------------------------------------------------------------
// Trained tensors, in used_param_fields order: the head (emb weight / bias when d_static > 0, mlp_static.0, mlp_static.2),
// 12 per encoder layer, the two lin_value pairs.
int dp_head_fields(const Shape& s) { return s.ds > 0 ? 6 : 4; }
int dp_n_fields(const Shape& s) { return dp_head_fields(s) + 12 * s.L + 4; }

// Field table of the flat gradient bucket (TrainStep's layout): each trained tensor at a 4-aligned offset, in the order
// above.  Returns the bucket length.
int64_t bucket_fields(const Shape& s, DpFields* f) {
  int64_t n[DP_MAX_FIELDS];
  int k = 0;
  if (s.ds > 0) { n[k++] = (int64_t)s.emb * s.ds; n[k++] = s.emb; }
  n[k++] = (int64_t)s.Df * s.Df; n[k++] = s.Df; n[k++] = (int64_t)s.ncls * s.Df; n[k++] = s.ncls;
  for (int l = 0; l < s.L; ++l) {
    const int64_t D = s.D, H = s.nhid;
    const int64_t v[12] = {3 * D * D, 3 * D, D * D, D, H * D, H, D * H, D, D, D, D, D};
    for (int i = 0; i < 12; ++i) n[k++] = v[i];
  }
  for (int i = 0; i < 2; ++i) { n[k++] = (int64_t)s.C * s.C; n[k++] = s.C; }
  int64_t off = 0;
  for (int i = 0; i < k; ++i) { f->off[i] = off; f->numel[i] = n[i]; off += round_up(n[i], 4); }
  f->n = k;
  return off;
}

// EK-FAC blocks: one per queued linear layer, in bucket order (per encoder layer in_proj, out_proj, linear1, linear2;
// then lin_value of ob-prop layers 1 and 2).  a, s: offsets (doubles) of A [(Kin + 1)^2] and S [Nout^2] in the caller's
// factors; qs, qa, qb: offsets (floats) of Q_S^T [Nout, Nout], Q_A[:Kin]^T [Np, Kin] and Q_A[Kin] [Np] in the caller's
// bases, Np = Kin + 1 rounded up to 4 (rows past Kin + 1 are 0); each piece starts 4-aligned.
struct KfacBlock { int Nout, Kin, Np; int64_t a, s, qs, qa, qb; };
struct KfacBlocks { KfacBlock b[4 * RD_MAX_LAYERS + 2]; int n; int64_t factor_doubles, base_floats; };
KfacBlocks kfac_blocks(const Shape& s) {
  KfacBlocks k;
  k.n = 0;
  int64_t a = 0, q = 0;
  auto add = [&](int Nout, int Kin) {
    KfacBlock& o = k.b[k.n++];
    o.Nout = Nout; o.Kin = Kin; o.Np = (int)round_up(Kin + 1, 4);
    o.a = a; a += (int64_t)(Kin + 1) * (Kin + 1);
    o.s = a; a += (int64_t)Nout * Nout;
    o.qs = q; q += round_up((int64_t)Nout * Nout, 4);
    o.qa = q; q += (int64_t)o.Np * Kin;
    o.qb = q; q += o.Np;
  };
  for (int l = 0; l < s.L; ++l) { add(3 * s.D, s.D); add(s.D, s.D); add(s.nhid, s.D); add(s.D, s.nhid); }
  add(s.C, s.C); add(s.C, s.C);
  k.factor_doubles = a; k.base_floats = q;
  return k;
}
// the block of the weight field fw (a queued item's)
int kfac_block_of(const Shape& s, int fw) {
  const int f = fw - dp_head_fields(s);
  return f < 12 * s.L ? 4 * (f / 12) + (f % 12) / 2 : 4 * s.L + (f - 12 * s.L) / 2;
}

// Per-sample items of one backward phase, queued where the training path queues the weight-gradient items of the same
// (dY, X) pairs, and flushed as one group launch.  Modes: squared norms into `sqnorms` (dp_norm_group; the partial
// sums of a phase start at `partial` again: the previous phase's launches have completed by then, stream order); with
// G set, the per-sample gradient rows themselves (psg_group), scaled by `scale`, and with `bases` also set, the EK-FAC
// rows: each item's operands rotated into `rot` first (kfac_flush); with `factors` set, the EK-FAC factor sums of
// every item (kfac_flush).
struct DpQueue;
int kfac_flush(DpQueue& q, cudaStream_t st);
struct DpQueue {
  DpNormGroup g;
  PsgGroup pg;
  long long blk = 0;
  int B = 0, nf = 0;
  double* sqnorms = nullptr; double* partial = nullptr;
  float* G = nullptr; long long ldg = 0; float scale = 1.f; DpFields fields;     // rows mode
  const Shape* shape = nullptr; const KfacBlocks* kb = nullptr; int blk_of[DP_MAX_ITEMS];   // EK-FAC modes
  const float* bases = nullptr; const float* bases_lo = nullptr; float* rot = nullptr;     // rotated rows
  double* factors = nullptr; float* kws = nullptr; float* kpartial = nullptr;             // factors
  DpQueue() { g.n = 0; pg.n = 0; }
  void add(const float* Y, int64_t ldy, const float* X, int64_t ldx, int Nout, int Kin, int R, int64_t sstride,
           int64_t rstride, int fw) {
    if (G || factors) {
      if (kb) blk_of[pg.n] = kfac_block_of(*shape, fw);
      PsgItem& o = pg.it[pg.n++];
      o.Y = Y; o.X = X; o.ldy = ldy; o.ldx = ldx; o.sstride = sstride; o.rstride = rstride; o.blk0 = blk;
      o.gw = G ? fields.off[fw] : 0; o.gb = G ? fields.off[fw + 1] : 0;
      o.Nout = Nout; o.Kin = Kin; o.R = R; o.ntiles = psg_tiles(Nout, Kin, &o.tn);
      blk += (long long)B * o.ntiles;
      return;
    }
    DpNormItem& o = g.it[g.n++];
    o.Y = Y; o.X = X; o.ldy = ldy; o.ldx = ldx; o.sstride = sstride; o.rstride = rstride; o.blk0 = blk;
    o.Nout = Nout; o.Kin = Kin; o.R = R; o.ghost = dp_ghost(R, Nout, Kin) ? 1 : 0;
    o.ntiles = dp_norm_tiles(R, Nout, Kin, &o.tm, &o.tn);
    o.fw = fw; o.fb = fw + 1;
    blk += (long long)B * o.ntiles;
  }
  int ln(const float* x, const float* stats, const float* dy, int T, int D, int fw, int fb, cudaStream_t st) {
    if (factors) return 0;
    if (G) return psg_ln(x, stats, dy, T, B, D, G, ldg, fields.off[fw], fields.off[fb], scale, st);
    return dp_ln_sqnorm(x, stats, dy, T, B, D, sqnorms, nf, fw, fb, st);
  }
  int head(const Shape& s, const float* dlogits, const float* hpre, const float* dh, const float* feat, const float* dfeat,
           const float* statics, cudaStream_t st) {
    if (factors) return 0;
    if (G) return psg_head(B, s.D, s.Df, s.ds, s.ncls, dlogits, hpre, dh, feat, dfeat, statics, G, ldg, fields.off, scale, st);
    return dp_head_sqnorm(B, s.D, s.Df, s.ds, s.ncls, dlogits, hpre, dh, feat, dfeat, statics, sqnorms, nf, st);
  }
  int flush(cudaStream_t st) {
    int rc = kb ? kfac_flush(*this, st) : G ? psg_group(pg, B, G, ldg, scale, st) : dp_norm_group(g, B, partial, sqnorms, nf, st);
    g.n = 0; pg.n = 0; blk = 0;
    return rc;
  }
};

// CTAs (= partial pairs) of the larger of the two phases' group launches
int64_t dp_partial_blocks(const Shape& s) {
  int tm, tn;
  int64_t enc = (int64_t)s.L * (dp_norm_tiles(s.T, s.D, s.nhid, &tm, &tn) + dp_norm_tiles(s.T, s.nhid, s.D, &tm, &tn) +
                                dp_norm_tiles(s.T, s.D, s.D, &tm, &tn) + dp_norm_tiles(s.T, 3 * s.D, s.D, &tm, &tn));
  int64_t ob = 2LL * dp_norm_tiles(s.N, s.C, s.C, &tm, &tn);
  return (int64_t)s.B * (enc > ob ? enc : ob);
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

// ---- integrated gradients ------------------------------------------------------------------------------------------
// A chunk of mc path steps runs on B*mc rows.  The arithmetic of its ob-prop GEMMs is resolved once, from the FULL
// chunk's row count (obprop_mode 0 depends on it), and every chunk and the endpoint forward run with that explicit mode:
// a ragged tail chunk with fewer rows cannot switch arithmetic.
rd_dims ig_dims(const rd_dims* d, int rows, int mc) {
  rd_dims e = *d;
  e.obprop_mode = obprop_tc_exact((int64_t)d->B * mc * d->N, d->T * d->d_ob, d->obprop_mode) ? 2 : 1;
  e.B = rows;
  e.training = 0;
  return e;
}

// Scratch of rd_raindrop_v2_integrated_gradients: the forward workspace of max(B*mc, 2B) rows (chunks and the endpoint
// forward), the chunk's backward scratch, the input-gradient buffers (W1^T, its remainder, dX0), the expanded inputs
// (max(B*mc, 2B) rows), the chunk's one-hot d_logits and logits, and the running sums [B*N*T] and [B, d_static].
struct IgcLayout { int64_t ws, sc, W1t, W1tlo, dX0, src, statics, times, lengths, dlogits, logits, acc_src, acc_static, total; };
int ig_layout(const rd_dims* dims, int mc, IgcLayout* l) {
  if (mc < 1 || (int64_t)dims->B * mc > (1LL << 30)) { set_error("steps_per_chunk = %d out of range", mc); return -2; }
  const int Bc = dims->B * mc, Bx = Bc > 2 * dims->B ? Bc : 2 * dims->B;
  const rd_dims dc = ig_dims(dims, Bc, mc), dx = ig_dims(dims, Bx, mc);
  Shape sc, sx;
  RD_TRY(make_shape(&dc, &sc));
  RD_TRY(make_shape(&dx, &sx));
  Arena a;
  l->ws = a.take(ws_layout(sx).total);
  l->sc = a.take(bw_layout(sc).total);
  l->W1t = a.take((int64_t)sc.C * sc.C);
  l->W1tlo = a.take((int64_t)sc.C * sc.C);
  l->dX0 = a.take(sc.M1 * sc.C);
  l->src = a.take(sx.M2 * 2 * sx.N);
  l->statics = a.take((int64_t)Bx * sx.ds);
  l->times = a.take(sx.M2);
  l->lengths = a.take(2LL * Bx);
  l->dlogits = a.take((int64_t)Bc * sc.ncls);
  l->logits = a.take((int64_t)Bc * sc.ncls);
  l->acc_src = a.take((int64_t)dims->B * sc.N * sc.T);
  l->acc_static = a.take((int64_t)dims->B * sc.ds);
  l->total = a.off;
  return 0;
}

// ---- coalition attribution (Shapley-value sampling, ablation) -------------------------------------------------------
// Scratch of rd_raindrop_v2_coalition_attribution and rd_raindrop_v2_cell_coalition_attribution: the eval forward
// workspace and the expanded inputs of max(B*cc, 2B) rows (chunks of cc coalitions and the endpoint forward), the
// chunk's logits, the fp64 running sums [B, P] and the chunk's keep table [cc, P] (uint8, Shapley).  The ob-prop mode is pinned
// from B*cc rows by ig_dims, as for integrated gradients.
struct CoalLayout { int64_t ws, src, statics, times, lengths, logits, acc, keep, total; };
int coalition_layout(const rd_dims* dims, int n_players, int cc, CoalLayout* l) {
  if (cc < 1 || (int64_t)dims->B * cc > (1LL << 30)) { set_error("coalitions_per_chunk = %d out of range", cc); return -2; }
  if (n_players < 1) { set_error("n_players = %d must be >= 1", n_players); return -2; }
  const int Bc = dims->B * cc, Bx = Bc > 2 * dims->B ? Bc : 2 * dims->B;
  const rd_dims dx = ig_dims(dims, Bx, cc);
  Shape sx;
  RD_TRY(make_shape(&dx, &sx));
  Arena a;
  l->ws = a.take(ws_layout(sx).total);
  l->src = a.take(sx.M2 * 2 * sx.N);
  l->statics = a.take((int64_t)Bx * sx.ds);
  l->times = a.take(sx.M2);
  l->lengths = a.take(2LL * Bx);
  l->logits = a.take((int64_t)Bc * sx.ncls);
  l->acc = a.take(2LL * dims->B * n_players);
  l->keep = a.take(ceil_div((int64_t)cc * n_players, 4));
  l->total = a.off;
  return 0;
}

// ---- Monte Carlo dropout -------------------------------------------------------------------------------------------
// A chunk of cc replicates is one training-mode forward on B*cc replicate-major rows.  Its ob-prop arithmetic is pinned
// from the full chunk's row count, as for integrated gradients, so a ragged tail chunk cannot switch it.
rd_dims mc_dims(const rd_dims* d, int rows, int cc) {
  rd_dims e = ig_dims(d, rows, cc);
  e.training = 1;
  return e;
}
// Scratch of rd_raindrop_v2_mc_dropout: the training forward workspace of B*cc rows, the expanded inputs, the chunk's
// logits and the fp64 sums [B, 2*n_classes + 1].
struct McLayout { int64_t ws, src, statics, times, lengths, logits, acc, total; };
int mc_layout(const rd_dims* dims, int cc, McLayout* l) {
  if (cc < 1 || (int64_t)dims->B * cc > (1LL << 30)) { set_error("replicates_per_chunk = %d out of range", cc); return -2; }
  const int Bc = dims->B * cc;
  const rd_dims dc = mc_dims(dims, Bc, cc);
  Shape sc;
  RD_TRY(make_shape(&dc, &sc));
  Arena a;
  l->ws = a.take(ws_layout(sc).total);
  l->src = a.take(sc.M2 * 2 * sc.N);
  l->statics = a.take((int64_t)Bc * sc.ds);
  l->times = a.take(sc.M2);
  l->lengths = a.take(2LL * Bc);
  l->logits = a.take((int64_t)Bc * sc.ncls);
  l->acc = a.take(2LL * dims->B * (2 * sc.ncls + 1));
  l->total = a.off;
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

// ---- EK-FAC: the factor pass and the rotated rows (DpQueue's kfac modes) ------------------------------------------
namespace {
// Factors: per item, dW = X^T X with db = column sums of X, and dW = dY^T dY (tn: queued for one grouped tensor-core
// launch when the shape fits, else CUDA cores), then each block's sums are added into the fp64 factors (dY carries
// the gradient of l_b / B, so S is scaled by B^2).  Rotated rows: Y^ = dY Q_S and X^ = [X | 1] Q_A on the error-compensated
// tensor-core GEMM (linear_nt, bias = the last row of Q_A), then psg_group on the rotated operands without a ones column.
int kfac_flush(DpQueue& q, cudaStream_t st) {
  if (q.pg.n == 0) return 0;
  const KfacBlocks& K = *q.kb;
  if (q.factors) {
    WgradQueue wq;
    int64_t off = 0;
    float* ws = q.kws;
    const float* Aw[DP_MAX_ITEMS]; const float* Ab[DP_MAX_ITEMS]; const float* Sw[DP_MAX_ITEMS];
    for (int i = 0; i < q.pg.n; ++i) {
      const PsgItem& o = q.pg.it[i];
      const int64_t rows = (int64_t)q.B * o.R;
      float* aw = ws + off; off += round_up((int64_t)o.Kin * o.Kin, 64);
      float* ab = ws + off; off += round_up(o.Kin, 64);
      float* sw = ws + off; off += round_up((int64_t)o.Nout * o.Nout, 64);
      float* sb = ws + off; off += round_up(o.Nout, 64);
      float* pa = ws + off; off += round_up(tc_wgrad_partial_floats(o.Kin, o.Kin, rows), 64);
      float* ps = ws + off; off += round_up(tc_wgrad_partial_floats(o.Nout, o.Nout, rows), 64);
      RD_TRY(tn(&wq, o.X, o.ldx, o.X, o.ldx, aw, ab, o.Kin, o.Kin, rows, pa, q.kpartial, st));
      RD_TRY(tn(&wq, o.Y, o.ldy, o.Y, o.ldy, sw, sb, o.Nout, o.Nout, rows, ps, q.kpartial, st));
      Aw[i] = aw; Ab[i] = ab; Sw[i] = sw;
    }
    RD_TRY(wq.flush(st));
    for (int i = 0; i < q.pg.n; ++i) {
      const PsgItem& o = q.pg.it[i];
      const KfacBlock& b = K.b[q.blk_of[i]];
      RD_TRY(kfac_accumulate(Aw[i], Ab[i], Sw[i], o.Kin, o.Nout, (long long)q.B * o.R, (double)q.B * (double)q.B,
                             q.factors + b.a, q.factors + b.s, st));
    }
    return 0;
  }
  int64_t off = 0;
  for (int i = 0; i < q.pg.n; ++i) {
    PsgItem& o = q.pg.it[i];
    const KfacBlock& b = K.b[q.blk_of[i]];
    const int64_t rows = (int64_t)q.B * o.R;
    float* yh = q.rot + off; off += round_up(rows * o.Nout, 64);
    float* xh = q.rot + off; off += round_up(rows * b.Np, 64);
    RD_TRY(linear_nt(nt(o.Y, o.ldy, q.bases + b.qs, o.Nout, yh, o.Nout, rows, o.Nout, o.Nout), q.bases_lo + b.qs, st));
    GemmP g = nt(o.X, o.ldx, q.bases + b.qa, o.Kin, xh, b.Np, rows, b.Np, o.Kin);
    g.bias = q.bases + b.qb;
    RD_TRY(linear_nt(g, q.bases_lo + b.qa, st));
    o.Y = yh; o.ldy = o.Nout; o.X = xh; o.ldx = b.Np;
  }
  return psg_group(q.pg, q.B, q.G, q.ldg, q.scale, st, true);
}

// Scratch of the factor pass: the backward scratch, then per block the fp32 sums X^T X, x, dY^T dY, dY colsums and two
// tensor-core partial buffers (kfac_flush lays a phase's items out from the start of that region, in queue order), and
// the CUDA-core fallback's split-K partial buffer.
struct KfacLayout { int64_t bw, kws, kpartial, total; };
KfacLayout kfac_layout(const Shape& s) {
  KfacLayout l;
  Arena a;
  l.bw = a.take(bw_layout(s).total);
  const KfacBlocks K = kfac_blocks(s);
  int64_t ws = 0, pf = 0;
  for (int i = 0; i < K.n; ++i) {
    const KfacBlock& b = K.b[i];
    const int64_t rows = i < 4 * s.L ? s.M2 : s.M1;
    ws += round_up((int64_t)b.Kin * b.Kin, 64) + round_up(b.Kin, 64) + round_up((int64_t)b.Nout * b.Nout, 64) +
          round_up(b.Nout, 64) + round_up(tc_wgrad_partial_floats(b.Kin, b.Kin, rows), 64) +
          round_up(tc_wgrad_partial_floats(b.Nout, b.Nout, rows), 64);
    const int64_t p1 = splitk_partial_floats(b.Kin, b.Kin, rows), p2 = splitk_partial_floats(b.Nout, b.Nout, rows);
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
  const KfacBlocks K = kfac_blocks(s);
  l.lo = a.take(K.base_floats);
  int64_t enc = 0, ob = 0;
  for (int i = 0; i < K.n; ++i) {
    const KfacBlock& b = K.b[i];
    const int64_t rows = i < 4 * s.L ? s.M2 : s.M1;
    (i < 4 * s.L ? enc : ob) += round_up(rows * b.Nout, 64) + round_up(rows * b.Np, 64);
  }
  l.rot = a.take(enc > ob ? enc : ob);
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
  if (!encoder_only && (s.dpe != RD_D_PE || s.emb != s.N)) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
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
                        const float* nscale, const float* ws, const float* dlogits, const rd_grads* G, float* sc,
                        int phases, float* d_z0_out, cudaStream_t st, DpQueue* dp = nullptr) {
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if ((phases & ~3) || phases == 0) { set_error("rd_raindrop_v2_bwd: phases must be 1, 2 or 3"); return -2; }
  WsLayout w = ws_layout(s);
  BwLayout b = bw_layout(s);
  const uint64_t* rng = reinterpret_cast<const uint64_t*>(ws + w.rng);
  float* partial = sc + b.partial;
  const float ik = s.p > 0.f ? 1.f / (1.f - s.p) : 1.f;
  float* gA = sc + b.gA; float* gB = sc + b.gB; float* gD = sc + b.gD; float* dP = sc + b.dP;
  WgradQueue wq;     // weight gradients wait here for ONE grouped tensor-core launch per phase
  // G == NULL (frozen parameters): only the data-gradient chain runs -- no weight-gradient GEMMs, column sums or
  // head outer products; the scratch ends up holding the same d(loss)/d(activation) buffers
  const bool wg = G != nullptr;
  static const rd_grads kNoGrads = {};
  if (!wg) G = &kNoGrads;

  if (phases & RD_BWD_ENCODER) {
  // ---- head: logits = mlp2(relu(mlp0(feat))), pooled = masked mean          code/models_rd.py:366-385
  const float* feat = ws + w.feat; const float* hpre = ws + w.hpre;
  float* dfeat = sc + b.dfeat; float* dhpre = sc + b.dhpre;
  RD_TRY(head_bwd(s.B, s.T, s.D, s.emb, s.ds, s.ncls, lengths, statics, P->mlp0_weight, P->mlp2_weight, feat, hpre, dlogits,
                  dhpre, dfeat, gA, G->mlp0_weight, G->mlp0_bias, G->mlp2_weight, G->mlp2_bias, G->emb_weight, G->emb_bias, st));
  if (dp) RD_TRY(dp->head(s, dlogits, hpre, dhpre, feat, dfeat, statics, st));

  const float scale = 1.f / sqrtf((float)s.hd);
  const int64_t row3 = (int64_t)s.B * 3 * s.D;
  const int64_t TT = (int64_t)s.T * s.T;
  for (int l = s.L - 1; l >= 0; --l) {
    const rd_encoder_layer_params& E = P->layer[l];
    const rd_encoder_layer_grads& GE = G->layer[l];
    const int fl = dp ? dp_head_fields(s) + 12 * l : 0;     // this layer's first field (in_proj_weight)
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
    RD_TRY(layernorm_bwd(r2, ws + w.l[l].st2, E.norm2_weight, gA, s.M2, s.D, res, GE.norm2_weight, GE.norm2_bias,
                         sc + b.l[l].ln[0], K2, s.p, rng, SITE_RESID2 + l, &chunks, st, m2, mld));
    if (dp) RD_TRY(dp->ln(r2, ws + w.l[l].st2, gA, s.T, s.D, fl + 10, fl + 11, st));
    if (wg) RD_TRY(wq.colsum(sc + b.l[l].ln[0], 2 * s.D, chunks, s.D, GE.norm2_weight, st));
    if (wg) RD_TRY(wq.colsum(sc + b.l[l].ln[0] + s.D, 2 * s.D, chunks, s.D, GE.norm2_bias, st));
    if (wg) RD_TRY(tn(&wq, K2, s.D, f, s.nhid, GE.linear2_weight, GE.linear2_bias, s.D, s.nhid, s.M2, sc + b.l[l].wp[0], partial, st));
    if (dp) dp->add(K2, s.D, f, s.nhid, s.D, s.nhid, s.T, 1, s.B, fl + 6);
    {   // gF = (K2 . W2) * [f > 0] / (1-p)   ("NT" against W2^T so that the tensor-core kernel applies)
      GemmP g = nt(K2, s.D, ws + w.wsp[l].l2_t, s.D, gF, s.nhid, s.M2, s.nhid, s.D);
      g.gate = f; g.gate_ld = s.nhid; g.gate_scale = ik;  // relu' and the FFN dropout mask in one
      RD_TRY(linear_nt(g, ws + w.wsp[l].l2_tlo, st));
    }
    if (wg) RD_TRY(tn(&wq, gF, s.nhid, x1, s.D, GE.linear1_weight, GE.linear1_bias, s.nhid, s.D, s.M2, sc + b.l[l].wp[1], partial, st));
    if (dp) dp->add(gF, s.nhid, x1, s.D, s.nhid, s.D, s.T, 1, s.B, fl + 4);
    {
      GemmP g = nt(gF, s.nhid, ws + w.wsp[l].l1_t, s.nhid, gA, s.D, s.M2, s.D, s.nhid);
      g.resid = res; g.resid_ld = s.D;
      RD_TRY(linear_nt(g, ws + w.wsp[l].l1_tlo, st));
    }
    // norm1 + self-attention block
    res = s.p > 0.f ? gB : K1;
    RD_TRY(layernorm_bwd(r1, ws + w.l[l].st1, E.norm1_weight, gA, s.M2, s.D, res, GE.norm1_weight, GE.norm1_bias,
                         sc + b.l[l].ln[1], K1, s.p, rng, SITE_RESID1 + l, &chunks, st, m1, mld));
    if (dp) RD_TRY(dp->ln(r1, ws + w.l[l].st1, gA, s.T, s.D, fl + 8, fl + 9, st));
    if (wg) RD_TRY(wq.colsum(sc + b.l[l].ln[1], 2 * s.D, chunks, s.D, GE.norm1_weight, st));
    if (wg) RD_TRY(wq.colsum(sc + b.l[l].ln[1] + s.D, 2 * s.D, chunks, s.D, GE.norm1_bias, st));
    if (wg) RD_TRY(tn(&wq, K1, s.D, ctx, s.D, GE.out_proj_weight, GE.out_proj_bias, s.D, s.D, s.M2, sc + b.l[l].wp[2], partial, st));
    if (dp) dp->add(K1, s.D, ctx, s.D, s.D, s.D, s.T, 1, s.B, fl + 2);
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
    if (wg) RD_TRY(tn(&wq, dqkv, 3 * s.D, x, s.D, GE.in_proj_weight, GE.in_proj_bias, 3 * s.D, s.D, s.M2, sc + b.l[l].wp[3], partial, st));
    if (dp) dp->add(dqkv, 3 * s.D, x, s.D, 3 * s.D, s.D, s.T, 1, s.B, fl);
    {
      // the first layer's input gradient is d(loss)/d(encoder input): optionally delivered straight to the caller
      GemmP g = nt(dqkv, 3 * s.D, ws + w.wsp[l].in_t, 3 * s.D, (l == 0 && d_z0_out) ? d_z0_out : gA, s.D, s.M2, s.D, 3 * s.D);
      g.resid = res; g.resid_ld = s.D;
      RD_TRY(linear_nt(g, ws + w.wsp[l].in_tlo, st));
    }
  }
  if (!(phases & RD_BWD_OBPROP)) RD_TRY(wq.flush(st));   // encoder + head gradients complete: the caller may reduce them now
  if (dp) RD_TRY(dp->flush(st));
  }

  if (phases & RD_BWD_OBPROP) {
  // ---- observation propagation: gA = d(loss)/d(Z0) [T,B,D]          code/models_rd.py:322-343
  float* gO2 = sc + b.gO2; float* gO1 = sc + b.gO1;
  const float* X0 = ws + w.X0; const float* H1 = ws + w.H1;
  const int tc = s.tc;
  RD_TRY(obprop_out_grad(gA, ws + w.Z[0], nscale, s.B, s.T, s.N, s.dob, s.D, tc && !s.exact, gO2, st));
  if (wg) RD_TRY(tn(&wq, gO2, s.C, H1, s.C, G->ob2_value_weight, G->ob2_value_bias, s.C, s.C, s.M1, sc + b.wp_ob[0], partial, st));
  const int fob = dp ? dp_head_fields(s) + 12 * s.L : 0;    // ob1 weight, ob1 bias, ob2 weight, ob2 bias
  if (dp) dp->add(gO2, s.C, H1, s.C, s.C, s.C, s.N, s.N, 1, fob + 2);
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
  if (wg) RD_TRY(tn(&wq, gO1, s.C, X0, s.C, G->ob1_value_weight, G->ob1_value_bias, s.C, s.C, s.M1, sc + b.wp_ob[1], partial, st));
  if (dp) dp->add(gO1, s.C, X0, s.C, s.C, s.C, s.N, s.N, 1, fob);
  RD_TRY(wq.flush(st));
  if (dp) RD_TRY(dp->flush(st));
  }
  return 0;
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
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, grads,
                      (float*)scratch, phases, nullptr, (cudaStream_t)stream);
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
    if (s.tc) {
      const WeightSplit it = {params->ob1_value_weight, s.C, s.C, nullptr, W1t, W1tlo};
      RD_TRY(split_weights(&it, 1, st));
    }
    RD_TRY(input_grad_dx0(s, params, sc + b.gO1, W1t, W1tlo, dX0, st));
  }
  return input_grad(src, params->R_u, dX0, s.B, s.T, s.N, s.dob, s.p, reinterpret_cast<const uint64_t*>(ws + w.rng), d_src,
                    times, sc + b.gA, s.M2, s.D, s.Dm, dims->pe_timescales, s.dpe, lengths, d_times, sc + b.dfeat, s.Df, s.D,
                    params->emb_weight, s.emb, s.ds, d_statics, st);
}

size_t rd_integrated_gradients_scratch_bytes(const rd_dims* dims, int32_t steps_per_chunk) {
  if (!dims) return 0;
  IgcLayout l;
  if (ig_layout(dims, steps_per_chunk, &l) != 0) return 0;
  return (size_t)l.total * sizeof(float);
}

int rd_raindrop_v2_integrated_gradients(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                        const float* times, const int64_t* lengths, const float* node_scale,
                                        const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                        const float* alphas, const float* weights, int32_t n_steps, int32_t steps_per_chunk,
                                        void* scratch, float* attr_src, float* attr_statics, float* endpoint_logits,
                                        void* stream) {
  if (!dims || !params || !src || !times || !lengths || !node_scale || !baseline_src || !alphas || !weights || !scratch ||
      !attr_src || !endpoint_logits || !params->R_u || !params->ob1_value_weight) {
    set_error("rd_raindrop_v2_integrated_gradients: NULL argument");
    return -2;
  }
  if (n_steps < 1 || steps_per_chunk < 1) { set_error("rd_raindrop_v2_integrated_gradients: n_steps and steps_per_chunk must be >= 1"); return -2; }
  if (dims->training) { set_error("rd_raindrop_v2_integrated_gradients: runs eval arithmetic, dims->training must be 0"); return -2; }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.dpe != RD_D_PE || s0.emb != s0.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s0.ds > 0 && (!statics || !baseline_statics)) {
    set_error("rd_raindrop_v2_integrated_gradients: d_static > 0 needs statics and baseline_statics");
    return -2;
  }
  IgcLayout l;
  RD_TRY(ig_layout(dims, steps_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, mc = steps_per_chunk;
  float* S = (float*)scratch;
  float* ws = S + l.ws; float* sc = S + l.sc; float* dX0 = S + l.dX0;
  float* src_e = S + l.src; float* stat_e = s0.ds > 0 ? S + l.statics : nullptr; float* times_e = S + l.times;
  int64_t* len_e = reinterpret_cast<int64_t*>(S + l.lengths);
  float* dlog = S + l.dlogits;
  float* W1t = S + l.W1t; float* W1tlo = S + l.W1tlo;
  float* attr_st = s0.ds > 0 ? attr_statics : nullptr;

  // 1. the endpoints: one forward on 2B rows (baseline rows, then input rows) -> endpoint_logits [2, B, ncls]
  const rd_dims de = ig_dims(dims, 2 * B, mc);
  RD_TRY(ig_expand(src, baseline_src, statics, baseline_statics, times, lengths, nullptr, 2, B, s0.T, s0.N, s0.ds, s0.ncls,
                   nullptr, nullptr, src_e, stat_e, times_e, len_e, nullptr, st));
  RD_TRY(raindrop_fwd(&de, params, src_e, stat_e, times_e, len_e, node_scale, nullptr, ws, endpoint_logits, nullptr, nullptr,
                      nullptr, 0, st));
  // 2. W1^T with its remainder, once per call
  {
    const rd_dims dc = ig_dims(dims, B * mc, mc);
    Shape s;
    RD_TRY(make_shape(&dc, &s));
    if (s.tc) {
      const WeightSplit it = {params->ob1_value_weight, s.C, s.C, nullptr, W1t, W1tlo};
      RD_TRY(split_weights(&it, 1, st));
    }
  }
  // 3. chunks of mc steps (the last one possibly shorter, same scratch, same arithmetic mode)
  for (int c0 = 0; c0 < n_steps; c0 += mc) {
    const int m = n_steps - c0 < mc ? n_steps - c0 : mc;
    const rd_dims dc = ig_dims(dims, B * m, mc);
    Shape s;
    RD_TRY(make_shape(&dc, &s));
    const BwLayout b = bw_layout(s);
    RD_TRY(ig_expand(src, baseline_src, statics, baseline_statics, times, lengths, alphas + c0, m, B, s.T, s.N, s.ds, s.ncls,
                     target, endpoint_logits + (int64_t)B * s.ncls, src_e, stat_e, times_e, len_e, dlog, st));
    RD_TRY(raindrop_fwd(&dc, params, src_e, stat_e, times_e, len_e, node_scale, nullptr, ws, S + l.logits, nullptr, nullptr,
                        nullptr, 0, st));
    RD_TRY(raindrop_bwd(&dc, params, stat_e, len_e, node_scale, ws, dlog, nullptr, sc, RD_BWD_ALL, nullptr, st));
    RD_TRY(input_grad_dx0(s, params, sc + b.gO1, W1t, W1tlo, dX0, st));
    RD_TRY(ig_accumulate(src, baseline_src, alphas + c0, weights + c0, m, B, s.T, s.N, s.dob, params->R_u, dX0, S + l.acc_src,
                         attr_src, statics, baseline_statics, sc + b.dfeat, s.Df, s.D, params->emb_weight, s.emb, s.ds,
                         S + l.acc_static, attr_st, c0 == 0, c0 + m >= n_steps, st));
  }
  return 0;
}

size_t rd_coalition_attribution_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t coalitions_per_chunk) {
  if (!dims) return 0;
  CoalLayout l;
  if (coalition_layout(dims, n_players, coalitions_per_chunk, &l) != 0) return 0;
  return (size_t)l.total * sizeof(float);
}

// What every coalition entry point (Shapley sampling and ablation, KernelSHAP) shares: the argument checks, the scratch
// carved by coalition_layout and the endpoint forward.  `fn` names the caller in error messages.
struct CoalRun {
  Shape s0;
  int P, G, B, cc;
  float* ws; float* logits; float* src_e; float* stat_e; float* times_e; int64_t* len_e; double* acc; uint8_t* keep;
};
static int coalition_setup(const char* fn, const rd_dims* dims, const rd_params* params, const float* src,
                           const float* statics, const float* times, const int64_t* lengths, const float* node_scale,
                           const float* baseline_src, const float* baseline_statics, const int32_t* cell_player,
                           int64_t stride_t, int64_t stride_b, int32_t n_players, int32_t coalitions_per_chunk, void* scratch,
                           const float* attr, const float* endpoint_logits, CoalRun* r) {
  if (!dims || !params || !src || !times || !lengths || !node_scale || !baseline_src || !cell_player || !scratch || !attr ||
      !endpoint_logits || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (dims->training) { set_error("%s: runs eval arithmetic, dims->training must be 0", fn); return -2; }
  Shape& s0 = r->s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.dpe != RD_D_PE || s0.emb != s0.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s0.ds > 0 && (!statics || !baseline_statics)) {
    set_error("%s: d_static > 0 needs statics and baseline_statics", fn);
    return -2;
  }
  const int P = n_players, G = P - (s0.ds > 0 ? 1 : 0);
  if (G < 1) { set_error("%s: n_players = %d gives %d players of the value cells, need >= 1", fn, P, G); return -2; }
  if (stride_t < 0 || stride_b < 0) {
    set_error("%s: player strides must be >= 0, got (%lld, %lld)", fn, (long long)stride_t, (long long)stride_b);
    return -2;
  }
  CoalLayout l;
  RD_TRY(coalition_layout(dims, P, coalitions_per_chunk, &l));
  r->P = P; r->G = G; r->B = s0.B; r->cc = coalitions_per_chunk;
  float* S = (float*)scratch;
  r->ws = S + l.ws; r->logits = S + l.logits;
  r->src_e = S + l.src; r->stat_e = s0.ds > 0 ? S + l.statics : nullptr; r->times_e = S + l.times;
  r->len_e = reinterpret_cast<int64_t*>(S + l.lengths);
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
  const rd_dims de = ig_dims(dims, 2 * r.B, r.cc);
  RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, stride_t, stride_b,
                          nullptr, r.P, r.G, COALITION_ENDPOINTS, 0, 2, r.B, r.s0.T, r.s0.N, r.s0.ds, nullptr, r.src_e,
                          r.stat_e, r.times_e, r.len_e, st));
  return raindrop_fwd(&de, params, r.src_e, r.stat_e, r.times_e, r.len_e, node_scale, nullptr, r.ws, endpoint_logits, nullptr,
                      nullptr, nullptr, 0, st);
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
      const rd_dims dc = ig_dims(dims, B * nc, cc);
      RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, stride_t, stride_b,
                              orders, P, G, method, c0, nc, B, r.s0.T, r.s0.N, r.s0.ds, r.keep, r.src_e, r.stat_e, r.times_e,
                              r.len_e, st));
      RD_TRY(raindrop_fwd(&dc, params, r.src_e, r.stat_e, r.times_e, r.len_e, node_scale, nullptr, r.ws, r.logits, nullptr,
                          nullptr, nullptr, 0, st));
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
      const rd_dims dc = ig_dims(dims, B * nc, cc);
      RD_TRY(coalition_expand(src, baseline_src, statics, baseline_statics, times, lengths, cell_player, player_stride_t,
                              player_stride_b, nullptr, P, G, COALITION_TABLE, (int)c0, nc, B, r.s0.T, r.s0.N, r.s0.ds,
                              const_cast<uint8_t*>(coalitions + c0 * P), r.src_e, r.stat_e, r.times_e, r.len_e, st));
      RD_TRY(raindrop_fwd(&dc, params, r.src_e, r.stat_e, r.times_e, r.len_e, node_scale, nullptr, r.ws, r.logits, nullptr,
                          nullptr, nullptr, 0, st));
    }
    RD_TRY(kernel_shap_accumulate(r.logits, endpoint_logits, target, coalitions, weights, P, (int)c0, nc, B, r.s0.ncls, r.acc,
                                  c0 == 0, st));
    c0 += cc;
  } while (c0 < M);
  // 3. attr = acc . K^T + (F(x) - F(x')) k^T
  return kernel_shap_solve(r.acc, solve, endpoint_logits, target, P, B, r.s0.ncls, attr, st);
}

size_t rd_mc_dropout_scratch_bytes(const rd_dims* dims, int32_t replicates_per_chunk) {
  if (!dims) return 0;
  McLayout l;
  if (mc_layout(dims, replicates_per_chunk, &l) != 0) return 0;
  return (size_t)l.total * sizeof(float);
}

// Chunks of cc replicates: the inputs expanded when the chunk size changes (the first and a ragged last chunk), one
// training forward whose dropout draws replicate m0 + m at step rng[1] + m0 + m (the prologue captures {seed, step + m0},
// rep_remap adds m), and one launch that adds the chunk to the fp64 sums and, after the last chunk, writes the statistics.
int rd_raindrop_v2_mc_dropout(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                              const float* times, const int64_t* lengths, const float* node_scale, const uint64_t* rng,
                              int32_t n_samples, int32_t replicates_per_chunk, void* scratch, float* mean_probs,
                              float* variance, float* entropies, float* samples, void* stream) {
  const char* fn = "rd_raindrop_v2_mc_dropout";
  if (!dims || !params || !src || !times || !lengths || !node_scale || !rng || !scratch || !mean_probs || !variance ||
      !entropies || !params->R_u || !params->ob1_value_weight) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (n_samples < 1 || replicates_per_chunk < 1) { set_error("%s: n_samples and replicates_per_chunk must be >= 1", fn); return -2; }
  Shape s0;
  RD_TRY(make_shape(dims, &s0));
  if (s0.dpe != RD_D_PE || s0.emb != s0.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s0.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  McLayout l;
  RD_TRY(mc_layout(dims, replicates_per_chunk, &l));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s0.B, cc = replicates_per_chunk;
  const int64_t M = n_samples;
  float* S = (float*)scratch;
  float* src_e = S + l.src; float* stat_e = s0.ds > 0 ? S + l.statics : nullptr; float* times_e = S + l.times;
  int64_t* len_e = reinterpret_cast<int64_t*>(S + l.lengths);
  double* acc = reinterpret_cast<double*>(S + l.acc);
  int expanded = 0;
  for (int64_t c0 = 0; c0 < M; c0 += cc) {
    const int nc = (int)(M - c0 < cc ? M - c0 : cc);
    const rd_dims dc = mc_dims(dims, B * nc, cc);
    if (nc != expanded) {
      RD_TRY(mc_expand(src, statics, times, lengths, B, nc, s0.T, s0.N, s0.ds, src_e, stat_e, times_e, len_e, st));
      expanded = nc;
    }
    RD_TRY(raindrop_fwd(&dc, params, src_e, stat_e, times_e, len_e, node_scale, const_cast<uint64_t*>(rng), S + l.ws,
                        S + l.logits, nullptr, nullptr, nullptr, 0, st, B, (uint64_t)c0));
    RD_TRY(mc_accumulate(S + l.logits, nc, B, s0.ncls, c0, M, acc, samples, mean_probs, variance, entropies, c0 == 0,
                         c0 + nc >= M, st));
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
  if (!dims || !params || !lengths || !node_scale || !workspace || !d_logits || !scratch || !sqnorms) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (s.dpe != RD_D_PE || s.emb != s.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  const DpLayout l = dp_layout(s);
  DpQueue q;
  q.B = s.B; q.nf = dp_n_fields(s); q.sqnorms = sqnorms;
  q.partial = reinterpret_cast<double*>((float*)scratch + l.partial);
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, nullptr,
                      (float*)scratch + l.bw, RD_BWD_ALL, nullptr, (cudaStream_t)stream, &q);
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
  if (!dims || !params || !lengths || !node_scale || !workspace || !d_logits || !scratch || !G) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (s.dpe != RD_D_PE || s.emb != s.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  DpQueue q;
  const int64_t bucket = bucket_fields(s, &q.fields);
  if (ldg != bucket) { set_error("%s: ldg = %lld must be the bucket length %lld", fn, (long long)ldg, (long long)bucket); return -2; }
  if (reinterpret_cast<uintptr_t>(G) & 15) { set_error("%s: G must be 16-byte aligned", fn); return -2; }
  q.B = s.B; q.nf = q.fields.n; q.G = G; q.ldg = ldg;
  q.scale = (float)s.B;      // d_logits holds the gradient of l_b / B (the forward's batch mean): rows are of l_b
  cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(psg_pad(q.fields, s.B, G, ldg, st));
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, nullptr, (float*)scratch,
                      RD_BWD_ALL, nullptr, st, &q);
}

int64_t rd_kfac_factors_doubles(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return kfac_blocks(s).factor_doubles;
}

int64_t rd_ekfac_bases_floats(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return kfac_blocks(s).base_floats;
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
  if (!dims || !params || !lengths || !node_scale || !workspace || !d_logits || !scratch || !factors) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (s.dpe != RD_D_PE || s.emb != s.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  if (reinterpret_cast<uintptr_t>(scratch) & 15) { set_error("%s: scratch must be 16-byte aligned", fn); return -2; }
  const KfacBlocks K = kfac_blocks(s);
  const KfacLayout l = kfac_layout(s);
  DpQueue q;
  q.B = s.B; q.shape = &s; q.kb = &K; q.factors = factors;
  q.kws = (float*)scratch + l.kws; q.kpartial = (float*)scratch + l.kpartial;
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, nullptr,
                      (float*)scratch + l.bw, RD_BWD_ALL, nullptr, (cudaStream_t)stream, &q);
}

size_t rd_ekfac_rows_scratch_bytes(const rd_dims* dims) {
  Shape s;
  if (make_shape(dims, &s) != 0) return 0;
  return (size_t)ekfac_layout(s).total * sizeof(float);
}

int rd_raindrop_v2_ekfac_rows(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                              const float* node_scale, const void* workspace, const float* d_logits, const float* bases,
                              void* scratch, float* G, int64_t ldg, void* stream) {
  const char* fn = "rd_raindrop_v2_ekfac_rows";
  if (!dims || !params || !lengths || !node_scale || !workspace || !d_logits || !bases || !scratch || !G) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  Shape s;
  RD_TRY(make_shape(dims, &s));
  if (s.dpe != RD_D_PE || s.emb != s.N) { set_error("Raindrop_v2 has d_pe = 16 and emb_dim = d_inp"); return -2; }
  if (s.ds > 0 && !statics) { set_error("%s: d_static > 0 needs statics", fn); return -2; }
  DpQueue q;
  const int64_t bucket = bucket_fields(s, &q.fields);
  if (ldg != bucket) { set_error("%s: ldg = %lld must be the bucket length %lld", fn, (long long)ldg, (long long)bucket); return -2; }
  if ((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(bases) | reinterpret_cast<uintptr_t>(scratch)) & 15) {
    set_error("%s: G, bases and scratch must be 16-byte aligned", fn);
    return -2;
  }
  const KfacBlocks K = kfac_blocks(s);
  const EkfacLayout l = ekfac_layout(s);
  float* S = (float*)scratch;
  q.B = s.B; q.nf = q.fields.n; q.G = G; q.ldg = ldg;
  q.scale = (float)s.B;      // as rd_raindrop_v2_per_sample_grads: rows are of l_b
  q.shape = &s; q.kb = &K; q.bases = bases; q.bases_lo = S + l.lo; q.rot = S + l.rot;
  cudaStream_t st = (cudaStream_t)stream;
  RD_TRY(grad_lo_image(bases, K.base_floats, S + l.lo, st));
  RD_TRY(psg_pad(q.fields, s.B, G, ldg, st));
  return raindrop_bwd(dims, params, statics, lengths, node_scale, (const float*)workspace, d_logits, nullptr, S + l.bw,
                      RD_BWD_ALL, nullptr, st, &q);
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
  return dp_clip(sqnorms, s.B, dp_n_fields(s), s.ncls, weight, (double)max_grad_norm, (double)expected_batch_size,
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
  return raindrop_bwd(dims, params, statics, lengths, nullptr, (const float*)workspace, d_logits, grads, (float*)scratch,
                      RD_BWD_ENCODER, d_enc_in, (cudaStream_t)stream);
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

}  // extern "C"
