"""Times TracIn (raindrop_b200.influence.tracin) on one GPU: one checkpoint, n_query queries against a DeviceDataset of
n_train synthetic samples.  Prints one JSON line per shape: seconds per checkpoint, train samples/s, the split of the
time (rows = forward + data-gradient backward + materialisation, the forward alone, dot = remainder image + wgmma dot +
reduce), the dot kernel's achieved bytes/s and TFLOP/s against the H100 SXM data sheet (3.35 TB/s, 495 TFLOP/s TF32
dense; 3xTF32 issues three TF32 products per fp32 product), the share of the row kernels' time spent in the
materialisation kernels (torch.profiler over the first four train chunks, applied to the rows time as an estimate), the
paper bound of writing each train row once and reading it once per query block, and the loop of one-sample module backwards timed on
`--loop` samples and extrapolated to n_train.  The card's name and power limit are printed with the numbers.

    python tools/bench_tracin.py --shape P19 --n-query 128 --n-train 31000

--projection DIM times TracIn-RP instead (influence.project / tracin_sketch): the train set's sketch, split into rows
and the projection launches (CUDA events, in project's chunk plan), the projection kernel's TF32 rate counting both
passes (2 x 2 x rows x columns x dim) against the 495 TFLOP/s data sheet, the query sketch and scoring times, and the
whole-set exact time, extrapolated from tracin timed on --exact-train training samples (labelled as extrapolated).

    python tools/bench_tracin.py --shape PAM --n-query 533 --n-train 4266 --projection 4096

--ekfac times EK-FAC influence functions instead (influence.ekfac_*): the factor pass (kfac_covariances), the host
eigendecompositions and the Lambda pass (the rest of ekfac_factors), and the scoring of n_query queries against
--exact-train training samples next to tracin on the same samples, both extrapolated linearly to n_train (labelled as
extrapolated).  The rotations' cost is the difference between the rotated and the plain row passes over those samples.

    python tools/bench_tracin.py --shape P19 --n-query 3880 --n-train 31000 --ekfac

--trak times TRAK instead (influence.trak_features / trak, one model): the margin rows plus their projection, the fp64
Gram kernel (rd_trak_gram), torch.linalg.eigh in float64, the rotation kernel (rd_trak_rotate) and the scoring of
n_query queries, each on its own.  On the same Phi it times the cuBLAS DGEMM Phi.double().T @ Phi.double(), with and
without the conversion, and reports the FP64 TFLOP/s of both (2 n dim^2 for the full product, the Gram kernel's
issued triangle tiles apart) with the card's name and power limit.

    python tools/bench_tracin.py --shape P19 --n-query 128 --n-train 31000 --trak --projection 4096
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from helpers import build_dropin, to_dev  # noqa: E402
from raindrop_b200 import influence as IF  # noqa: E402
from raindrop_b200 import lib as L  # noqa: E402
from raindrop_b200.data import BatchBuffers, DeviceDataset  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


PSG_KERNELS = ("psg_tile_kernel", "psg_ln_kernel", "psg_head_kernel", "psg_pad_kernel")


def materialisation_share(model, ds, idx, tc, R, ldg, n):
    """Share of the row computation's GPU kernel time spent in the materialisation kernels (psg_tile / ln / head / pad),
    from a torch.profiler run (CUDA activity) over the rows of the first n train samples, in tracin's chunks."""
    from torch.profiler import ProfilerActivity, profile
    st_w = 0 if ds.Pstatic is None else ds.Pstatic.shape[1]

    def fetch(a, b):
        buf = BatchBuffers(ds.T, b - a, ds.width, st_w)
        ds.fill(buf, idx[a:b])
        return buf.src, buf.static, buf.times, buf.lengths, buf.y
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t0 in range(0, n, tc):
            IF._rows_aligned(model, fetch, t0, min(n, t0 + tc), R, ldg)
        torch.cuda.synchronize()
    mat = tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if t <= 0 or "Memcpy" in e.key or "Memset" in e.key:
            continue
        tot += t
        if any(k in e.key for k in PSG_KERNELS):
            mat += t
    return mat / tot if tot else float("nan")


def run(shape, nq, nt, loop_n):
    cfg = model_config(shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=1))
    dt = make_batch(cfg, nt, seed=2)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    IF.tracin(model, q, (ds, torch.arange(min(nt, 64))))          # warm-up: modules, tensor maps, allocator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    S = IF.tracin(model, q, ds)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0

    # the split, with CUDA events, over the same chunk plan
    lib, plan = L.load(), model._plan
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    off, ln = IF.plan_segments(layout)
    n_seg = len(off)
    offs, lens = (C.c_int64 * n_seg)(*off.tolist()), (C.c_int64 * n_seg)(*ln.tolist())
    qb, tc, R = IF._blocks(lib, plan, ldg, n_seg, nq, nt, None)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t_rows = t_fwd = t_dot = 0.0
    scores = torch.zeros(nq, nt, dtype=torch.float64, device="cuda")
    idx = torch.arange(nt, device="cuda")
    with torch.no_grad():
        for q0 in range(0, nq, qb):
            q1 = min(nq, q0 + qb)
            qf = lambda a, b: (dq["src"][:, a:b], None if dq["static"] is None else dq["static"][a:b], dq["times"][:, a:b],
                               dq["lengths"][a:b], None)
            Gq = IF._rows_aligned(model, qf, q0, q1, R, ldg)
            for t0_ in range(0, nt, tc):
                t1_ = min(nt, t0_ + tc)
                bufs = []
                for s0 in range(t0_, t1_, R):
                    buf = BatchBuffers(ds.T, min(t1_, s0 + R) - s0, ds.width, 0 if ds.Pstatic is None else ds.Pstatic.shape[1])
                    ds.fill(buf, idx[s0:s0 + buf.src.shape[1]])
                    bufs.append(buf)
                tf = lambda a, b: (lambda bb: (bb.src, bb.static, bb.times, bb.lengths, bb.y))(bufs[(a - t0_) // R])
                e = [ev() for _ in range(6)]
                e[0].record()
                for buf in bufs:
                    model.forward(buf.src, buf.static, buf.times, buf.lengths)
                e[1].record()
                Gt = IF._rows_aligned(model, tf, t0_, t1_, R, ldg)
                e[2].record()
                nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1_ - t0_, ldg, n_seg)
                sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device="cuda")
                e[3].record()
                L.check(lib.rd_per_sample_grad_dot(Gq.data_ptr(), q1 - q0, Gt.data_ptr(), t1_ - t0_, ldg, offs, lens, n_seg,
                                                   1.0, scores.data_ptr() + 8 * (q0 * nt + t0_), nt, sc.data_ptr(),
                                                   L.stream_ptr()), "dot")
                e[4].record()
                torch.cuda.synchronize()
                t_fwd += e[0].elapsed_time(e[1]) / 1e3
                t_rows += e[1].elapsed_time(e[2]) / 1e3
                t_dot += e[3].elapsed_time(e[4]) / 1e3
                del Gt, sc
    assert torch.equal(scores, S), "the split run must reproduce tracin bitwise"
    # the materialisation apart from forward and backward: kernel times of a profiled run over the first train chunks
    mat_share = materialisation_share(model, ds, idx, tc, R, ldg, min(nt, 4 * tc))
    K = int(ln.sum())
    dot_bytes = 4 * nt * K * ((nq + qb - 1) // qb) + 4 * 2 * nq * K * ((nt + tc - 1) // tc)   # Gt per query block; Gq, Gq_lo per chunk
    dot_flop = 2.0 * nq * nt * K
    # the loop a user would write without this: one-sample module backwards, timed on loop_n samples
    dl = to_dev(make_batch(cfg, loop_n, seed=3))
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(loop_n):
        sl = slice(b, b + 1)
        logits, _, _ = model.forward(dl["src"][:, sl], None if dl["static"] is None else dl["static"][sl],
                                     dl["times"][:, sl], dl["lengths"][sl])
        g = torch.autograd.grad(F.cross_entropy(logits, dl["y"][sl]), model.used_parameters())
        torch.cat([x.reshape(-1) for x in g])
    torch.cuda.synchronize()
    loop = (time.perf_counter() - t0) / loop_n * (nt + nq)
    return dict(shape=shape, card=card(), n_query=nq, n_train=nt, bucket=ldg, query_block=qb, train_chunk=tc,
                seconds_per_checkpoint=total, train_samples_per_s=nt / total,
                split_s=dict(forward_only=t_fwd, rows=t_rows, dot=t_dot),
                dot_bytes_per_s=dot_bytes / t_dot, dot_hbm_fraction=dot_bytes / t_dot / 3.35e12,
                dot_tflops_fp32_products=dot_flop / t_dot / 1e12,
                dot_tf32_fraction=3 * dot_flop / t_dot / 495e12,
                materialisation_share_of_row_kernels=mat_share, materialisation_s_estimated=mat_share * t_rows,
                paper_bound_s_per_train_sample=8 * ldg / 3.35e12, measured_s_per_train_sample=total / nt,
                one_sample_loop_s_extrapolated=loop, loop_samples_timed=loop_n)


def run_projection(shape, nq, nt, dim, exact_nt):
    cfg = model_config(shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=1))
    dt = make_batch(cfg, nt, seed=2)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    IF.tracin_sketch(IF.project(model, q, dim=dim), IF.project(model, (ds, torch.arange(min(nt, 64))), dim=dim))  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = IF.project(model, ds, dim=dim)
    torch.cuda.synchronize()
    t_train = time.perf_counter() - t0
    t0 = time.perf_counter()
    sq = IF.project(model, q, dim=dim)
    torch.cuda.synchronize()
    t_query = time.perf_counter() - t0
    t0 = time.perf_counter()
    S = IF.tracin_sketch(sq, st)
    torch.cuda.synchronize()
    t_score = time.perf_counter() - t0

    # the split of the train sketch, with CUDA events, over project's chunk plan
    lib, plan = L.load(), model._plan
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    off, ln = IF.plan_segments(layout)
    n_seg = len(off)
    offs, lens = (C.c_int64 * n_seg)(*off.tolist()), (C.c_int64 * n_seg)(*ln.tolist())
    R = IF._row_batch(lib, plan, ldg)
    chunk = max(R, IF._largest_chunk(lambda b: 4 * b * ldg + IF._rows_bytes(lib, plan, min(b, R), ldg) +
                                     lib.rd_grad_projection_scratch_bytes(b, ldg, dim, n_seg), nt) // R * R)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    feats = torch.empty(nt, dim, dtype=torch.float32, device="cuda")
    idx = torch.arange(nt, device="cuda")
    st_w = 0 if ds.Pstatic is None else ds.Pstatic.shape[1]

    def fetch(a, b):
        buf = BatchBuffers(ds.T, b - a, ds.width, st_w)
        ds.fill(buf, idx[a:b])
        return buf.src, buf.static, buf.times, buf.lengths, buf.y
    t_rows = t_proj = 0.0
    with torch.no_grad():
        for i0 in range(0, nt, chunk):
            i1 = min(nt, i0 + chunk)
            e = [ev() for _ in range(3)]
            e[0].record()
            G = IF._rows_aligned(model, fetch, i0, i1, R, ldg)
            nb = lib.rd_grad_projection_scratch_bytes(i1 - i0, ldg, dim, n_seg)
            sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device="cuda")
            e[1].record()
            L.check(lib.rd_grad_projection(G.data_ptr(), i1 - i0, ldg, offs, lens, n_seg, dim, 0, feats[i0:i1].data_ptr(),
                                           dim, sc.data_ptr(), L.stream_ptr()), "rd_grad_projection")
            e[2].record()
            torch.cuda.synchronize()
            t_rows += e[0].elapsed_time(e[1]) / 1e3
            t_proj += e[1].elapsed_time(e[2]) / 1e3
            del G, sc
    assert torch.equal(feats, st.features[0]), "the split run must reproduce project bitwise"
    K = int(ln.sum())
    proj_flop = 2 * 2.0 * nt * K * dim           # two TF32 passes (Omega.G_lo, Omega.G_hi)
    # exact TracIn on a subset of the train set, extrapolated linearly in n_train
    ne = min(nt, exact_nt)
    IF.tracin(model, q, (ds, torch.arange(min(ne, 64))))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    IF.tracin(model, q, (ds, torch.arange(ne)))
    torch.cuda.synchronize()
    t_exact = (time.perf_counter() - t0) * nt / ne
    return dict(shape=shape, card=card(), projection_dim=dim, n_query=nq, n_train=nt, bucket=ldg, chunk=chunk,
                train_sketch_s=t_train, train_sketch_split_s=dict(rows=t_rows, projection=t_proj),
                projection_tflops_tf32=proj_flop / t_proj / 1e12, projection_tf32_fraction=proj_flop / t_proj / 495e12,
                query_sketch_s=t_query, scoring_s=t_score, scores_finite=bool(torch.isfinite(S).all()),
                sketch_total_s=t_train + t_query + t_score, exact_timed_train_samples=ne,
                exact_s_extrapolated=t_exact, sketch_bytes=4 * (nt + nq) * dim)


def run_ekfac(shape, nq, nt, exact_nt):
    cfg = model_config(shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=1))
    dt = make_batch(cfg, nt, seed=2)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    warm = (ds, torch.arange(min(nt, 64)))
    IF.ekfac_influence(model, q, warm, IF.ekfac_factors(model, warm))                                    # warm-up

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0
    _, t_cov = timed(lambda: IF.kfac_covariances(model, ds))
    f, t_all = timed(lambda: IF.ekfac_factors(model, ds))
    ne = min(nt, exact_nt)
    sub = (ds, torch.arange(ne))
    S, t_score = timed(lambda: IF.ekfac_influence(model, q, sub, f))
    _, t_exact = timed(lambda: IF.tracin(model, q, sub))
    # rotated against plain rows over the same samples, in the same row batches
    lib, plan = L.load(), model._plan
    ldg = IF._bucket_length(IF.grad_layout(model))
    R = IF._row_batch(lib, plan, ldg)
    _, fetch = IF._source(sub, "train")
    bases = f.bases_flat.cuda()
    with torch.no_grad():
        _, t_plain = timed(lambda: [IF._rows_aligned(model, fetch, i, min(ne, i + R), R, ldg) for i in range(0, ne, R)])
        _, t_rot = timed(lambda: [IF._ekfac_rows_aligned(model, fetch, i, min(ne, i + R), R, ldg, bases)
                                  for i in range(0, ne, R)])
    scale = nt / ne
    return dict(shape=shape, card=card(), n_query=nq, n_train=nt, bucket=ldg, row_batch=R,
                factor_pass_s=t_cov, eigh_and_lambda_pass_s=t_all - t_cov, factors_total_s=t_all,
                scored_train_samples=ne, ekfac_scoring_s_extrapolated=t_score * scale,
                tracin_s_extrapolated=t_exact * scale, scoring_ratio=t_score / t_exact,
                rows_plain_s=t_plain, rows_rotated_s=t_rot, rotation_share_of_rows=(t_rot - t_plain) / t_rot,
                scores_finite=bool(torch.isfinite(S).all()))


def run_trak(shape, nq, nt, dim, reps=5):
    cfg = model_config(shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=1))
    dt = make_batch(cfg, nt, seed=2)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    warm = (ds, torch.arange(min(nt, 256)))
    IF.trak(model, q, IF.trak_features(model, warm, dim=dim), damping=1e-3)                              # warm-up

    def timed(fn, n=1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            out = fn()
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) / n
    lib, plan = L.load(), model._plan
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    seg = IF._segments(*IF.plan_segments(layout))
    R = IF._row_batch(lib, plan, ldg)
    chunk = IF._trak_chunk(lib, plan, ldg, dim, seg[2], nt, R, None)
    n, fetch = IF._source(ds, "train")
    with torch.no_grad():
        (Phi, Q), t_rows = timed(lambda: IF._trak_sketch(model, fetch, n, dim, 0, seg, chunk, R, ldg))
    IF._trak_gram(Phi)
    K, t_gram = timed(lambda: IF._trak_gram(Phi), reps)
    (lam, V), t_eigh = timed(lambda: IF._trak_eigh(K))
    Pr, t_rot = timed(lambda: IF._trak_rotate(Phi, V), reps)
    Pd = Phi.double()
    Kd, t_dgemm = timed(lambda: Pd.T @ Pd, reps)
    _, t_dgemm_conv = timed(lambda: Phi.double().T @ Phi.double(), reps)
    gram_err = ((K - Kd).norm() / Kd.norm()).item()
    del Pd, Kd
    feats, t_features = timed(lambda: IF.trak_features(model, ds, dim=dim))
    assert torch.equal(feats.features[0], Pr) and torch.equal(feats.eigenvalues[0], lam), \
        "the split run must reproduce trak_features bitwise"
    S, t_score = timed(lambda: IF.trak(model, q, feats))
    T = dim // 64
    full = 2.0 * nt * dim * dim
    issued = 2.0 * (-(-nt // 32) * 32) * 64 * 64 * T * (T + 1) // 2
    return dict(shape=shape, card=card(), projection_dim=dim, n_query=nq, n_train=nt, bucket=ldg, chunk=chunk,
                margin_rows_and_projection_s=t_rows, gram_s=t_gram, eigh_s=t_eigh, rotation_s=t_rot,
                scoring_s=t_score, trak_features_total_s=t_features,
                gram_fp64_tflops_full_product=full / t_gram / 1e12, gram_fp64_tflops_issued=issued / t_gram / 1e12,
                dgemm_s=t_dgemm, dgemm_fp64_tflops=full / t_dgemm / 1e12, dgemm_with_conversion_s=t_dgemm_conv,
                gram_vs_dgemm_rel_diff=gram_err, dgemm_faster=t_dgemm < t_gram,
                rotation_fp64_tflops=full / t_rot / 1e12, scores_finite=bool(torch.isfinite(S).all()),
                rank=int((IF.trak_weights(lam) > 0).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="P19")
    ap.add_argument("--n-query", type=int, default=128)
    ap.add_argument("--n-train", type=int, default=31000)
    ap.add_argument("--loop", type=int, default=64)
    ap.add_argument("--projection", type=int, help="time TracIn-RP with this many projection dimensions")
    ap.add_argument("--exact-train", type=int, default=1024,
                    help="--projection, --ekfac: train samples of the timed exact (and EK-FAC) scoring calls")
    ap.add_argument("--ekfac", action="store_true", help="time EK-FAC influence functions")
    ap.add_argument("--trak", action="store_true", help="time TRAK (--projection DIM, default 4096)")
    a = ap.parse_args()
    if a.trak:
        print(json.dumps(run_trak(a.shape, a.n_query, a.n_train, a.projection or 4096)), flush=True)
        return
    if a.ekfac:
        print(json.dumps(run_ekfac(a.shape, a.n_query, a.n_train, a.exact_train)), flush=True)
        return
    if a.projection:
        print(json.dumps(run_projection(a.shape, a.n_query, a.n_train, a.projection, a.exact_train)), flush=True)
        return
    print(json.dumps(run(a.shape, a.n_query, a.n_train, a.loop)), flush=True)


if __name__ == "__main__":
    main()
