#!/usr/bin/env python
"""Writes Laplace_uncertainty_<name>.npz: a Laplace approximation (raindrop_b200.laplace) fitted on one part of a data
split and evaluated on another, next to Monte Carlo dropout, with the calibration and selective-prediction numbers of
each:

    python tools/laplace_uncertainty.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --name P19
    python tools/laplace_uncertainty.py --synthetic P19

The checkpoint, data, split and normalisation are read as tools/mc_uncertainty.py reads them; labels are required (the
fit needs the training labels).  --synthetic without --checkpoint uses the synthetic weights of that configuration and
synthetic train / eval sets (--n-train, --n-samples).  The fit runs on --fit-part (default train) with --fisher and, by
default, the prior precision that maximises the log marginal likelihood.  On the --part samples it runs, per batch, one
mc_dropout call (--mc-samples, skipped for a model with dropout 0), one laplace_predictive call per link (probit; mc with
--laplace-samples draws) and one deterministic eval forward.

It prints delta, log Z and, per method, the NLL, the Brier score, the 15-bin expected calibration error and the accuracy
at 100 / 90 / 80 / 70 % coverage (coverage_accuracy of tools/mc_uncertainty.py; samples ranked by mutual information
where the method defines it, else by predictive entropy).  The file holds float32 [n, C] probabilities of every method
(mc_dropout_probs, probit_probs, mc_probs, eval_probs), the scores used for the ranking, labels [n] and delta / log Z.

--swag PATH (an SWAG posterior of this model, raindrop_b200.swag.SWAG.save; tools/swag_train.py writes one) adds three
rows: SWA (the eval forward at the posterior's mean weights, ranked by predictive entropy), SWAG (swag_predictive with
--swag-samples weight samples, ranked by mutual information) and, with --multi PATH ..., MultiSWAG over the --swag
posterior and every --multi one (--swag-samples per member).  The file then also holds swa_probs, swag_probs and
multiswag_probs with their scores.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mc_uncertainty import coverage_accuracy  # noqa: E402

ECE_BINS = 15


def calibration(probs, labels):
    """(NLL, Brier score, 15-bin ECE) of probabilities [n, C] against integer labels [n] (float64)."""
    p = np.clip(np.asarray(probs, dtype=np.float64), 1e-12, 1.0)
    n = len(labels)
    nll = float(-np.log(p[np.arange(n), labels]).mean())
    onehot = np.eye(p.shape[1])[labels]
    brier = float(((p - onehot) ** 2).sum(axis=1).mean())
    conf, pred = p.max(axis=1), p.argmax(axis=1)
    bins = np.minimum((conf * ECE_BINS).astype(np.int64), ECE_BINS - 1)
    ece = 0.0
    for k in range(ECE_BINS):
        sel = bins == k
        if sel.any():
            ece += sel.mean() * abs(float(np.mean(pred[sel] == labels[sel])) - float(conf[sel].mean()))
    return nll, brier, float(ece)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict of a trained Raindrop_v2 (torch.save); optional with --synthetic")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2, help="the dropout probability the model was trained with")
    ap.add_argument("--seed", type=int, default=0)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col (required with --data)")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test)")
    ap.add_argument("--fit-part", default="train", choices=["train", "val", "test"])
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-train", type=int, default=4096, help="--synthetic: training samples of the fit")
    ap.add_argument("--n-samples", type=int, default=1024, help="--synthetic: evaluated samples")
    ap.add_argument("--fisher", default="true", choices=["true", "empirical"])
    ap.add_argument("--prior-precision", type=float, default=None, help="default: maximise the log marginal likelihood")
    ap.add_argument("--mc-samples", type=int, default=30, help="Monte Carlo dropout replicates")
    ap.add_argument("--laplace-samples", type=int, default=100, help="draws of the mc link")
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--swag", help="an SWAG posterior of this model (SWAG.save): SWA and SWAG rows")
    ap.add_argument("--multi", nargs="+", default=[], help="further SWAG posteriors (--swag needed): a MultiSWAG row")
    ap.add_argument("--swag-samples", type=int, default=30, help="weight samples per SWAG member")
    ap.add_argument("--name")
    ap.add_argument("--out-dir", default=".")
    args = ap.parse_args()

    from raindrop_b200 import data as RD
    from raindrop_b200.laplace import laplace_fit, laplace_predictive
    from raindrop_b200.synth import make_batch, model_config
    from raindrop_b200.uncertainty import mc_dropout
    if not torch.cuda.is_available():
        raise SystemExit("laplace_uncertainty runs on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    if args.checkpoint:
        from ig_sensor_ranking import model_from_state_dict
        model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                      dropout=args.dropout)
    elif args.synthetic:
        from bench import build_model
        model = build_model(model_config(args.synthetic, dropout=args.dropout), device)
    else:
        raise SystemExit("--data needs --checkpoint")
    model.eval()
    N, T = model.d_inp, model.max_len
    if args.synthetic:
        cfg = model_config(args.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (args.synthetic, N, T))
        tr = make_batch(cfg, args.n_train, seed=args.seed + 1, device=device)
        ev = make_batch(cfg, args.n_samples, seed=args.seed + 2, device=device)
        fit = (tr["src"], tr["static"], tr["times"], tr["y"])
        evl = (ev["src"], ev["static"], ev["times"], ev["y"])
        name = args.name or args.synthetic
    else:
        if not args.outcomes:
            raise SystemExit("--data needs --outcomes: the fit uses the training labels")
        raw = np.load(args.data, allow_pickle=True)
        is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
        P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
        if P_raw.shape[1] != T or P_raw.shape[2] != N:
            raise SystemExit("data [n, T=%d, F=%d] does not match the checkpoint (max_len %d, d_inp %d)"
                             % (P_raw.shape[1], P_raw.shape[2], T, N))
        n = len(P_raw)
        labels_all = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(n, -1)[:, args.label_col].astype(np.int64)
        parts = RD.load_split(args.split) if args.split else (np.arange(n),) * 3
        names = ("train", "val", "test")
        idx_fit, idx = parts[names.index(args.fit_part)], parts[names.index(args.part)]
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[parts[0]]).to(device))

        def tensors(ix):
            st = None if (static is None or not model.static) else static[ix]
            P, Pst, Pt, y = RD.tensorize_normalize(P_raw[ix], minutes[ix], st, labels_all[ix], mf, stdf, device=device)
            return P, Pst, Pt, torch.as_tensor(labels_all[ix], device=device)
        fit, evl = tensors(idx_fit), tensors(idx)
        name = args.name or "dataset"

    P, Pst, Pt, y = fit
    train = dict(src=P, static=Pst, times=Pt, lengths=torch.sum(Pt > 0, dim=0), y=y)
    la = laplace_fit(model, train, fisher=args.fisher, seed=args.seed, prior_precision=args.prior_precision)
    logz = la.log_marginal_likelihood()
    print("fit on %d samples (%s Fisher): delta %.6g, log Z %.6g, P %d, ||theta*||^2 %.6g, train log-likelihood %.6g"
          % (la.n, args.fisher, la.prior_precision, logz, la.n_params, la.theta_sqnorm, la.train_loglik))

    P, Pst, Pt, y = evl
    labels = y.cpu().numpy().astype(np.int64)
    if args.multi and not args.swag:
        raise SystemExit("--multi needs --swag")
    posts = []
    if args.swag:
        from raindrop_b200.swag import SWAG
        posts = [SWAG.load(p_, model) for p_ in [args.swag] + args.multi]
    methods = {"mc_dropout": args.dropout > 0, "probit": True, "mc": True}
    probs = {k: [] for k in methods}
    scores = {k: [] for k in methods}
    evalp = []
    n = P.shape[1]
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        a = (P[:, s:e], None if Pst is None else Pst[s:e], Pt[:, s:e], torch.sum(Pt[:, s:e] > 0, dim=0))
        if methods["mc_dropout"]:
            r = mc_dropout(model, *a, n_samples=args.mc_samples, seed=args.seed, step=0)
            probs["mc_dropout"].append(r.mean_probs.cpu().numpy())
            scores["mc_dropout"].append(r.mutual_information.cpu().numpy())
        r = laplace_predictive(model, la, *a, link="probit")
        probs["probit"].append(r.mean_probs.cpu().numpy())
        scores["probit"].append(r.predictive_entropy.cpu().numpy())
        r = laplace_predictive(model, la, *a, link="mc", n_samples=args.laplace_samples, seed=args.seed)
        probs["mc"].append(r.mean_probs.cpu().numpy())
        scores["mc"].append(r.mutual_information.cpu().numpy())
        with torch.no_grad():
            evalp.append(torch.softmax(model(*a)[0].double(), dim=1).float().cpu().numpy())
    out = {"labels": labels, "eval_probs": np.concatenate(evalp), "prior_precision": np.float64(la.prior_precision),
           "log_marginal_likelihood": np.float64(logz)}
    for k, on in methods.items():
        if on:
            out[k + "_probs"] = np.concatenate(probs[k])
            out[k + "_score"] = np.concatenate(scores[k])
    swag_rows = []
    if posts:
        from raindrop_b200.swag import swag_predictive
        swag_methods = {"swag": [posts[0]]}
        if len(posts) > 1:
            swag_methods["multiswag"] = posts
        res = {k: ([], []) for k in ["swa"] + list(swag_methods)}
        saved = [p_.detach().clone() for p_ in model.used_parameters()]
        posts[0].load_mean(model)
        for s in range(0, n, args.batch_size):
            e = min(n, s + args.batch_size)
            a = (P[:, s:e], None if Pst is None else Pst[s:e], Pt[:, s:e], torch.sum(Pt[:, s:e] > 0, dim=0))
            with torch.no_grad():
                p_swa = torch.softmax(model(*a)[0].double(), dim=1)
            res["swa"][0].append(p_swa.float().cpu().numpy())
            res["swa"][1].append((-(p_swa * torch.log(p_swa.clamp_min(1e-300))).sum(1)).float().cpu().numpy())
        with torch.no_grad():
            for p_, s_ in zip(model.used_parameters(), saved):
                p_.copy_(s_)
        for s in range(0, n, args.batch_size):
            e = min(n, s + args.batch_size)
            a = (P[:, s:e], None if Pst is None else Pst[s:e], Pt[:, s:e], torch.sum(Pt[:, s:e] > 0, dim=0))
            for k, members in swag_methods.items():
                r = swag_predictive(model, members, *a, n_samples=args.swag_samples, seed=args.seed)
                res[k][0].append(r.mean_probs.cpu().numpy())
                res[k][1].append(r.mutual_information.cpu().numpy())
        labels_of = {"swa": "SWA (entropy)", "swag": "SWAG (M=%d, MI)" % args.swag_samples,
                     "multiswag": "MultiSWAG (%d x %d, MI)" % (len(posts), args.swag_samples)}
        for k, (pp, sc) in res.items():
            out[k + "_probs"], out[k + "_score"] = np.concatenate(pp), np.concatenate(sc)
            swag_rows.append((labels_of[k], out[k + "_probs"], out[k + "_score"]))
    path = os.path.join(args.out_dir, "Laplace_uncertainty_%s.npz" % name)
    np.savez(path, **out)
    print("wrote %s: %d samples" % (path, n))
    rows = [("eval forward", out["eval_probs"], None)] + \
        [({"mc_dropout": "MC dropout (M=%d, MI)" % args.mc_samples, "probit": "Laplace probit (entropy)",
           "mc": "Laplace mc (M=%d, MI)" % args.laplace_samples}[k], out[k + "_probs"], out[k + "_score"])
         for k, on in methods.items() if on] + swag_rows
    print("%-28s %8s %8s %8s   accuracy at coverage 100 / 90 / 80 / 70 %%" % ("method", "NLL", "Brier", "ECE"))
    for label, p, score in rows:
        nll, brier, ece = calibration(p, labels)
        pred = p.argmax(axis=1)
        acc = coverage_accuracy(pred, labels, score if score is not None else -p.max(axis=1))
        print("%-28s %8.4f %8.4f %8.4f   %s" % (label, nll, brier, ece, " ".join("%.4f" % v for v in acc.values())))


if __name__ == "__main__":
    main()
