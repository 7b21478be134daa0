"""The graph operators on seeded random graphs against the float64 oracles, forward and backward:
`TransformerConv` (rd_tconv.cu), `Observation_progation(use_beta=True)` (rd_obprop_beta.cu), `rd_node_scale` and the
`use_beta=False` module path, the autograd wrappers of raindrop_b200/functional.py around them, and legacy `Raindrop` v1.

The references are `TransformerConvOracle` / `ObPropOracle` of oracle/raindrop_oracle.py in float64 with float64
autograd.  tests/test_oracle_golden.py pins them to the reference's own layers on one 6-node fixture; the CPU tests at
the end of this file check them on the graphs used here against central finite differences.  Nothing here reads the
reference tree.

The two discontinuities of `use_beta=True` are handled when a case is built (`beta_case`), never by skipping: a case
whose float64 scores are closer than 1e-4 (relative) around the top-E//2 cut, or between neighbours of the kept order
where that order is compared exactly, and a case with a `lin_value` pre-activation within 1e-5 of zero, is rejected and
the next seed is taken.  So no assertion depends on how fp32 breaks a near-tie or on the sign of a rounding error.

What reaches which part of the kernels (E edges, F out_channels, H heads, C = 4 T channels, rows = n_nodes * n_graphs):
  second trip of the `e += 32` / `f += 32` warp loops of rd_tconv.cu   test_tconv: every graph with E > 32 (all but the
                                                                       tiny ones), F = 33, 64, 130
  second trip of `c += blockDim.x` (128 threads over H*F)              test_tconv: (36, 1, 130), (100, 8, 32), (20, 4, 64)
  second trip of the 256-thread channel loops of rd_obprop_beta.cu     test_obprop_beta: T = 70 (C = 280)
  split-K weight gradients with the fused bias sum                     test_tconv with N = 100, 200; test_tconv_batched
    (gemm_splitk_plan: nsplit = min(ceil(264 / tiles), ceil(rows / 64)),  with rows = 320 .. 23220 (nsplit 5 .. 132);
     so rows >= 65 splits while the weight has few 64 x 64 tiles)        test_obprop_beta with N = 100 (nsplit 2)
  `back(accumulate=true)` over more than one 64 x 64 tile              test_tconv with N >= 100 or in_ch = 100; batched
  E == 0, d_x / d_edge_w / d_alpha / d_p_t == NULL                     test_tconv[none-*], test_tconv_optional_gradients,
                                                                       test_obprop_beta (its `needs` parameter)
  nodes without incoming / outgoing edges, self loops, duplicates,     the `isolated`, `dense`, `dup`, `star_in`,
    a target collecting >= 70 edges                                    `star_out` patterns of `make_graph`
  softmax stability                                                    weights scaled by 60 (`x60`)
  heads > 2; edge weights together with heads > 1                      (64, 3, 33), (100, 8, 32), (20, 4, 64) with `w`
  graph-major geometry                                                 test_tconv_batched[*-graph_major]
  rank_and_prune with odd E, E = 2, 3, negative weights, a source      test_obprop_beta, test_obprop_beta_pruned_source,
    that keeps no edge, exact ties                                     test_obprop_beta_tie_rule
  rd_*_scratch_bytes against what the kernels write                    test_scratch_sizes_*
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import normwise, to_dev
from oracle.raindrop_oracle import ObPropOracle, TransformerConvOracle, node_scale_from_graph, round_tf32
from raindrop_b200 import functional as RF
from raindrop_b200.lib import RaindropB200Error

gpu = pytest.mark.gpu

# Bounds: about 5x the worst normwise error seen over this file on an H100 80GB HBM3 (700 W limit), which `report` prints
# per class: TransformerConv forward 3.3e-6 and gradients 8.5e-7, use_beta forward 8.1e-7 and gradients 2.3e-6,
# use_beta=False forward 7.5e-7 and gradients 4.6e-7, node_scale 2.4e-7 (absolute, on values of 1).
FWD_TOL = 2e-5
GRAD_TOL = 5e-6
BETA_FWD_TOL = 5e-6
BETA_GRAD_TOL = 1e-5
WORST = {}


def hold(cls, err, tol, what):
    WORST[cls] = max(WORST.get(cls, 0.0), err)
    assert err < tol, "%s: %s error %.3e >= %.1e" % (what, cls, err, tol)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k in sorted(WORST):
        print("worst %-22s %.3e" % (k, WORST[k]))


# ---- 1. seeded random graphs --------------------------------------------------------------------------------------
NODE_COUNTS = (1, 2, 6, 17, 36, 100, 200)
PATTERNS = ("er10", "er30", "er70", "dense", "star_in", "star_out", "dup", "isolated", "none", "one", "odd")
WEIGHTS = ("uniform", "normal", "x60")


def make_graph(pattern, N, seed, weights="uniform"):
    """edge_index [2, E] int64 (row 0 = source, row 1 = target) and weights [E] float32 of a named pattern on N nodes.
    Every pattern but `dense` (which keeps the row-major order the models produce) shuffles its edge order."""
    g = torch.Generator().manual_seed(seed * 7919 + N)
    er = lambda p: torch.nonzero(torch.rand(N, N, generator=g) < p).T
    if pattern.startswith("er"):
        ei = er(int(pattern[2:]) / 100.0)
    elif pattern == "dense":                                   # all N^2 pairs, self loops included
        ei = torch.nonzero(torch.ones(N, N)).T
    elif pattern in ("star_in", "star_out"):                   # one node collecting >= 70 edges (duplicates when N < 70)
        hub = N // 2
        spokes = torch.arange(max(N, 70)) % N
        ei = torch.cat([torch.stack([spokes, torch.full_like(spokes, hub)]), er(0.05)], 1)
        if pattern == "star_out":
            ei = ei.flip(0)
    elif pattern == "dup":                                     # every edge of the first half listed twice
        ei = er(0.3)
        ei = torch.cat([ei, ei[:, : ei.shape[1] // 2 + 1]], 1)
    elif pattern == "isolated":                                # thirds of the nodes: no edge / only outgoing / only incoming
        ei = er(0.5)
        role = torch.arange(N) % 4                             # 0: ordinary, 1: isolated, 2: only outgoing, 3: only incoming
        s, t = role[ei[0]], role[ei[1]]
        ei = ei[:, (s != 1) & (t != 1) & (t != 2) & (s != 3)]
    elif pattern == "none":
        ei = torch.zeros(2, 0, dtype=torch.int64)
    elif pattern == "one":
        ei = torch.tensor([[N - 1], [0]])
    elif pattern == "odd":                                     # E = 17 mod 32 where the graph has that many pairs
        ei = er(0.6)
        ei = ei[:, : max(1, ei.shape[1] - (ei.shape[1] - 17) % 32)]
    else:
        raise KeyError(pattern)
    ei = ei.to(torch.int64).contiguous()
    E = ei.shape[1]
    if pattern != "dense":
        ei = ei[:, torch.randperm(E, generator=g)].contiguous()
    w = {"uniform": lambda: torch.rand(E, generator=g), "normal": lambda: torch.randn(E, generator=g),
         "x60": lambda: torch.rand(E, generator=g) * 60}[weights]()
    return ei, w.float()


def test_graph_generator_patterns():
    for N in NODE_COUNTS:
        for pat in PATTERNS:
            ei, w = make_graph(pat, N, 1)
            assert ei.dtype == torch.int64 and ei.shape[0] == 2 and w.shape == (ei.shape[1],)
            assert ei.numel() == 0 or (int(ei.min()) >= 0 and int(ei.max()) < N)
            assert torch.equal(ei, make_graph(pat, N, 1)[0])
    deg = lambda ei, row, N: torch.bincount(ei[row], minlength=N)
    assert int(deg(make_graph("star_in", 100, 1)[0], 1, 100).max()) >= 70
    assert int(deg(make_graph("star_out", 6, 1)[0], 0, 6).max()) >= 70
    assert make_graph("dense", 17, 1)[0].shape[1] == 17 * 17 and make_graph("none", 6, 1)[0].shape[1] == 0
    assert make_graph("odd", 36, 1)[0].shape[1] % 32 == 17 and make_graph("one", 6, 1)[0].shape[1] == 1
    ei = make_graph("isolated", 36, 1)[0]
    din, dout = deg(ei, 1, 36), deg(ei, 0, 36)
    role = torch.arange(36) % 4
    assert int((din + dout)[role == 1].sum()) == 0 and int(din[role == 2].sum()) == 0 and int(dout[role == 3].sum()) == 0
    assert int(dout[role == 2].sum()) > 0 and int(din[role == 3].sum()) > 0
    ei = make_graph("dup", 17, 1)[0]
    assert len({(int(a), int(b)) for a, b in ei.T}) < ei.shape[1]
    assert float(make_graph("er30", 36, 1, "normal")[1].min()) < 0 and float(make_graph("er30", 36, 1, "x60")[1].max()) > 30


# ---- 2. TransformerConv ---------------------------------------------------------------------------------------------
TCONV_KEYS = ("lin_query", "lin_key", "lin_value", "lin_skip")


def tconv_oracle(in_ch, H, Fo, seed):
    torch.manual_seed(seed)
    return TransformerConvOracle(in_ch, Fo, H)


def tconv_reference(orc, x, ei, ew, G, x_grad=True):
    """float64 forward and autograd of the oracle under loss = sum(out * G).  Returns out, alpha, the gradients by
    name and the natural scale of d_edge_w, max |alpha * d loss / d alpha| (a saturated softmax leaves d_edge_w itself
    far below it)."""
    orc = orc.double()
    orc.zero_grad()
    xd = x.detach().double().clone().requires_grad_(x_grad)
    wd = None if ew is None else ew.double().requires_grad_(True)
    out, alpha = orc(xd, ei, wd)
    alpha.retain_grad()
    (out * G.double()).sum().backward()
    grads = {k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in orc.named_parameters()}
    grads["x"] = xd.grad
    if wd is not None:
        grads["edge_w"] = wd.grad if wd.grad is not None else torch.zeros_like(wd)
        grads["edge_w.scale"] = float((alpha.detach() * alpha.grad).abs().max()) if alpha.numel() else 0.0
    return out.detach(), alpha.detach(), grads


def tconv_gpu(orc, x, ei, ew, G, via, geom=None, x_grad=True, w_grad=True):
    """The same through `models_rd.TransformerConv` (via='module') or `functional.transformer_conv`."""
    from raindrop_b200.models_rd import TransformerConv
    H, Fo = orc.heads, orc.out_channels
    conv = TransformerConv(x.shape[1], Fo, heads=H)
    conv.load_state_dict({k: v.float() for k, v in orc.state_dict().items()})
    conv = conv.cuda()
    xg = x.cuda().requires_grad_(x_grad)
    wg = None if ew is None else ew.cuda().requires_grad_(w_grad)
    if via == "module":
        out, (_, alpha) = conv(xg, edge_index=ei.cuda(), edge_weights=wg, edge_attr=None, return_attention_weights=True)
    else:
        P = [getattr(getattr(conv, k), n) for k in TCONV_KEYS for n in ("weight", "bias")]
        out, alpha = RF.transformer_conv(xg, ei.cuda(), wg, H, Fo, *P, geom=geom)
    (out * G.cuda()).sum().backward()
    grads = {k: p.grad for k, p in conv.named_parameters()}
    grads["x"], grads["edge_w"] = xg.grad, None if wg is None else wg.grad
    return out.detach(), alpha.detach(), grads


def check_tconv(what, got, ref, with_w, H):
    out, alpha, grads = got
    r_out, r_alpha, r_grads = ref
    hold("forward", normwise(out, r_out), FWD_TOL, what + " out")
    if r_alpha.numel():
        assert alpha.shape[-1] == H
        hold("forward", normwise(alpha, r_alpha.expand(-1, H).reshape(alpha.shape)), FWD_TOL, what + " alpha")
    hold("gradient", normwise(grads["x"], r_grads["x"]), GRAD_TOL, what + " d_x")
    names = [k + "." + n for k in TCONV_KEYS for n in ("weight", "bias")]
    scale = max(float(r_grads[k].abs().max()) for k in names)
    qk_scale = max(float(r_grads[k].abs().max()) for k in names[:4])
    for k in names:
        r, g_ = r_grads[k], grads[k]
        if (with_w or r_alpha.numel() == 0) and k.startswith(("lin_query", "lin_key")):
            assert float(r.abs().max()) == 0.0 and float(g_.abs().max()) == 0.0, k     # unused: exact zeros
        elif k == "lin_key.bias":
            # a constant shift of every logit of one target: softmax-invariant, zero up to rounding in both
            assert float(r.abs().max()) < 1e-9 * (qk_scale + 1e-30) + 1e-30
            hold("gradient", float(g_.abs().max()) / (qk_scale + 1e-30), GRAD_TOL, what + " " + k)
        elif float(r.abs().max()) < 1e-3 * scale or r.numel() < 8:
            # nearly invariant (q/k under a saturated softmax), or a handful of entries that are each one long
            # cancelling sum (in_ch = 1): held against the scale of the other gradients
            hold("gradient", float((g_.double().cpu() - r).abs().max()) / scale, GRAD_TOL, what + " " + k)
        else:
            hold("gradient", normwise(g_, r), GRAD_TOL, what + " " + k)
    if with_w and r_alpha.numel():
        d = float((grads["edge_w"].double().cpu() - r_grads["edge_w"]).abs().max())
        hold("gradient", d / max(float(r_grads["edge_w"].abs().max()), r_grads["edge_w.scale"], 1e-30), GRAD_TOL, what + " d_edge_w")


TCONV_SHAPES = [(1, 1, 1), (7, 2, 5), (64, 3, 33), (100, 8, 32), (36, 1, 130), (20, 4, 64)]
# (pattern, N, weights or None for q.k logits); every shape runs every line
TCONV_GRAPHS = [("none", 6, None), ("none", 17, "uniform"), ("one", 2, None), ("one", 1, "uniform"), ("dense", 1, None),
                ("er30", 6, "uniform"), ("er70", 17, None), ("dense", 17, "normal"), ("odd", 36, None), ("odd", 36, "x60"),
                ("dup", 36, "uniform"), ("dup", 17, None), ("isolated", 36, None), ("isolated", 100, "uniform"),
                ("star_in", 100, None), ("star_in", 6, "x60"), ("star_out", 100, "normal"), ("star_out", 36, None),
                ("er10", 200, None), ("er10", 200, "x60"), ("dense", 36, None), ("er30", 100, "normal")]


@gpu
@pytest.mark.parametrize("shape", TCONV_SHAPES, ids=lambda s: "%dx%dx%d" % s)
@pytest.mark.parametrize("graph", TCONV_GRAPHS, ids=lambda c: "%s-%d-%s" % (c[0], c[1], c[2] or "qk"))
def test_tconv(shape, graph):
    """One graph through `functional.transformer_conv` and, where it accepts the case, `models_rd.TransformerConv` (bitwise
    the same): out, alpha, d_x, the eight parameter gradients and d_edge_w under loss = sum(out * G)."""
    in_ch, H, Fo = shape
    pattern, N, weights = graph
    seed = TCONV_GRAPHS.index(graph) * 10 + TCONV_SHAPES.index(shape)
    ei, ew = make_graph(pattern, N, seed, weights or "uniform")
    ew = ew if weights else None
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, in_ch, generator=g)
    G = torch.randn(N, H * Fo, generator=g)
    orc = tconv_oracle(in_ch, H, Fo, seed)
    got = tconv_gpu(orc, x, ei, ew, G, "functional")
    if ew is None or H == 1:          # the module refuses edge weights with heads > 1 (test_module_refuses_...)
        mod = tconv_gpu(orc, x, ei, ew, G, "module")
        assert torch.equal(mod[0], got[0]) and torch.equal(mod[1], got[1])
        assert all(torch.equal(mod[2][k], got[2][k]) for k in got[2] if got[2][k] is not None)
    ref = tconv_reference(orc, x, ei, ew, G)
    what = "tconv %s %s" % (shape, graph)
    check_tconv(what, got, ref, ew is not None, H)
    out, r_out = got[0].cpu(), ref[0]
    skip = (x.double() @ orc.lin_skip.weight.T + orc.lin_skip.bias).detach()
    no_in = torch.bincount(ei[1], minlength=N) == 0
    if no_in.any():                   # nodes without incoming edges (all of them when E == 0) get the skip term alone
        hold("forward", normwise(out[no_in], skip[no_in]), FWD_TOL, what + " skip rows")
        assert normwise(r_out[no_in], skip[no_in]) < 1e-12
    if ei.shape[1] == 0:
        assert all(float(got[2][k + "." + n].abs().max()) == 0.0 for k in TCONV_KEYS[:3] for n in ("weight", "bias"))


@gpu
def test_tconv_rows_without_outgoing_edges_carry_no_value_gradient():
    """d_v of a node without outgoing edges is zero, so the value projection's gradients must not see its row of x:
    changing that row's input changes neither d_Wv nor d_bv (its skip and q contributions go elsewhere)."""
    N, in_ch, H, Fo = 36, 20, 4, 64
    ei, ew = make_graph("isolated", N, 3)
    no_out = torch.bincount(ei[0], minlength=N) == 0
    assert no_out.any() and (~no_out).any()
    g = torch.Generator().manual_seed(3)
    x, G = torch.randn(N, in_ch, generator=g), torch.randn(N, H * Fo, generator=g)
    x2 = x.clone()
    x2[no_out] = torch.randn(int(no_out.sum()), in_ch, generator=g)
    orc = tconv_oracle(in_ch, H, Fo, 3)
    for w in (ew, None):
        a, b = tconv_gpu(orc, x, ei, w, G, "functional")[2], tconv_gpu(orc, x2, ei, w, G, "functional")[2]
        if w is not None:             # with supplied weights alpha does not depend on x at all: bitwise the same
            assert torch.equal(a["lin_value.weight"], b["lin_value.weight"]) and torch.equal(a["lin_value.bias"], b["lin_value.bias"])
        ref = tconv_reference(orc, x2, ei, w, G)[2]
        hold("gradient", normwise(b["lin_value.weight"], ref["lin_value.weight"]), GRAD_TOL, "d_Wv")
        hold("gradient", normwise(b["lin_value.bias"], ref["lin_value.bias"]), GRAD_TOL, "d_bv")


@gpu
@pytest.mark.parametrize("x_grad,w_grad", [(False, True), (True, False), (False, False)])
def test_tconv_optional_gradients(x_grad, w_grad):
    """x or the edge weights without requires_grad (d_x == NULL, d_edge_w == NULL): the other gradients are bitwise
    what the full backward gives, and no gradient appears for the tensor that asked for none."""
    N, (in_ch, H, Fo) = 100, (64, 3, 33)
    ei, ew = make_graph("er30", N, 5)
    g = torch.Generator().manual_seed(5)
    x, G = torch.randn(N, in_ch, generator=g), torch.randn(N, H * Fo, generator=g)
    orc = tconv_oracle(in_ch, H, Fo, 5)
    full = tconv_gpu(orc, x, ei, ew, G, "functional")
    part = tconv_gpu(orc, x, ei, ew, G, "functional", x_grad=x_grad, w_grad=w_grad)
    assert torch.equal(full[0], part[0])
    assert (part[2]["x"] is None) == (not x_grad) and (part[2]["edge_w"] is None) == (not w_grad)
    for k, v in part[2].items():
        assert v is None or torch.equal(v, full[2][k]), k
    check_tconv("optional", full, tconv_reference(orc, x, ei, ew, G), True, H)


def test_module_refuses_edge_weights_with_several_heads():
    from raindrop_b200.models_rd import TransformerConv
    with pytest.raises(ValueError, match="heads == 1"):
        TransformerConv(7, 5, heads=2)(torch.zeros(3, 7), torch.zeros(2, 1, dtype=torch.int64), edge_weights=torch.ones(1))


# ---- 3. batched geometry ------------------------------------------------------------------------------------------------
def block_graph(ei, N, n_graphs, node_major):
    """The edge list of `n_graphs` copies of a graph laid out as the rows of x are: applying the oracle to this one graph
    is applying it to every graph on its own (no edge crosses graphs), and autograd of the repeated weights sums
    d_edge_w over the graphs."""
    g = torch.arange(n_graphs)[:, None, None]
    return (ei[None] * n_graphs + g if node_major else ei[None] + g * N).permute(1, 0, 2).reshape(2, -1)


# rows = n_nodes * n_graphs crosses 64 and 128; gemm_splitk_plan gives nsplit = min(ceil(264 / tiles), ceil(rows / 64)):
#   (36, 1, 72) x 36 nodes x 645 graphs: rows 23220, 2 tiles -> nsplit 132      (7, 2, 5) x 17 x 64: rows 1088 -> 17
#   (64, 3, 33) x 17 x 645: rows 10965, 2 tiles -> 132      (20, 4, 64) x 6 x 5: rows 30 -> 1      (100, 8, 32) x 5 x 64 -> 5
BATCHED = [((36, 1, 72), 36, 645, "er30", "uniform"), ((7, 2, 5), 17, 64, "dup", None), ((64, 3, 33), 17, 645, "odd", None),
           ((20, 4, 64), 6, 5, "dense", "normal"), ((100, 8, 32), 5, 64, "star_in", "x60"), ((7, 2, 5), 36, 1, "er30", None),
           ((20, 4, 64), 2, 64, "none", None)]


@gpu
@pytest.mark.parametrize("layout", ["node_major", "graph_major"])
@pytest.mark.parametrize("case", BATCHED, ids=lambda c: "%dx%dx%d-n%d-g%d-%s-%s" % (c[0] + c[1:4] + (c[4] or "qk",)))
def test_tconv_batched(case, layout):
    """Many graphs sharing one edge list in one call, rows node-major (as legacy v1 lays them out) or graph-major, against
    the oracle on the block-diagonal graph; parameter gradients and d_edge_w sum over the graphs."""
    (in_ch, H, Fo), N, n_graphs, pattern, weights = case
    node_major = layout == "node_major"
    seed = 100 + BATCHED.index(case)
    ei, ew = make_graph(pattern, N, seed, weights or "uniform")
    ew = ew if weights else None
    E, rows = ei.shape[1], N * n_graphs
    g = torch.Generator().manual_seed(seed)
    x, G = torch.randn(rows, in_ch, generator=g), torch.randn(rows, H * Fo, generator=g)
    geom = (N, n_graphs, n_graphs, 1) if node_major else (N, n_graphs, 1, N)
    orc = tconv_oracle(in_ch, H, Fo, seed)
    got = tconv_gpu(orc, x, ei, ew, G, "functional", geom=geom)
    again = tconv_gpu(orc, x, ei, ew, G, "functional", geom=geom)
    assert got[1].shape == (n_graphs, E, H)
    # no atomics, fixed reduction order: two identical calls agree to the bit
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])
    assert all(torch.equal(got[2][k], again[2][k]) for k in got[2] if got[2][k] is not None)
    big = block_graph(ei, N, n_graphs, node_major)
    orc = orc.double()
    orc.zero_grad()
    xd = x.double().requires_grad_(True)
    wd = None if ew is None else ew.double().requires_grad_(True)
    out, alpha = orc(xd, big, None if wd is None else wd.repeat(n_graphs))
    alpha.retain_grad()
    (out * G.double()).sum().backward()
    grads = {k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in orc.named_parameters()}
    grads["x"] = xd.grad
    if wd is not None:
        grads["edge_w"] = wd.grad
        grads["edge_w.scale"] = float((alpha.detach() * alpha.grad).abs().reshape(n_graphs, E, -1).sum((0, 2)).max())
    check_tconv("batched %s %s" % (case, layout), got, (out.detach(), alpha.detach(), grads), ew is not None, H)


# ---- 4. Observation_progation(use_beta=True) ----------------------------------------------------------------------------
def beta_scores(orc, x, p_t, ei, ew):
    """float64 per-NODE restatement of the score the pruning ranks by (the oracle evaluates it per edge):
    score[e] = w[e] * mean_t beta[tgt(e), t].  Returns (scores, lin_value pre-activations)."""
    N, T = x.shape[0], p_t.shape[0]
    with torch.no_grad():
        d = lambda t: t.detach().double()
        lifted = (x.double() @ d(orc.increase_dim.weight).T + d(orc.increase_dim.bias)).view(N, T, 32)
        code = torch.cat([d(orc.map_weights)[:, None, :].expand(N, T, 16), p_t.double()[None].expand(N, T, 16)], -1)
        mean_beta = (lifted * code).mean(-1).mean(-1)
        return ew.double() * mean_beta[ei[1]], x.double() @ d(orc.lin_value.weight).T + d(orc.lin_value.bias)


def ties_or_flat_gates(scores, pre, exact_order, rel=1e-4, gate=1e-5):
    """True when a case must be rejected: scores closer than `rel` (relative to the largest) around the cut at E // 2,
    or between neighbours of the kept order when that order is compared exactly, or a pre-activation within `gate` of 0."""
    E = scores.numel()
    s = torch.sort(scores, descending=True).values
    gaps = s[:-1] - s[1:]
    K = E // 2
    watched = gaps[:K] if exact_order else gaps[K - 1:K]
    return bool((watched < rel * float(s.abs().max())).any()) or bool((pre.abs() < gate).any())


def beta_case(N, T, edges, weights, seed0):
    """A use_beta case that stays clear of both discontinuities: seeds seed0, seed0 + 1, ... until one passes.
    `edges`: an edge count (random pairs, duplicates allowed) or a `make_graph` pattern.  The kept order is compared
    exactly up to 64 edges; beyond that hundreds of kept scores cannot all lie 1e-4 apart, so only the cut is guarded
    and the kept list is compared as a set ordered by a non-increasing alpha."""
    C = 4 * T
    for seed in range(seed0, seed0 + 200):
        g = torch.Generator().manual_seed(seed)
        if isinstance(edges, int):
            ei = torch.randint(0, N, (2, edges), generator=g)
            ew = {"uniform": torch.rand, "normal": torch.randn}[weights](edges, generator=g)
        else:
            ei, ew = make_graph(edges, N, seed, weights)
        x = torch.randn(N, C, generator=g)
        p_t = torch.rand(T, 16, generator=g)
        torch.manual_seed(seed)
        orc = ObPropOracle(C, N, 4)
        exact = ei.shape[1] <= 64
        if not ties_or_flat_gates(*beta_scores(orc, x, p_t, ei, ew), exact):
            return dict(N=N, T=T, ei=ei, ew=ew, x=x, p_t=p_t, orc=orc, exact=exact, seed=seed)
    raise AssertionError("no seed clear of ties")


def beta_run_gpu(c, d_alpha=True, x_grad=True, pt_grad=True, G=None, gfull=None):
    from raindrop_b200.models_rd import Observation_progation
    N, C = c["x"].shape
    layer = Observation_progation(in_channels=C, out_channels=C, heads=1, n_nodes=N, ob_dim=4)
    layer.load_state_dict({k: v.float() for k, v in c["orc"].state_dict().items()})
    layer = layer.cuda()
    x = c["x"].cuda().requires_grad_(x_grad)
    p_t = c["p_t"].cuda().requires_grad_(pt_grad)
    ew = c["ew"].cuda().requires_grad_(True)
    out, (ei2, alpha) = layer(x, p_t=p_t, edge_index=c["ei"].cuda(), edge_weights=ew, use_beta=True, edge_attr=None,
                              return_attention_weights=True)
    loss = (out * G.cuda()).sum()
    if d_alpha:
        loss = loss + (alpha * gfull.cuda()[ei2[0] * N + ei2[1]]).sum()
    loss.backward()
    grads = {k: p.grad for k, p in layer.named_parameters()}
    grads.update(x=x.grad, p_t=p_t.grad, edge_w=ew.grad)
    return out.detach(), ei2, alpha.detach(), grads


def beta_run_oracle(c, d_alpha, G, gfull):
    N = c["x"].shape[0]
    orc = ObPropOracle(c["x"].shape[1], N, 4)
    orc.load_state_dict(c["orc"].state_dict())
    orc = orc.double()
    x, p_t, ew = (c[k].double().requires_grad_(True) for k in ("x", "p_t", "ew"))
    out, (ei2, alpha) = orc(x, p_t, c["ei"], ew, use_beta=True)
    loss = (out * G.double()).sum()
    if d_alpha:
        loss = loss + (alpha * gfull.double()[ei2[0] * N + ei2[1]]).sum()
    loss.backward()
    grads = {k: p.grad for k, p in orc.named_parameters()}
    grads.update(x=x.grad, p_t=p_t.grad, edge_w=ew.grad)
    return out.detach(), ei2, alpha.detach(), grads


BETA_PARAMS = ("increase_dim.weight", "increase_dim.bias", "map_weights", "lin_value.weight", "lin_value.bias")
# (N, T, edges, weights); C = 4 T reaches 280 (past 256 threads); N = 100 puts the weight gradients' contraction over the
# nodes on split-K (nsplit = 2); E = 2, 3, 17 and N^2; `normal` weights are negative half of the time
BETA_SPECS = [(2, 1, 2, "uniform"), (2, 5, 3, "normal"), (6, 5, 17, "normal"), (6, 60, "dense", "uniform"), (36, 5, 17, "uniform"),
              (36, 70, "dense", "normal"), (100, 5, "er30", "normal"), (100, 70, 17, "normal"), (100, 60, "er10", "uniform"),
              (6, 1, "dup", "normal"), (6, 70, 3, "uniform"), (2, 60, 17, "normal")]
BETA_CASES = [beta_case(*spec, seed0=1000 * (i + 1)) for i, spec in enumerate(BETA_SPECS)]
# (d_alpha given, x requires grad, p_t requires grad): the backward's optional outputs
BETA_NEEDS = [(True, True, True), (False, True, True), (True, False, True), (True, True, False), (False, False, False)]


def check_beta(what, c, got, ref, d_alpha, x_grad, pt_grad):
    N = c["N"]
    out, ei2, alpha, grads = got
    r_out, r_ei, r_alpha, r_grads = ref
    ei2 = ei2.cpu()
    K = c["ei"].shape[1] // 2
    assert ei2.shape == (2, K)
    if c["exact"]:
        assert torch.equal(ei2, r_ei), what
    else:                              # same kept set (the graph has no duplicate pair), listed by non-increasing alpha
        key, r_key = ei2[0] * N + ei2[1], r_ei[0] * N + r_ei[1]
        assert torch.equal(torch.sort(key).values, torch.sort(r_key).values), what
        assert bool((alpha[:-1] >= alpha[1:]).all())
        r_alpha = r_alpha[torch.argsort(r_key)][torch.searchsorted(torch.sort(r_key).values, key)]
    hold("beta forward", normwise(alpha, r_alpha), BETA_FWD_TOL, what + " alpha")
    hold("beta forward", normwise(out, r_out), BETA_FWD_TOL, what + " out")
    kept_src = torch.zeros(N, dtype=torch.bool)
    kept_src[ei2[0]] = True
    assert float(out.cpu()[~kept_src].abs().sum()) == 0.0          # a node that keeps no outgoing edge: exactly zero
    scale = max(float(r_grads[k].abs().max()) for k in BETA_PARAMS)
    for k in BETA_PARAMS + ("x", "p_t", "edge_w"):
        if (k == "x" and not x_grad) or (k == "p_t" and not pt_grad):
            assert grads[k] is None
            continue
        r = r_grads[k]
        if float(r.abs().max()) < 1e-3 * scale:                    # e.g. p_t without d_alpha on a 2-edge graph
            hold("beta gradient", float((grads[k].double().cpu() - r).abs().max()) / scale, BETA_GRAD_TOL, what + " " + k)
        else:
            hold("beta gradient", normwise(grads[k], r), BETA_GRAD_TOL, what + " " + k)
    pruned = torch.ones(c["ei"].shape[1], dtype=torch.bool)
    pruned[torch.topk(beta_scores(c["orc"], c["x"], c["p_t"], c["ei"], c["ew"])[0], K).indices] = False
    assert float(r_grads["edge_w"][pruned].abs().sum()) == 0.0
    assert float(grads["edge_w"].cpu()[pruned].abs().sum()) == 0.0  # pruned edges get exactly no gradient


@gpu
@pytest.mark.parametrize("needs", BETA_NEEDS, ids=lambda n: "alpha%d-x%d-pt%d" % n)
@pytest.mark.parametrize("i", range(len(BETA_SPECS)), ids=lambda i: "N%d-T%d-%s-%s" % BETA_SPECS[i])
def test_obprop_beta(i, needs):
    """`Observation_progation(use_beta=True)`: pruned edge list, alpha, out and every gradient, with the backward's
    optional outputs (d_alpha, d_x, d_p_t) present or not."""
    c = BETA_CASES[i]
    d_alpha, x_grad, pt_grad = needs
    g = torch.Generator().manual_seed(c["seed"])
    G = torch.randn(c["N"], 4 * c["T"], generator=g)
    gfull = torch.randn(c["N"] * c["N"], generator=g)
    got = beta_run_gpu(c, d_alpha, x_grad, pt_grad, G, gfull)
    ref = beta_run_oracle(c, d_alpha, G, gfull)
    check_beta("beta %s %s" % (BETA_SPECS[i], needs), c, got, ref, d_alpha, x_grad, pt_grad)


@gpu
def test_obprop_beta_pruned_source():
    """A source all of whose edges fall below the cut keeps nothing: its output row is exactly 0 although it has
    outgoing edges, and those edges get exactly no gradient."""
    c = beta_case(17, 5, 60, "uniform", 77000)
    s0 = int(c["ei"][0, 0])
    mb, _ = beta_scores(c["orc"], c["x"], c["p_t"], c["ei"], torch.ones(60))            # mean beta of each edge's target
    mine = c["ei"][0] == s0
    low = -(3 + 0.1 * torch.arange(60)) * mb.abs().max() / mb                             # scores below every other edge's
    c["ew"] = torch.where(mine, low.float(), c["ew"])
    assert not ties_or_flat_gates(*beta_scores(c["orc"], c["x"], c["p_t"], c["ei"], c["ew"]), True)
    g = torch.Generator().manual_seed(1)
    G, gfull = torch.randn(17, 20, generator=g), torch.randn(17 * 17, generator=g)
    got = beta_run_gpu(c, True, True, True, G, gfull)
    check_beta("pruned source", c, got, beta_run_oracle(c, True, G, gfull), True, True, True)
    assert not bool((got[1][0].cpu() == s0).any())
    assert float(got[0][s0].abs().sum()) == 0.0 and float(got[3]["edge_w"].cpu()[mine].abs().sum()) == 0.0


@gpu
@pytest.mark.parametrize("E", [4, 6])
def test_obprop_beta_tie_rule(E):
    """Exactly tied scores (two edges into one target with the same weight) are ranked lower edge id first, at the cut
    (E = 4: edges 1 and 2 tie for the last kept place) and inside the kept list (E = 6).  torch's CPU argsort is not
    stable and may order such a pair either way, so this pins the documented rule, not the oracle's choice."""
    c = beta_case(6, 5, 17, "uniform", 88000)
    mb = beta_scores(c["orc"], c["x"], c["p_t"], c["ei"], torch.ones(17))[0]       # mean beta of each edge's target
    mean_beta = torch.zeros(6, dtype=torch.float64)
    mean_beta[c["ei"][1]] = mb
    t = int(torch.argmax(mean_beta.abs()))
    sg = float(torch.sign(mean_beta[t]))
    others = [n for n in range(6) if n != t]
    # scores: edge 0 highest, edges 1 and 2 tied, the rest negative
    src = torch.tensor([others[0], others[1], others[2], others[3], others[4], t][:E])
    ew = torch.tensor([3.0, 2.0, 2.0, -1.0, -2.0, -3.0][:E]) * sg
    c["ei"], c["ew"] = torch.stack([src, torch.full_like(src, t)]), ew
    from raindrop_b200.models_rd import Observation_progation
    layer = Observation_progation(in_channels=20, out_channels=20, heads=1, n_nodes=6, ob_dim=4)
    layer.load_state_dict(c["orc"].state_dict())
    layer = layer.cuda()
    _, (ei2, alpha) = layer(c["x"].cuda(), p_t=c["p_t"].cuda(), edge_index=c["ei"].cuda(), edge_weights=ew.cuda(),
                            use_beta=True, edge_attr=None, return_attention_weights=True)
    assert torch.equal(ei2.cpu(), c["ei"][:, : E // 2])
    if E == 6:
        assert float(alpha[1].detach()) == float(alpha[2].detach())


# ---- 5. rd_node_scale and the use_beta=False module path ------------------------------------------------------------
@gpu
@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_node_scale(pattern, weights):
    for N in NODE_COUNTS:
        ei, ew = make_graph(pattern, N, 11, weights)
        s = RF.node_scale(ei.cuda(), ew.cuda(), N).cpu()
        ref = node_scale_from_graph(ei, ew.double(), N, dtype=torch.float64)
        no_in = torch.bincount(ei[1], minlength=N) == 0
        assert bool((s[no_in] == 0).all()) and bool((ref[no_in] == 0).all())
        hold("node_scale", float((s.double() - ref).abs().max()), 1.5e-6, "node_scale %s %s N=%d" % (pattern, weights, N))


@gpu
@pytest.mark.parametrize("N,B,T,pattern", [(6, 3, 5, "er30"), (17, 5, 15, "isolated"), (36, 5, 60, "odd"), (36, 2, 7, "star_in")])
def test_obprop_module_without_beta(N, B, T, pattern):
    """`Observation_progation.forward(use_beta=False)` on B samples stacked as B*N rows (one block-diagonal graph, as
    PyG batches them) against the edge-wise oracle.  x and W are TF32-representable, which the operator's documented
    rounding then leaves alone; at these sizes the operator runs error-compensated, so forward and gradients are held
    at fp32 level."""
    from raindrop_b200.models_rd import Observation_progation
    C, rows = 4 * T, B * N
    ei1, _ = make_graph(pattern, N, 13)
    ei = block_graph(ei1, N, B, node_major=False)
    g = torch.Generator().manual_seed(N + B)
    ew = torch.rand(ei.shape[1], generator=g)
    x = round_tf32(torch.randn(rows, C, generator=g))
    G = torch.randn(rows, C, generator=g)
    torch.manual_seed(N)
    orc = ObPropOracle(C, rows, 4)
    with torch.no_grad():
        orc.lin_value.weight.copy_(round_tf32(orc.lin_value.weight))
    layer = Observation_progation(in_channels=C, out_channels=C, heads=1, n_nodes=rows, ob_dim=4)
    layer.load_state_dict(orc.state_dict())
    layer = layer.cuda()
    xg, wg = x.cuda().requires_grad_(True), ew.cuda().requires_grad_(True)
    out, (ei2, alpha) = layer(xg, p_t=None, edge_index=ei.cuda(), edge_weights=wg, use_beta=False, edge_attr=None,
                              return_attention_weights=True)
    assert torch.equal(ei2.cpu(), ei) and torch.equal(alpha.detach().cpu(), ew[:, None])      # pre-softmax weights, bit exact
    (out * G.cuda()).sum().backward()
    orc = orc.double()
    xd = x.double().requires_grad_(True)
    r_out, _ = orc(xd, None, ei, ew.double(), use_beta=False)
    (r_out * G.double()).sum().backward()
    hold("obprop forward", normwise(out.detach(), r_out.detach()), BETA_FWD_TOL, "obprop out")
    no_in = torch.bincount(ei[1], minlength=rows) == 0
    assert float(out.detach().cpu()[no_in].abs().sum()) == 0.0
    for name, got, ref in (("d_x", xg.grad, xd.grad), ("d_W", layer.lin_value.weight.grad, orc.lin_value.weight.grad),
                           ("d_b", layer.lin_value.bias.grad, orc.lin_value.bias.grad)):
        hold("obprop gradient", normwise(got, ref), GRAD_TOL, "obprop " + name)


# ---- 6. scratch sizes ---------------------------------------------------------------------------------------------------
TAIL = 1024          # floats (4 KB) owned by the test past the reported scratch size
SENTINEL = 0x5A5A5A5A


def padded_scratch(nbytes):
    assert nbytes > 0 and nbytes % 4 == 0
    return torch.full((nbytes // 4 + TAIL,), SENTINEL, dtype=torch.int32, device="cuda")


def tail_untouched(sc):
    return bool((sc[-TAIL:] == SENTINEL).all())


@gpu
@pytest.mark.parametrize("case", [((7, 2, 5), 6, 1, "er30", None), ((64, 3, 33), 100, 1, "er30", "uniform"),
                                  ((36, 1, 72), 36, 64, "odd", "uniform"), ((20, 4, 64), 17, 5, "dup", None),
                                  ((1, 1, 1), 2, 1, "one", None)], ids=str)
def test_scratch_sizes_transformer_conv(case):
    """rd_transformer_conv_fwd / _bwd called directly with exactly the reported scratch plus a sentinel tail: the tail
    stays untouched and the results equal the autograd wrapper's to the bit."""
    from raindrop_b200 import lib as L
    lib = L.load()
    (in_ch, H, Fo), N, n_graphs, pattern, weights = case
    ei, ew = make_graph(pattern, N, 21, weights or "uniform")
    ew = ew if weights else None
    E, rows, HF = ei.shape[1], N * n_graphs, H * Fo
    g = torch.Generator().manual_seed(21)
    x, G = torch.randn(rows, in_ch, generator=g), torch.randn(rows, HF, generator=g)
    orc = tconv_oracle(in_ch, H, Fo, 21)
    geom = (N, n_graphs, n_graphs, 1)
    want = tconv_gpu(orc, x, ei, ew, G, "functional", geom=geom)
    P = [getattr(getattr(orc, k), n).detach().float().cuda() for k in TCONV_KEYS for n in ("weight", "bias")]
    xg, Gg, src, tgt = x.cuda(), G.cuda(), ei[0].contiguous().cuda(), ei[1].contiguous().cuda()
    wg = None if ew is None else ew.cuda()
    out, alpha = torch.empty(rows, HF, device="cuda"), torch.empty(n_graphs, E, H, device="cuda")
    sc = padded_scratch(lib.rd_transformer_conv_scratch_bytes(N, n_graphs, in_ch, H, Fo, E, 0))
    L.check(lib.rd_transformer_conv_fwd(xg.data_ptr(), *geom, in_ch, H, Fo, src.data_ptr(), tgt.data_ptr(), L.ptr(wg), E,
                                        *[p.data_ptr() for p in P], out.data_ptr(), alpha.data_ptr(), sc.data_ptr(),
                                        L.stream_ptr()), "rd_transformer_conv_fwd")
    assert tail_untouched(sc)
    assert torch.equal(out, want[0]) and torch.equal(alpha, want[1])
    d_x = torch.empty_like(xg)
    gr = [torch.empty_like(p) for p in P]
    d_w = None if wg is None else torch.zeros(E, device="cuda")
    sc = padded_scratch(lib.rd_transformer_conv_scratch_bytes(N, n_graphs, in_ch, H, Fo, E, 1))
    L.check(lib.rd_transformer_conv_bwd(xg.data_ptr(), *geom, in_ch, H, Fo, src.data_ptr(), tgt.data_ptr(), L.ptr(wg), E,
                                        *[p.data_ptr() for p in P[:7]], alpha.data_ptr(), Gg.data_ptr(), d_x.data_ptr(),
                                        *[t.data_ptr() for t in gr], L.ptr(d_w), sc.data_ptr(), L.stream_ptr()),
            "rd_transformer_conv_bwd")
    assert tail_untouched(sc)
    assert torch.equal(d_x, want[2]["x"]) and (d_w is None or torch.equal(d_w, want[2]["edge_w"]))
    names = [k + "." + n for k in TCONV_KEYS for n in ("weight", "bias")]
    assert all(torch.equal(a, want[2][k]) for a, k in zip(gr, names))


@gpu
@pytest.mark.parametrize("N,T,edges", [(6, 5, 17), (36, 70, "dense"), (100, 60, "er10"), (100, 96, 40)])
def test_scratch_sizes_obprop_beta(N, T, edges):
    """The same for rd_obprop_beta_fwd / _bwd.  (100, 96, .): C = 384, where the [8C, C] weight gradient has too many tiles
    to split over the nodes but the [C, C] one still does, so the shared partial buffer is sized by the smaller GEMM."""
    from raindrop_b200 import lib as L
    lib = L.load()
    c = beta_case(N, T, edges, "normal", 99000 + N + T)
    C, E = 4 * T, c["ei"].shape[1]
    K = E // 2
    g = torch.Generator().manual_seed(5)
    G, gfull = torch.randn(N, C, generator=g), torch.randn(N * N, generator=g)
    want = beta_run_gpu(c, True, True, True, G, gfull)
    sd = c["orc"].state_dict()
    P = [sd[k].float().cuda() for k in BETA_PARAMS]
    x, p_t, w = c["x"].cuda(), c["p_t"].cuda(), c["ew"].cuda()
    src, tgt = c["ei"][0].contiguous().cuda(), c["ei"][1].contiguous().cuda()
    out, ei2, alpha = torch.empty(N, C, device="cuda"), torch.empty(2, K, dtype=torch.int64, device="cuda"), torch.empty(K, device="cuda")
    sc = padded_scratch(lib.rd_obprop_beta_scratch_bytes(N, T, 4, E))
    L.check(lib.rd_obprop_beta_fwd(x.data_ptr(), p_t.data_ptr(), src.data_ptr(), tgt.data_ptr(), w.data_ptr(), E, N, T, 4,
                                   *[p.data_ptr() for p in P], out.data_ptr(), ei2[0].data_ptr(), ei2[1].data_ptr(),
                                   alpha.data_ptr(), sc.data_ptr(), L.stream_ptr()), "rd_obprop_beta_fwd")
    assert tail_untouched(sc)
    assert torch.equal(out, want[0]) and torch.equal(ei2, want[1]) and torch.equal(alpha, want[2])
    d_alpha = gfull.cuda()[ei2[0] * N + ei2[1]].contiguous()
    d_x, d_w, d_pt = torch.empty_like(x), torch.empty(E, device="cuda"), torch.empty(T, 16, device="cuda")
    gr = [torch.empty_like(p) for p in P]
    sc = padded_scratch(lib.rd_obprop_beta_bwd_scratch_bytes(N, T, 4, E))
    L.check(lib.rd_obprop_beta_bwd(x.data_ptr(), p_t.data_ptr(), src.data_ptr(), tgt.data_ptr(), w.data_ptr(), E, N, T, 4,
                                   *[p.data_ptr() for p in P], G.cuda().data_ptr(), d_alpha.data_ptr(), d_x.data_ptr(),
                                   d_w.data_ptr(), d_pt.data_ptr(), *[t.data_ptr() for t in gr], sc.data_ptr(),
                                   L.stream_ptr()), "rd_obprop_beta_bwd")
    assert tail_untouched(sc)
    assert torch.equal(d_x, want[3]["x"]) and torch.equal(d_w, want[3]["edge_w"]) and torch.equal(d_pt, want[3]["p_t"])
    assert all(torch.equal(a, want[3][k]) for a, k in zip(gr, BETA_PARAMS))
    ref = beta_run_oracle(c, True, G, gfull)
    check_beta("scratch beta", c, want, ref, True, True, True)


# ---- 7. argument checks (on the host: no device needed) ---------------------------------------------------------------
def _tconv_args(rows=6, in_ch=3):
    P = [torch.zeros(4, in_ch), torch.zeros(4)] * 4
    return torch.zeros(rows, in_ch), torch.zeros(2, 5, dtype=torch.int64), P


@pytest.mark.parametrize("geom,match", [((3, 2, 1, 1), "node_stride"), ((3, 2, 2, 2), "node_stride"), ((3, 2, 3, 1), "node_stride"),
                                        ((3, 2, 1, 4), "graph_stride"), ((6, 1, 2, 0), "node_stride"), ((0, 2, 2, 1), "n_nodes"),
                                        ((3, 3, 3, 1), "rows"), ((4, 2, 1, 4), "rows")])
def test_transformer_conv_refuses_geometry_that_does_not_tile_the_rows(geom, match):
    x, ei, P = _tconv_args()
    with pytest.raises(RaindropB200Error, match=match):
        RF.transformer_conv(x, ei, None, 2, 2, *P, geom=geom)


@pytest.mark.parametrize("ei,ew,match", [
    (torch.zeros(2, 5, dtype=torch.int32), None, "edge_index"), (torch.zeros(5, 2, dtype=torch.int64), None, "edge_index"),
    (torch.zeros(10, dtype=torch.int64), None, "edge_index"), (torch.zeros(2, 5), None, "edge_index"),
    (torch.zeros(2, 5, dtype=torch.int64), torch.zeros(4), "edge_weights"),
    (torch.zeros(2, 5, dtype=torch.int64), torch.zeros(5, 1), "edge_weights")])
def test_operators_refuse_malformed_edge_lists(ei, ew, match):
    x, _, P = _tconv_args()
    with pytest.raises(RaindropB200Error, match=match):
        RF.transformer_conv(x, ei, ew, 2, 2, *P)
    ew1 = torch.zeros(5) if ew is None else ew
    with pytest.raises(RaindropB200Error, match=match):
        RF.node_scale(ei, ew1, 6)
    with pytest.raises(RaindropB200Error, match=match):
        RF.obprop_beta(torch.zeros(6, 4), torch.zeros(1, 16), ei, ew1, 4, *[None] * 5)


@pytest.mark.parametrize("E", [0, 1])
def test_obprop_beta_refuses_fewer_than_two_edges(E):
    """use_beta keeps the top E // 2 edges; with E < 2 nothing would be kept, and forward, backward and the scratch
    queries used to disagree about that.  The forward refuses."""
    with pytest.raises(RaindropB200Error, match="E >= 2"):
        RF.obprop_beta(torch.zeros(6, 4), torch.zeros(1, 16), torch.zeros(2, E, dtype=torch.int64), torch.zeros(E), 4, *[None] * 5)


@gpu
def test_c_abi_refuses_what_the_wrappers_refuse():
    from raindrop_b200 import lib as L
    lib = L.load()
    assert lib.rd_obprop_beta_scratch_bytes(6, 5, 4, 1) == 0 and lib.rd_obprop_beta_bwd_scratch_bytes(6, 5, 4, 1) == 0
    t = torch.zeros(4096, device="cuda")
    i = torch.zeros(16, dtype=torch.int64, device="cuda")
    p, q = t.data_ptr(), i.data_ptr()
    assert lib.rd_obprop_beta_fwd(p, p, q, q, p, 1, 6, 5, 4, p, p, p, p, p, p, q, q, p, p, L.stream_ptr()) == -2
    assert b"E >= 2" in lib.rd_last_error_string()
    assert lib.rd_transformer_conv_fwd(p, 3, 2, 1, 1, 3, 1, 2, q, q, 0, 5, p, p, p, p, p, p, p, p, p, p, p, L.stream_ptr()) == -2
    assert b"node_stride" in lib.rd_last_error_string()


# ---- 8. legacy Raindrop v1 on more than one fixture ---------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["v1_sparse_b5", "v1_b1"])
def test_legacy_raindrop_v1_fixtures(golden_dir, name):
    """Legacy `Raindrop` v1 against fixtures of the reference's own class (oracle/make_golden.py V1_CASES), with the
    tolerances of test_gpu_parity.py::test_legacy_raindrop_v1_against_reference.  The reference hard-codes 36 sensors
    and 215 steps, so the cases vary what it lets vary: B = 5 (1075 rows) on a sparse sensor graph in which sensor 7
    keeps only its forced self loop, with a one-layer encoder on d_model = 36; and B = 1 with four heads."""
    import json
    from raindrop_b200.models_rd import Raindrop
    from raindrop_b200.synth import CONFIGS, make_batch
    z = np.load(golden_dir + "/" + name + ".npz")
    meta = json.loads(bytes(z["meta"]).decode())
    cfg = dict(CONFIGS["P12"]); cfg["name"] = "P12"
    batch = make_batch(dict(cfg, d_ob=2), meta["batch"], seed=meta["data_seed"])
    gs = torch.from_numpy(z["global_structure"])
    if name == "v1_sparse_b5":
        assert float(gs[7].abs().sum() + gs[:, 7].abs().sum()) == 0.0
    model = Raindrop(*meta["ctor"], gs)
    assert sorted(model.state_dict()) == sorted(k[3:] for k in z.files if k.startswith("sd."))
    model.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")})
    model = model.cuda().eval()
    d = to_dev(batch)
    logits, distance, third = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    assert third is None and float(distance) == float(z["distance"]) == 0.0
    assert normwise(logits, z["logits"]) < 1e-4, normwise(logits, z["logits"])
    loss = F.cross_entropy(logits, d["y"])
    assert abs(loss.item() - float(z["loss"])) < 1e-4
    loss.backward()
    params = dict(model.named_parameters())
    with_grad = sorted(k[5:] for k in z.files if k.startswith("grad."))
    assert sorted(k for k, p in params.items() if p.grad is not None and float(p.grad.abs().max()) > 0) == with_grad
    worst = max((normwise(params[k].grad, z["grad." + k]), k) for k in with_grad)
    hold("v1 gradient", worst[0], 2e-3, "v1 %s %s" % (name, worst[1]))


# ---- 9. the oracle side, without a GPU ----------------------------------------------------------------------------------
def central_differences(loss, t, idx, h=1e-6):
    out = []
    for i in idx:
        flat = t.data.view(-1)
        keep = float(flat[i])
        flat[i] = keep + h
        up = float(loss())
        flat[i] = keep - h
        dn = float(loss())
        flat[i] = keep
        out.append((up - dn) / (2 * h))
    return torch.tensor(out, dtype=torch.float64)


def check_autograd_against_differences(loss, leaves):
    """autograd of `loss()` w.r.t. each named leaf against central differences at 12 seeded entries, to 1e-6 of the
    largest gradient entry."""
    g = torch.Generator().manual_seed(0)
    grads = torch.autograd.grad(loss(), list(leaves.values()), allow_unused=True)
    scale = max(float(v.abs().max()) for v in grads if v is not None)
    for (k, t), a in zip(leaves.items(), grads):
        idx = torch.randint(0, t.numel(), (min(12, t.numel()),), generator=g).tolist()
        with torch.no_grad():
            fd = central_differences(loss, t, idx)
        a = torch.zeros_like(t) if a is None else a
        assert float((a.reshape(-1)[idx] - fd).abs().max()) < 1e-6 * scale, k


@pytest.mark.parametrize("shape,pattern,N,weights", [((7, 2, 5), "isolated", 17, None), ((20, 4, 64), "star_in", 6, "normal"),
                                                    ((36, 1, 130), "dup", 17, "uniform")])
def test_tconv_oracle_autograd_against_finite_differences(shape, pattern, N, weights):
    in_ch, H, Fo = shape
    ei, ew = make_graph(pattern, N, 31, weights or "uniform")
    g = torch.Generator().manual_seed(31)
    x = torch.randn(N, in_ch, generator=g).double().requires_grad_(True)
    G = torch.randn(N, H * Fo, generator=g).double()
    orc = tconv_oracle(in_ch, H, Fo, 31).double()
    leaves = dict(orc.named_parameters(), x=x)
    wd = None
    if weights:
        wd = leaves["edge_w"] = ew.double().requires_grad_(True)
    check_autograd_against_differences(lambda: (orc(x, ei, wd)[0] * G).sum(), leaves)


@pytest.mark.parametrize("i", [2, 4, 9])
def test_obprop_oracle_autograd_against_finite_differences(i):
    c = BETA_CASES[i]
    N, C = c["x"].shape
    orc = ObPropOracle(C, N, 4)
    orc.load_state_dict(c["orc"].state_dict())
    orc = orc.double()
    g = torch.Generator().manual_seed(i)
    G, ga = torch.randn(N, C, generator=g).double(), torch.randn(c["ei"].shape[1] // 2, generator=g).double()
    x, p_t, ew = (c[k].double().requires_grad_(True) for k in ("x", "p_t", "ew"))

    def loss():
        out, (_, alpha) = orc(x, p_t, c["ei"], ew, use_beta=True)
        return (out * G).sum() + (alpha * ga).sum()
    leaves = {k: p for k, p in orc.named_parameters() if k in BETA_PARAMS}
    leaves.update(x=x, p_t=p_t, edge_w=ew)
    check_autograd_against_differences(loss, leaves)


def test_tie_guard_rejects_near_ties_and_flat_gates():
    pre = torch.ones(3, dtype=torch.float64)
    clear = torch.tensor([4.0, 3.0, 2.0, 1.0], dtype=torch.float64)
    assert not ties_or_flat_gates(clear, pre, True)
    at_cut = torch.tensor([4.0, 3.0, 3.0 - 2e-4, 1.0], dtype=torch.float64)        # 5e-5 relative, around the cut at K = 2
    assert ties_or_flat_gates(at_cut, pre, True) and ties_or_flat_gates(at_cut, pre, False)
    in_kept = torch.tensor([4.0, 4.0 - 2e-4, 2.0, 1.0], dtype=torch.float64)       # between the two kept edges
    assert ties_or_flat_gates(in_kept, pre, True) and not ties_or_flat_gates(in_kept, pre, False)
    below = torch.tensor([4.0, 3.0, 1.0, 1.0], dtype=torch.float64)                # ties among pruned edges change nothing
    assert not ties_or_flat_gates(below, pre, True)
    assert ties_or_flat_gates(clear, torch.tensor([1.0, -5e-6], dtype=torch.float64), True)
    for c in BETA_CASES:                                                           # every committed case passed the guard
        assert not ties_or_flat_gates(*beta_scores(c["orc"], c["x"], c["p_t"], c["ei"], c["ew"]), c["exact"])


def test_float64_oracles_reproduce_the_operator_fixtures(golden_dir):
    z, zg = np.load(golden_dir + "/operators.npz"), np.load(golden_dir + "/operators_grad.npz")
    ei = torch.from_numpy(z["obprop.edge_index"])
    N, C = z["obprop.x"].shape
    layer = ObPropOracle(C, N, 4)
    layer.load_state_dict({k[len("obprop.sd."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("obprop.sd.")})
    layer = layer.double()
    G = torch.from_numpy(zg["obprop.G"]).double()
    for ub in (False, True):
        tag = "obprop.beta%d." % int(ub)
        layer.zero_grad()
        x, p_t, ew = (torch.from_numpy(z["obprop." + k]).double().requires_grad_(True) for k in ("x", "p_t", "edge_w"))
        out, (ei2, alpha) = layer(x, p_t, ei, ew, use_beta=ub)
        assert normwise(out.detach(), z[tag + "out"]) < 1e-6 and normwise(alpha.detach(), z[tag + "alpha"]) < 1e-6
        assert torch.equal(ei2, torch.from_numpy(z[tag + "edge_index"]))
        loss = (out * G).sum()
        if ub:
            loss = loss + (alpha * torch.from_numpy(zg[tag + "g_alpha"]).double()).sum()
        loss.backward()
        assert normwise(x.grad, zg[tag + "d_x"]) < 1e-6
        if ub:
            assert normwise(ew.grad, zg[tag + "d_edge_w"]) < 1e-6 and normwise(p_t.grad, zg[tag + "d_p_t"]) < 1e-6
        params = dict(layer.named_parameters())
        for k in zg.files:
            if k.startswith(tag + "grad."):
                assert normwise(params[k[len(tag + "grad."):]].grad, zg[k]) < 1e-6, k
    xn = torch.from_numpy(z["tconv.x"]).double()
    for tag, heads, use_w in (("tconv.w.", 1, True), ("tconv.qk.", 2, False)):
        conv = TransformerConvOracle(7, 5, heads)
        conv.load_state_dict({k[len(tag + "sd."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "sd.")})
        ew = torch.from_numpy(z["obprop.edge_w"]) if use_w else None
        out, alpha, grads = tconv_reference(conv, xn, ei, ew, torch.from_numpy(zg[tag + "G"]))
        assert normwise(out, z[tag + "out"]) < 1e-6 and normwise(alpha, z[tag + "alpha"]) < 1e-6
        assert normwise(grads["x"], zg[tag + "d_x"]) < 1e-6
        scale = max(float(np.abs(zg[k]).max()) for k in zg.files if k.startswith(tag + "grad."))
        for k in zg.files:
            if k.startswith(tag + "grad."):       # the fixture is float32: invariant gradients are its rounding noise
                assert float((grads[k[len(tag + "grad."):]] - torch.from_numpy(zg[k]).double()).abs().max()) < 1e-6 * scale, k
