"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs
may import this file; the product path (raindrop_b200/) never does.

What is restated (reference file:line given at each function):
  * PyG `utils.softmax` / `torch_scatter.scatter(reduce='add')` (third-party, NOT under
    the reference tree, unpinned in requirements.txt:1-9)        -> segment_softmax, scatter_rows
  * `Observation_progation.forward/message/aggregate`            -> ObPropOracle
    (code/Ob_propagation.py:94-132, 157-211, 213-228)
  * `TransformerConv.forward/message`                            -> TransformerConvOracle
    (code/transformer_conv.py:139-207)
  * `PositionalEncodingTF.getPE`                                 -> positional_encoding
    (code/models_rd.py:28-43)
  * `Raindrop_v2.__init__/forward`                               -> RaindropV2Oracle
    (code/models_rd.py:208-387)
  * one post-LN `nn.TransformerEncoderLayer` written out in matmuls (the reference calls the torch
    module at code/models_rd.py:232-237,358)                      -> encoder_layer_explicit

Pinning status: the reference has NO tests / golden vectors / KATs for this path (SURVEY.md
section 4).  The oracle is pinned instead against outputs of the reference's own unmodified files
run in the build container under `oracle/ref_harness.py` (fixtures in tests/golden/, generator
`oracle/make_golden.py`).  At the PyG boundary itself parity is UNPINNED (PyG is absent and its
version is not recorded by the reference); the shim semantics used are the ones stable across
PyG 1.6 - 2.x and are additionally cross-checked by the dense closed form `forward_dense`.

Two evaluation modes of the same model:
  * `forward(...)`        -- the reference's own structure: Python loop over samples, gather per
                             edge, per-edge lin_value GEMM, segment softmax, scatter-add.  This is
                             what `cpu_baseline` times (kind = "port").
  * `forward_dense(...)`  -- independent closed form: per node, out = relu(W x + b) * sum_e alpha_e.
                             Used to cross-check the edge-wise path and at sizes where the loop
                             is too slow.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------
# PyG / torch_scatter primitives (third-party semantics, see module docstring)
# --------------------------------------------------------------------------------------------
def segment_softmax(logits, seg, n_seg):
    """exp(x - max_seg) / (sum_seg + 1e-16) along dim 0, grouped by seg[e].
    Called from code/Ob_propagation.py:195 and code/transformer_conv.py:201."""
    tail = tuple(logits.shape[1:])
    idx = seg.view((-1,) + (1,) * len(tail)).expand_as(logits)
    mx = torch.full((n_seg,) + tail, -math.inf, dtype=logits.dtype)
    mx = mx.scatter_reduce(0, idx, logits.detach(), reduce="amax", include_self=True)
    ex = torch.exp(logits - mx.gather(0, idx))
    den = torch.zeros((n_seg,) + tail, dtype=logits.dtype).scatter_add(0, idx, ex)
    return ex / (den.gather(0, idx) + 1e-16)


def scatter_rows(msg, seg, n_seg):
    """out[n] = sum_{e: seg[e] == n} msg[e]; rows without any message stay exactly zero.
    `torch_scatter.scatter(..., dim=0, dim_size=N, reduce='add')`, code/Ob_propagation.py:227."""
    idx = seg.view((-1,) + (1,) * (msg.dim() - 1)).expand_as(msg)
    return torch.zeros((n_seg,) + tuple(msg.shape[1:]), dtype=msg.dtype).scatter_add(0, idx, msg)


def glorot_(t):
    """PyG inits.glorot: U(+-sqrt(6/(size(-2)+size(-1)))) (code/models_rd.py:276)."""
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


def graph_from_adjacency(adj):
    """code/models_rd.py:307-311: force the diagonal to one, list non-zeros row-major.
    edge_index[0] = row = source, edge_index[1] = col = target."""
    adj = adj.clone()
    n = adj.shape[0]
    adj[torch.arange(n), torch.arange(n)] = 1
    edge_index = torch.nonzero(adj).T.contiguous()
    return edge_index, adj[edge_index[0], edge_index[1]]


def node_scale_from_graph(edge_index, edge_w, n_nodes, dtype=torch.float32):
    """Closed form of 'segment softmax then scatter-add' when the message only depends on the
    target: s[n] = sum_{e -> n} softmax_e(w).  1 (up to the 1e-16) for nodes with an incoming
    edge, exactly 0 for isolated ones."""
    a = segment_softmax(edge_w.to(dtype)[:, None], edge_index[1], n_nodes)
    return scatter_rows(a, edge_index[1], n_nodes)[:, 0]


# --------------------------------------------------------------------------------------------
# Observation propagation layer (code/Ob_propagation.py)
# --------------------------------------------------------------------------------------------
class ObPropOracle(nn.Module):
    """Parameter names/shapes as code/Ob_propagation.py:39-70 so state dicts interchange."""

    def __init__(self, channels, n_nodes, ob_dim, heads=1):
        super().__init__()
        assert heads == 1
        C = channels
        self.C, self.n_nodes, self.ob_dim = C, n_nodes, ob_dim
        # construction order follows code/Ob_propagation.py:39-70 so that a seeded construction
        # draws the same random numbers as the reference
        self.lin_key = nn.Linear(C, C)
        self.lin_query = nn.Linear(C, C)
        self.lin_value = nn.Linear(C, C)
        self.lin_skip = nn.Linear(C, C)
        self.weight = nn.Parameter(torch.empty(C, C))
        self.bias = nn.Parameter(torch.empty(C))
        self.nodewise_weights = nn.Parameter(torch.empty(n_nodes, C))
        self.increase_dim = nn.Linear(C, C * 8)
        self.map_weights = nn.Parameter(torch.empty(n_nodes, 16))
        # reset_parameters(), code/Ob_propagation.py:76-92
        for lin in (self.lin_key, self.lin_query, self.lin_value, self.lin_skip):
            lin.reset_parameters()
        glorot_(self.weight)
        with torch.no_grad():
            self.bias.uniform_(-1 / math.sqrt(C), 1 / math.sqrt(C))
        glorot_(self.nodewise_weights)
        glorot_(self.map_weights)
        self.increase_dim.reset_parameters()

    def forward(self, x, p_t, edge_index, edge_w, use_beta=False):
        """x [N, C]; returns (out [N, C], (edge_index', alpha)).
        Follows propagate -> message -> aggregate, code/Ob_propagation.py:114,157-228."""
        n = x.shape[0]
        src_of, tgt_of = edge_index[0], edge_index[1]
        x_tgt = x.index_select(0, tgt_of)                    # PyG x_i  (x_j is gathered, unused)
        seg = tgt_of
        if use_beta:
            # code/Ob_propagation.py:161-186
            T = p_t.shape[0]
            E = x_tgt.shape[0]
            lifted = self.increase_dim(x_tgt).view(E, T, 32)
            node_code = self.map_weights[tgt_of][:, None, :].expand(E, T, 16)
            time_code = p_t[None, :, :].expand(E, T, 16)
            beta = (lifted * torch.cat([node_code, time_code], -1)).mean(-1)        # [E, T]
            gamma = torch.repeat_interleave(beta * edge_w[:, None], self.ob_dim, dim=-1)  # [E, C]
            keep = torch.argsort(gamma.mean(1), descending=True)[: int(E * 0.5)]
            gamma = gamma[keep]
            edge_index = edge_index[:, keep]
            seg = edge_index[0]                               # NB: regrouped by SOURCE (:183)
            x_tgt = x_tgt[keep]
            alpha_ret = gamma.mean(-1)
        else:
            gamma = edge_w[:, None]                           # :187
            alpha_ret = gamma                                 # pre-softmax (:193)
        gamma = segment_softmax(gamma, seg, n)                # :195
        msg = F.relu(self.lin_value(x_tgt)) * gamma           # :200,208-210  (per-edge GEMM)
        out = scatter_rows(msg, seg, n)                       # :226-228
        return out, (edge_index, alpha_ret)

    def forward_dense(self, x, node_scale, gate=None):
        """Live path (use_beta=False) closed form for a batch of node rows x [..., C]; `gate`: relu_or_gate."""
        return relu_or_gate(self.lin_value(x), gate) * node_scale


# --------------------------------------------------------------------------------------------
# TransformerConv (code/transformer_conv.py)
# --------------------------------------------------------------------------------------------
class TransformerConvOracle(nn.Module):
    """heads*out concat variant, no edge features, no beta gate (code/transformer_conv.py:105-124
    with the constructor arguments used at code/models_rd.py:87)."""

    def __init__(self, in_channels, out_channels, heads=1):
        super().__init__()
        self.heads, self.out_channels = heads, out_channels
        self.lin_key = nn.Linear(in_channels, heads * out_channels)
        self.lin_query = nn.Linear(in_channels, heads * out_channels)
        self.lin_value = nn.Linear(in_channels, heads * out_channels)
        self.lin_skip = nn.Linear(in_channels, heads * out_channels)

    def forward(self, x, edge_index, edge_w=None):
        """x [nodes, in] -> (out [nodes, H*F], alpha [E, H]); code/transformer_conv.py:139-207."""
        H, Fo = self.heads, self.out_channels
        n = x.shape[0]
        src_of, tgt_of = edge_index[0], edge_index[1]
        q = self.lin_query(x.index_select(0, tgt_of)).view(-1, H, Fo)      # :189
        k = self.lin_key(x.index_select(0, src_of)).view(-1, H, Fo)        # :190
        logit = (q * k).sum(-1) / math.sqrt(Fo)                            # :198
        if edge_w is not None:
            logit = edge_w[:, None]                                        # :199-200
        alpha = segment_softmax(logit, tgt_of, n)                          # :201
        v = self.lin_value(x.index_select(0, src_of)).view(-1, H, Fo)      # :205
        out = scatter_rows(v * alpha.view(-1, alpha.shape[1], 1), tgt_of, n).reshape(n, -1)
        out = out + self.lin_skip(x)                                       # :168-175
        return out, alpha


# --------------------------------------------------------------------------------------------
# Positional encoding (code/models_rd.py:28-43)
# --------------------------------------------------------------------------------------------
def pe_timescales(max_len, d_pe=16):
    """fp64 numpy, cast to fp32 by torch.Tensor(...) at code/models_rd.py:31,34."""
    return (max_len ** np.linspace(0, 1, d_pe // 2)).astype(np.float32)


def positional_encoding(times, max_len, d_pe=16):
    ts = torch.from_numpy(pe_timescales(max_len, d_pe)).to(times)
    scaled = times[:, :, None] / ts[None, None, :]
    return torch.cat([torch.sin(scaled), torch.cos(scaled)], -1)


# --------------------------------------------------------------------------------------------
# Transformer encoder layer written out (torch.nn.TransformerEncoderLayer, post-LN, relu)
# --------------------------------------------------------------------------------------------
def relu_or_gate(x, gate=None):
    """relu(x), or with `gate` (bool, x's shape) the ReLU whose on/off decisions are given: x where gate, else 0.  With
    gate = x > 0 this is relu bitwise, forward and backward."""
    if gate is None:
        return F.relu(x)
    return torch.where(torch.as_tensor(gate, device=x.device).reshape(x.shape), x, x.new_zeros(()))


def encoder_layer_explicit(x, pad, p, nhead, eps=1e-5, masks=None, ffn_pre=None, ffn_gate=None):
    """x [T, B, D]; pad [B, T] bool (True = padded key); p = dict of the layer's tensors with the
    state-dict suffixes as keys.  Eval-mode math of the module called at code/models_rd.py:358.

    `masks` (optional) = dict of dropout multipliers (0 or 1/(1-p)), each optional, applied where the module's
    dropouts sit in training: "attn" [B, H, T, T] (query, key) on the attention weights after the softmax,
    "resid1" [T*B, D] on the out-projection (dropout1), "ffn" [T*B, nhid] on relu(linear1) (dropout) and
    "resid2" [T*B, D] on linear2 (dropout2).  Train-mode math with those masks instead of torch's RNG.
    `ffn_pre` (optional list): the linear1 pre-activation [T, B, nhid] (the FFN's ReLU input) is appended to it.
    `ffn_gate` (optional, bool [T*B, nhid]): the FFN ReLU's decisions (relu_or_gate)."""
    T, B, D = x.shape
    hd = D // nhead
    m = masks or {}

    def drop(t, key):
        mk = m.get(key)
        return t if mk is None else t * torch.as_tensor(mk, dtype=t.dtype, device=t.device).reshape(t.shape)

    qkv = x @ p["self_attn.in_proj_weight"].T + p["self_attn.in_proj_bias"]
    q, k, v = qkv.split(D, dim=-1)

    def heads(t):  # [T, B, D] -> [B, H, T, hd]
        return t.reshape(T, B, nhead, hd).permute(1, 2, 0, 3)

    s = (heads(q) / math.sqrt(hd)) @ heads(k).transpose(-1, -2)
    s = s.masked_fill(pad[:, None, None, :], -math.inf)
    a = drop(torch.softmax(s, -1), "attn")
    o = (a @ heads(v)).permute(2, 0, 1, 3).reshape(T, B, D)
    y = drop(o @ p["self_attn.out_proj.weight"].T + p["self_attn.out_proj.bias"], "resid1")
    x1 = F.layer_norm(x + y, (D,), p["norm1.weight"], p["norm1.bias"], eps)
    f_pre = x1 @ p["linear1.weight"].T + p["linear1.bias"]
    if ffn_pre is not None:
        ffn_pre.append(f_pre.detach())
    f = drop(relu_or_gate(f_pre, ffn_gate), "ffn")
    g = drop(f @ p["linear2.weight"].T + p["linear2.bias"], "resid2")
    return F.layer_norm(x1 + g, (D,), p["norm2.weight"], p["norm2.bias"], eps)


def encoder_head_oracle(z0, static, lengths, params, nhead, eps=1e-5, masks=None, gates=None, stages=None, encoder=None):
    """Temporal encoder + masked mean + head on a given encoder input: code/models_rd.py:354-385 (Raindrop_v2) and
    :168-189 (legacy v1), what rd_encoder_head_fwd computes.

    z0 [T, B, D] (any D = features + positional encoding); lengths [B]; static [B, d_static] or None (no emb branch);
    params: state-dict keys -> tensors, "transformer_encoder.layers.<l>.<suffix>" (encoder_layer_explicit's suffixes;
    the layer count is read from them), "emb.weight" [emb_dim, d_static] / "emb.bias" (any emb_dim) and
    "mlp_static.{0,2}.{weight,bias}".  Post-LN layers with key-padding mask, pooled = sum of the valid rows /
    (lengths + 1), cat emb(static), mlp_static written out (Linear, ReLU, Linear).
    `masks`: one encoder_layer_explicit mask dict per layer (train mode with given dropout masks), or None (eval).
    `gates` (optional dict, bool): "ffn" [[T*B, nhid]] * nlayers and "head" [B, Df], the ReLU decisions (relu_or_gate).
    `stages` (optional dict) receives "enc" (the encoder output [T, B, D]), "ffn_pre" (one [T, B, nhid] linear1 output
    per layer; empty when `encoder` is given) and "head_pre" (mlp_static.0 output [B, Df]).
    `encoder` (optional callable (z0, pad) -> output) replaces the written-out layers, e.g. by the torch module."""
    T, B = z0.shape[0], z0.shape[1]
    g = gates or {}
    pad = torch.arange(T, device=z0.device)[None, :] >= lengths.to(z0.device)[:, None]          # [B, T], True = padded
    ffn_pre = []
    if encoder is not None:
        r = encoder(z0, pad)
    else:
        pre = "transformer_encoder.layers."
        L = 1 + max(int(k[len(pre):].split(".")[0]) for k in params if k.startswith(pre))
        masks = masks or [None] * L
        ffn_gates = g.get("ffn") or [None] * L
        assert len(masks) == L and len(ffn_gates) == L, (len(masks), len(ffn_gates), L)
        r = z0
        for l in range(L):
            lp = "%s%d." % (pre, l)
            p = {k[len(lp):]: v for k, v in params.items() if k.startswith(lp)}
            r = encoder_layer_explicit(r, pad, p, nhead, eps, masks[l], ffn_pre, ffn_gates[l])
    keep = (~pad).T[:, :, None].to(r.dtype)                                                        # [T, B, 1]
    pooled = (r * keep).sum(0) / (lengths.to(z0.device)[:, None] + 1)
    if static is not None:
        pooled = torch.cat([pooled, F.linear(static, params["emb.weight"], params["emb.bias"])], dim=1)
    h = F.linear(pooled, params["mlp_static.0.weight"], params["mlp_static.0.bias"])
    if stages is not None:
        stages.update(enc=r, ffn_pre=ffn_pre, head_pre=h.detach())
    return F.linear(relu_or_gate(h, g.get("head")), params["mlp_static.2.weight"], params["mlp_static.2.bias"])


# --------------------------------------------------------------------------------------------
# Raindrop_v2 (code/models_rd.py:194-387)
# --------------------------------------------------------------------------------------------
class RaindropV2Oracle(nn.Module):
    """Same constructor arguments, registered parameters and state-dict keys as the reference
    class; `sensor_wise_mask=True` is not restated (it raises a shape error in the reference)."""

    def __init__(self, d_inp=36, d_model=64, nhead=4, nhid=128, nlayers=2, dropout=0.3, max_len=215,
                 d_static=9, MAX=100, perc=0.5, aggreg="mean", n_classes=2, global_structure=None,
                 sensor_wise_mask=False, static=True):
        super().__init__()
        assert not sensor_wise_mask and aggreg == "mean"
        self.d_inp, self.d_model, self.max_len, self.static = d_inp, d_model, max_len, static
        self.nhead, self.nlayers = nhead, nlayers
        self.global_structure = global_structure
        self.d_ob = int(d_model / d_inp)
        d_pe = 16
        # module creation order = code/models_rd.py:224-264 (keeps seeded inits aligned)
        if static:
            self.emb = nn.Linear(d_static, d_inp)
        self.encoder = nn.Linear(d_inp * self.d_ob, d_inp * self.d_ob)
        layer = nn.TransformerEncoderLayer(d_model + d_pe, nhead, nhid, dropout)
        self.transformer_encoder = nn.TransformerEncoder(layer, nlayers)
        self.R_u = torch.empty(1, d_inp * self.d_ob)          # plain tensor, NOT a parameter (:241)
        C = max_len * self.d_ob
        self.ob_propagation = ObPropOracle(C, d_inp, self.d_ob)
        self.ob_propagation_layer2 = ObPropOracle(C, d_inp, self.d_ob)
        d_final = d_model + d_pe + (d_inp if static else 0)
        self.mlp_static = nn.Sequential(nn.Linear(d_final, d_final), nn.ReLU(), nn.Linear(d_final, n_classes))
        self.mlp = nn.Sequential(nn.Linear(d_model, d_model), nn.ReLU(), nn.Linear(d_model, n_classes))
        self.dropout = nn.Dropout(dropout)
        # init_weights(), code/models_rd.py:270-276
        with torch.no_grad():
            self.encoder.weight.uniform_(-1e-10, 1e-10)
            if static:
                self.emb.weight.uniform_(-1e-10, 1e-10)
        glorot_(self.R_u)

    # -- pieces shared by both evaluation modes ------------------------------------------------
    def _lift(self, src, mask=None):
        """code/models_rd.py:285-296: drop the mask half, repeat each sensor d_ob times, scale by
        R_u, relu, dropout (or the given [T, B, N*d_ob] dropout multipliers in its place)."""
        vals = src[:, :, : src.shape[2] // 2]
        h = F.relu(torch.repeat_interleave(vals, self.d_ob, dim=-1) * self.R_u.to(src))   # R_u: not moved by .to()
        if mask is not None:
            return h * torch.as_tensor(mask, dtype=h.dtype, device=h.device).reshape(h.shape)
        return self.dropout(h)

    def _graph(self):
        gs = self.global_structure
        if gs is None:
            gs = torch.ones(self.d_inp, self.d_inp)
        return graph_from_adjacency(gs.float())

    def _tail(self, obs, pe, static, lengths, layer_masks=None, ffn_pre=None, gates=None, head_pre=None):
        """code/models_rd.py:354-385: concat PE, temporal self-attention, masked mean, head (encoder_head_oracle).
        Without `layer_masks` the encoder is the torch module itself; with them (one encoder_layer_explicit mask dict
        per layer) the layers run written out, with those dropout masks, and append their FFN pre-activations to
        `ffn_pre` (a list) when one is given.  `gates` (forward_dense) gives the decisions of the FFN ("ffn",
        written-out layers only) and head ("head") ReLUs; the head's pre-activation is appended to `head_pre` (a list)
        when one is given.  The key-padding mask is built from `lengths`."""
        g = gates or {}
        encoder = None
        if layer_masks is None:
            assert g.get("ffn") is None, "FFN gates need the written-out layers (masks)"
            encoder = lambda z, pad_: self.transformer_encoder(z, src_key_padding_mask=pad_)
        else:
            assert len(layer_masks) == self.nlayers, (len(layer_masks), self.nlayers)
        st = {}
        logits = encoder_head_oracle(torch.cat([obs, pe], dim=2), static, lengths, dict(self.named_parameters()),
                                     self.nhead, self.transformer_encoder.layers[0].norm1.eps, layer_masks, g, st,
                                     encoder=encoder)
        if ffn_pre is not None:
            ffn_pre.extend(st["ffn_pre"])
        if head_pre is not None:
            head_pre.append(st["head_pre"])
        return logits, st["enc"]

    # -- the reference's own structure (what cpu_baseline times) ---------------------------------
    def forward(self, src, static, times, lengths, use_beta=False, stages=None):
        T, B = src.shape[0], src.shape[1]
        N, d_ob = self.d_inp, self.d_ob
        h = self._lift(src)
        pe = positional_encoding(times, self.max_len).to(src.dtype)
        edge_index, edge_w = self._graph()
        edge_w = edge_w.to(src.dtype)
        obs = torch.zeros(T, B, N * d_ob, dtype=src.dtype)
        n_alpha = edge_index.shape[1] // 2 if use_beta else edge_index.shape[1]
        alpha_all = torch.zeros(n_alpha, B, dtype=src.dtype)
        for b in range(B):                                                # :322-343
            x = h[:, b, :].reshape(T, N, d_ob).permute(1, 0, 2).reshape(N, T * d_ob)
            x, (ei2, a1) = self.ob_propagation(x, pe[:, b, :], edge_index, edge_w, use_beta=use_beta)
            a1 = a1.reshape(-1)
            x, (_, a2) = self.ob_propagation_layer2(x, pe[:, b, :], ei2, a1, use_beta=False)
            obs[:, b, :] = x.view(N, T, d_ob).permute(1, 0, 2).reshape(T, N * d_ob)
            alpha_all[:, b] = a2.reshape(-1)
        distance = torch.cdist(alpha_all.T, alpha_all.T, p=2).mean()      # :345-346
        logits, r = self._tail(obs, pe, static, lengths)
        if stages is not None:
            stages.update(lift=h, pe=pe, obs=obs, enc=r, alpha_all=alpha_all)
        return logits, distance, None

    # -- independent closed form -----------------------------------------------------------------
    def forward_dense(self, src, static, times, lengths, stages=None, tf32_model=False, masks=None, gates=None,
                      h1_value=None):
        """`masks` (optional, oracle/dropout_masks.model_masks layout): {"lift": [T, B, N*d_ob], "layers": [one
        encoder_layer_explicit mask dict per layer]} replace every dropout of the training forward, so that the
        train-mode output and its autograd gradient are those of the given masks (run in float64 for an exact
        reference).  Without masks the modules' own dropout applies (identity in eval).

        `gates` (optional dict, every entry optional, bool) replaces the on/off decisions of the ReLUs a rounding error
        can flip by given ones (relu_or_gate), so that the output is a smooth function of the inputs and parameters
        around the decisions another implementation took:
          "h1"   [B, N, C]            ob-prop layer 1
          "obs"  [T, B, N*d_ob]       ob-prop layer 2, in the layout of its output `obs`
          "ffn"  [[T*B, nhid]] * nlayers, the FFN of each encoder layer (needs masks: the written-out layers)
          "head" [B, Df]              mlp_static.0
        The lift's ReLU has none: the sign of src * R_u is exact in fp32.

        `h1_value` (tf32_model only, [B, N, C]): the TF32-rounded layer-1 output another implementation computed.  Layer
        2 takes its value; the gradient flows on into layer 1 as if it were the model's own.  A rounding that lands on
        the other side of a TF32 rounding boundary then cannot move layer 2.  `stages["h1_own"]` keeps the model's own
        layer-1 output, so that the value fed in can itself be checked.

        `stages` also receives the ReLU inputs: "obprop_pre" (the two ob-prop layers' lin_value outputs [B, N, C]),
        "head_pre" [B, Df] and, with masks, "ffn_pre" (one [T, B, nhid] linear1 output per encoder layer).

        Runs on the device and in the dtype of `src` (the model's parameters must be there too)."""
        T, B = src.shape[0], src.shape[1]
        N, d_ob = self.d_inp, self.d_ob
        g = gates or {}
        h = self._lift(src, None if masks is None else masks["lift"])
        pe = positional_encoding(times, self.max_len).to(src.dtype)
        lengths = lengths.to(src.device)
        edge_index, edge_w = self._graph()
        s = node_scale_from_graph(edge_index, edge_w, N, src.dtype).to(src.device)[None, :, None]   # [1, N, 1]
        x = h.reshape(T, B, N, d_ob).permute(1, 2, 0, 3).reshape(B, N, T * d_ob)
        gate2 = g.get("obs")
        if gate2 is not None:       # obs layout [T, B, N*d_ob] -> ob-prop rows [B, N, C]
            gate2 = torch.as_tensor(gate2, device=src.device).reshape(T, B, N, d_ob).permute(1, 2, 0, 3).reshape(B, N, -1)
        l1, l2 = self.ob_propagation.lin_value, self.ob_propagation_layer2.lin_value
        if tf32_model:
            rows = x.reshape(B * N, T * d_ob)
            gr = lambda t: None if t is None else torch.as_tensor(t, device=src.device).reshape(B * N, -1)
            h1, h2, h1_own = obprop_two_layers_tf32(rows, self.ob_propagation, self.ob_propagation_layer2,
                                            s.expand(B, N, 1).reshape(B * N, 1), gr(g.get("h1")), gr(gate2),
                                            None if h1_value is None else h1_value.to(src).reshape(B * N, -1))
            h1, h2, h1_own = h1.view(B, N, -1), h2.view(B, N, -1), h1_own.view(B, N, -1)
            # ReLU inputs as the rounding model computes them
            pre = lambda lin, t: round_tf32(t) @ round_tf32(lin.weight).T + lin.bias
            l1, l2 = (lambda t: pre(self.ob_propagation.lin_value, t)), (lambda t: pre(self.ob_propagation_layer2.lin_value, t))
        else:
            h1 = self.ob_propagation.forward_dense(x, s, g.get("h1"))
            h2 = self.ob_propagation_layer2.forward_dense(h1, s, gate2)
            h1_own = h1
        obs = h2.view(B, N, T, d_ob).permute(2, 0, 1, 3).reshape(T, B, N * d_ob)
        ffn_pre = [] if stages is not None and masks is not None else None
        head_pre = [] if stages is not None else None
        logits, r = self._tail(obs, pe, static, lengths, None if masks is None else masks["layers"], ffn_pre, g,
                               head_pre)
        if stages is not None:
            with torch.no_grad():
                obprop_pre = [l1(x), l2(h1)]
            stages.update(lift=h, pe=pe, x0=x, h1=h1, h1_own=h1_own.detach(), obs=obs, enc=r, obprop_pre=obprop_pre,
                          head_pre=head_pre[0])
            if ffn_pre is not None:
                stages["ffn_pre"] = ffn_pre
        return logits, torch.zeros((), dtype=src.dtype, device=src.device), None


# --------------------------------------------------------------------------------------------
# Precision model of the CUDA path (NOT part of the reference): the tensor-core observation
# propagation kernels take TF32 operands.  `forward_dense(..., tf32_model=True)` rounds exactly what
# the kernels round (lifted input, both lin_value weights, the layer-1 output; in backward the
# layer-2 output gradient and W2) and keeps everything else fp32, so that the CUDA gradients can be
# checked tightly even though a ReLU network's gradient is discontinuous in forward perturbations.
# --------------------------------------------------------------------------------------------
def round_tf32(t):
    """Round-to-nearest (ties away) to 10 explicit mantissa bits, like cvt.rna.tf32.f32.  A float64 value is first
    rounded to fp32, as the kernels hold it, and the result is returned in t's dtype."""
    i = t.detach().float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype)


class _RoundSTE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return round_tf32(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _LinearTF32(torch.autograd.Function):
    """y = x . rn(W)^T + b for an already-rounded x; dX = rn(dY) . rn(W) when `round_dy`."""

    @staticmethod
    def forward(ctx, x, W, b, round_dy):
        Wr = round_tf32(W)
        ctx.save_for_backward(x, Wr)
        ctx.round_dy = round_dy
        return x @ Wr.T + b

    @staticmethod
    def backward(ctx, dy):
        x, Wr = ctx.saved_tensors
        dyr = round_tf32(dy) if ctx.round_dy else dy
        return dyr @ Wr, dyr.T @ x, dyr.sum(0), None


def obprop_two_layers_tf32(x, layer1, layer2, s, gate1=None, gate2=None, h1_value=None):
    """x [rows, C] -> (h1, h2, h1_own) with the kernels' rounding points (see above); fp32 or float64 between them.
    gate1 / gate2 (bool [rows, C], optional): the two ReLUs' decisions (relu_or_gate); h1_value: see forward_dense.
    h1_own is the model's own layer-1 output, h1 the one layer 2 took."""
    x = _RoundSTE.apply(x)
    h1 = h1_own = _RoundSTE.apply(relu_or_gate(_LinearTF32.apply(x, layer1.lin_value.weight, layer1.lin_value.bias, False),
                                               gate1) * s)
    if h1_value is not None:
        h1 = h1 + (h1_value - h1).detach()
    h2 = relu_or_gate(_LinearTF32.apply(h1, layer2.lin_value.weight, layer2.lin_value.bias, True), gate2) * s
    return h1, h2, h1_own


def dense_train_chunked(model, batch, masks=None, gates=None, chunk=None, tf32_model=False, input_grads=False,
                        on_chunk=None, h1_value=None):
    """Cross-entropy (mean over the batch) and its gradients through `forward_dense`, evaluated `chunk` samples at a
    time on the device and in the dtype of the model's parameters, so that a full-size batch fits in a bounded amount
    of memory.  Each chunk contributes sum(CE) / B; the parameter gradients accumulate in the parameters' .grad (their
    dtype).  `masks` (dropout_masks.model_masks layout) and `gates` (forward_dense layout) cover the whole batch and are
    sliced per chunk, as is `h1_value` [B, N, C] (forward_dense).  on_chunk(sl, stages, logits) sees each chunk's
    stages before they are dropped.

    Returns {"logits" [B, classes], "loss", and with input_grads "d_src", "d_times", "d_static"}."""
    from oracle.dropout_masks import slice_masks
    p0 = next(model.parameters())
    dev, dt = p0.device, p0.dtype
    T, B = batch["src"].shape[0], batch["src"].shape[1]
    chunk = B if chunk is None else int(chunk)
    model.zero_grad(set_to_none=True)
    logits_all, loss, grads_in = [], 0.0, {"d_src": [], "d_times": [], "d_static": []}
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        Bc = sl.stop - sl.start
        src = batch["src"][:, sl].to(dev, dt).requires_grad_(input_grads)
        times = batch["times"][:, sl].to(dev, dt).requires_grad_(input_grads)
        static = None if batch["static"] is None else batch["static"][sl].to(dev, dt).requires_grad_(input_grads)
        g = None
        if gates is not None:
            g = {}
            for k, v in gates.items():
                if v is None:
                    continue
                if k == "ffn":
                    g[k] = [f.reshape(T, B, -1)[:, sl].reshape(T * Bc, -1) for f in v]
                elif k == "obs":
                    g[k] = v[:, sl]
                else:
                    g[k] = v[sl]
        stages = {} if on_chunk is not None else None
        logits, _, _ = model.forward_dense(src, static, times, batch["lengths"][sl], stages=stages, tf32_model=tf32_model,
                                           masks=None if masks is None else slice_masks(masks, sl, T, B), gates=g,
                                           h1_value=None if h1_value is None else h1_value[sl])
        part = F.cross_entropy(logits, batch["y"][sl].to(dev), reduction="sum") / B
        part.backward()
        loss += part.item()
        logits_all.append(logits.detach())
        if input_grads:
            grads_in["d_src"].append(src.grad)
            grads_in["d_times"].append(times.grad)
            grads_in["d_static"].append(None if static is None else static.grad)
        if on_chunk is not None:
            on_chunk(sl, stages, logits.detach())
        del logits, part, stages
    out = dict(logits=torch.cat(logits_all), loss=loss)
    if input_grads:
        out.update(d_src=torch.cat(grads_in["d_src"], 1), d_times=torch.cat(grads_in["d_times"], 1),
                   d_static=None if batch["static"] is None else torch.cat(grads_in["d_static"]))
    return out


def build_oracle_model(cfg, seed=1):
    """Constructs the oracle with the positional-argument convention of code/Raindrop.py:245-251."""
    torch.manual_seed(seed)
    gs = cfg.get("global_structure")
    gs = torch.ones(cfg["d_inp"], cfg["d_inp"]) if gs is None else gs.clone()
    return RaindropV2Oracle(cfg["d_inp"], cfg["d_inp"] * cfg["d_ob"], cfg["nhead"], cfg["nhid"],
                            cfg["nlayers"], cfg["dropout"], cfg["max_len"], cfg["d_static"],
                            cfg.get("MAX", 100), 0.5, "mean", cfg["n_classes"], gs,
                            sensor_wise_mask=False, static=cfg.get("static", True))
