"""Register the sm_90a backend inside an importable `cogdl` package (the drop-in step).

Plug-in point (SURVEY 8b): the module-global dict `cogdl.utils.spmm_utils.CONFIGS` and the
`cogdl.operators.*` module attributes; layer modules capture the callables at construction
(SpMM.__init__ cogdl/utils/spmm_utils.py:131, EdgeSoftmax.__init__ :195, MultiHeadSpMM.__init__
:234-235, MaxAggregator.__init__ cogdl/layers/sage_layer.py:22-25), so call install() BEFORE
building models.

Every change install() makes goes through one primitive, _rebind(feature, owner, name, new): owner is an object
(a class or module, set with setattr) or a dict (sys.modules, CONFIGS).  It records (feature, owner, name, old) in
one undo log, old being _MISSING when owner had no such name of its own, and does nothing when owner.name already
is new: that is what makes a repeated install() a no-op.  A function of this module that it puts in place is
marked with the attribute _cogdl_b200 (True), so a caller can tell it from the reference's; install() never reads
the mark.  A replacement that falls back to the original finds it at owner._cogdl_b200_original_<name>, set (and
logged) by the same call, and read at call time, so assigning it routes the fallback elsewhere.  uninstall_<flag>() replays that flag's records newest first, uninstall() the whole log.

The base step (always) fills CONFIGS and the cogdl.operators.* modules, seeding a module that is not imported yet,
routes the sampler to the device, and, with rebind_dispatch, rebinds every imported cogdl.* module attribute that IS
the reference's spmm / edge_softmax / mh_spmm / fused_gat_op (or SpMM / EdgeSoftmax / MultiHeadSpMM / FusedGATOp
class) to this package's version, which keeps the int32 CSR, hub plan and transpose cached on the graph.  Each flag
is one entry of _FEATURES: the class methods it rebinds, or for correct_smooth, spspmm, actnn and readout a small
installer; what each replacement computes and when it falls back is documented on the replacement.  The Simple-HGN
example's layer is not part of the cogdl package, so install_simple_hgn(conv_cls) takes the class.
"""
import importlib
import sys
import types
from functools import partial

import torch

from .structure import graph_operands, unsupported_operands

_MISSING = object()
_log = []   # (feature, owner, name, old), oldest first


def _put(owner, name, value):
    if isinstance(owner, dict):
        if value is _MISSING:
            owner.pop(name, None)
        else:
            owner[name] = value
    elif value is _MISSING:
        if name in vars(owner):
            delattr(owner, name)
    else:
        setattr(owner, name, value)


def _rebind(feature, owner, name, new, label=None, keep_original=False):
    """owner.name (owner[name] for a dict) = new, logged under feature; nothing when it already is new.  With
    keep_original, the value it replaces also goes to owner._cogdl_b200_original_<name>.  Returns [label] when it
    rebinds and a label is given, else []."""
    own = owner if isinstance(owner, dict) else vars(owner)
    current = own.get(name, _MISSING) if own is owner else getattr(owner, name, _MISSING)
    if current is new:
        return []
    if keep_original:
        _rebind(feature, owner, "_cogdl_b200_original_" + name, current)
    if isinstance(new, types.FunctionType) and new.__module__ == __name__:
        new._cogdl_b200 = True     # tells a caller the name holds one of this module's replacements
    _log.append((feature, owner, name, own.get(name, _MISSING)))
    _put(owner, name, new)
    return [label] if label else []


def _undo(feature=None):
    """Put back what `feature` rebound (everything when None), newest first."""
    for i in reversed(range(len(_log))):
        f, owner, name, old = _log[i]
        if feature is None or f == feature:
            _put(owner, name, old)
            del _log[i]


def _rebind_everywhere(feature, pairs):
    """Rebind every attribute of an imported cogdl.* module that is the first of one of the (original, replacement)
    pairs to the second."""
    by_id = {id(old): new for old, new in pairs}
    patched = []
    for mname, mod in list(sys.modules.items()):
        if mod is None or not (mname == "cogdl" or mname.startswith("cogdl.")):
            continue
        for attr, val in list(vars(mod).items()):
            if id(val) in by_id:
                patched += _rebind(feature, mod, attr, by_id[id(val)], f"{mname}.{attr}")
    return patched


def _rebind_methods(feature, targets):
    """Rebind each (module, class, attribute, replacement) of targets, keeping the original for the fallback."""
    patched = []
    for mname, cname, attr, new in targets:
        cls = getattr(importlib.import_module(mname), cname)
        patched += _rebind(feature, cls, attr, new, f"{mname}.{cname}.{attr}", keep_original=True)
    return patched


_GENCONV_KERNEL_AGGRS = ("softmax_sg", "softmax", "mean", "sum", "max", "powermean")


def genconv_forward(self, graph, x):
    """GENConv.forward (cogdl/layers/deepergcn_layer.py:64-102) with the aggregation in the sm_90a kernels.  The
    message_norm, residual and MLP are the layer's own.  A bias-free EdgeEncoder on fp32 CUDA edge features of at
    most 16 columns that need no gradient is folded into the softmax aggregations (its product with the features is
    formed inside the kernels, so no [nnz, F] edge tensor exists); any other edge encoder runs as the layer's own
    module and its output goes in as the edge term.  Cases without a kernel -- CPU or non-fp32 input, an
    aggregation name GENConv does not define, max / powermean with an edge encoder -- run the original."""
    from .operators.softmax_aggr import genconv_aggregate

    original = type(self)._cogdl_b200_original_forward
    has_edge = self.edge_encoder is not None and graph.edge_attr is not None
    if (not x.is_cuda or x.dtype != torch.float32 or self.aggr not in _GENCONV_KERNEL_AGGRS
            or (has_edge and self.aggr in ("max", "powermean"))):
        return original(self, graph, x)
    st = graph_operands(graph).st
    edge = {}
    if has_edge:
        attr = graph.edge_attr                       # read after graph_operands: in CSR order
        weight = _fused_edge_encoder_weight(self.edge_encoder, attr, x.shape[1])
        if weight is not None:
            edge = {"edge_attr": attr, "edge_weight": weight}
        else:
            edge = {"edge_term": self.edge_encoder(attr)}
    h = genconv_aggregate(st, x, self.aggr, beta=self.beta, eps=self.eps, p=self.p, **edge)
    if self.use_msg_norm:
        h = self.message_norm(x, h)
    if self.residual:
        h = h + x
    return self.mlp(h)


def _fused_edge_encoder_weight(encoder, attr, F):
    """The [F, D] weight of `encoder` when the fused edge-encoder kernels can take it: an EdgeEncoder whose nn.Linear
    has no bias, fp32 CUDA weight and edge features, features that need no gradient, 1 <= D <= 16.  None otherwise
    (BondEncoder, wider or trainable features: the encoder runs as a module)."""
    from cogdl.layers.deepergcn_layer import EdgeEncoder

    from .operators._raw import GENCONV_EDGE_MAX_D

    if type(encoder) is not EdgeEncoder or not isinstance(encoder.nn, torch.nn.Linear) or encoder.nn.bias is not None:
        return None
    w = encoder.nn.weight
    if (attr.dtype != torch.float32 or not attr.is_cuda or attr.requires_grad or attr.dim() != 2
            or not 1 <= attr.shape[1] <= GENCONV_EDGE_MAX_D or w.dtype != torch.float32 or w.device != attr.device
            or w.shape != (F, attr.shape[1])):
        return None
    return w


def disengcn_forward(self, graph, x):
    """DisenGCNLayer.forward (cogdl/layers/disengcn_layer.py:40-91) with the routing in the sm_90a kernels: the
    layer's own weight, bias and activation give h, and cogdl_b200.disen_routing does the per-channel
    normalisation and the iterations.  CPU or non-fp32 input and channel widths without a kernel (d not a power
    of two up to 32, or out_feats not K * d) run the original."""
    from .operators.disen_routing import SUPPORTED_D, disen_routing

    original = type(self)._cogdl_b200_original_forward
    d, K = self.factor_dim, self.K
    if (not x.is_cuda or x.dtype != torch.float32 or self.weight.dtype != torch.float32 or d not in SUPPORTED_D
            or self.weight.shape[1] != K * d):
        return original(self, graph, x)
    h = self.activation(torch.matmul(x, self.weight) + self.bias)
    return disen_routing(graph_operands(graph).st, h, K, self.iterations, self.tau)


def compgcn_forward(self, graph, x, rel_embed):
    """CompGCNLayer.forward (cogdl/models/nn/compgcn.py:94-122) with the two per-edge message passings replaced by
    one cogdl_b200.compgcn_aggregate and two N-row GEMMs (the message is linear in W).  The layer's own weights,
    basis_weight, dropout (called in the reference's order: in, out, loop), BN, bias and activation are used, and
    the graph is read as COO in the order given, never sorted.  CPU or non-fp32 input or weights, and an opn
    other than sub / mult, run the original."""
    import torch.nn.functional as F

    from .operators.comp_aggr import COMPGCN_OPS, compgcn_aggregate

    original = type(self)._cogdl_b200_original_forward
    weights = (self.weight_in, self.weight_out, self.weight_rel, self.weight_loop, self.loop_rel)
    if (not x.is_cuda or x.dtype != torch.float32 or self.opn not in COMPGCN_OPS
            or any(w.dtype != torch.float32 for w in weights)
            or (not self.use_bases and rel_embed.dtype != torch.float32)):
        return original(self, graph, x, rel_embed)
    if self.use_bases:
        rel_embed = self.basis_weight()
    rel_embed = torch.cat((rel_embed, self.loop_rel), dim=0)
    agg_in, agg_out = compgcn_aggregate(graph.edge_index, graph.edge_attr, x, rel_embed, self.opn)
    emb = F.dropout(agg_in @ self.weight_in, p=self.dropout, training=self.training)
    rev_emb = F.dropout(agg_out @ self.weight_out, p=self.dropout, training=self.training)
    loop_emb = F.dropout(self.rel_transform(x, self.loop_rel) @ self.weight_loop, p=self.dropout, training=self.training)
    out = 1 / 3 * (emb + rev_emb + loop_emb)
    if self.bias is not None:
        out += self.bias
    out = self.bn(out)
    return self.activation(out), torch.matmul(rel_embed, self.weight_rel)[:-1]


def gat_forward(self, graph, x):
    """GATLayer.forward (cogdl/layers/gat_layer.py:59-86) with the attention, its dropout and the aggregation in the
    fused sm_90a GAT kernels, for any graph (the backward uses the cached transpose, not is_symmetric()).  The layer's
    own W, a_l, a_r, NaN zeroing, residual, norm and activation are used; the attention dropout is self.dropout.p
    when training and none in eval, drawn in the kernel (a fresh seed from torch's CPU generator per call).  CPU or
    non-fp32 input or weights, and a dropout of 1, run the original."""
    from .utils.spmm_utils import FusedGATFunction

    original = type(self)._cogdl_b200_original_forward
    p = self.dropout.p if self.training else 0.0
    if (not x.is_cuda or x.dtype != torch.float32 or self.W.dtype != torch.float32 or self.a_l.dtype != torch.float32
            or self.a_r.dtype != torch.float32 or p >= 1.0):
        return original(self, graph, x)
    h = torch.matmul(x, self.W).view(-1, self.nhead, self.out_features)
    h[torch.isnan(h)] = 0.0
    h_l = (self.a_l * h).sum(dim=-1)
    h_r = (self.a_r * h).sum(dim=-1)
    out = FusedGATFunction.apply(h_l, h_r, graph_operands(graph).st, None, None, None, self.alpha, h, p, None)
    out = out.view(out.shape[0], -1)
    if self.residual is not None:
        out = out + self.residual(x)
    if self.norm is not None:
        out = self.norm(out)
    if self.act is not None:
        out = self.act(out)
    return out


def gcnii_forward(self, graph, x, init_x):
    """GCNIILayer.forward (cogdl/layers/gcnii_layer.py:24-30) with the propagation `(1 - alpha) * spmm(graph, x) +
    alpha * init_x` in one cogdl_b200.spmm_residual launch, and the identity mapping `beta * linear(s) + (1 - beta) * s`
    folded into the GEMM operand: one addmm with beta * W + (1 - beta) * I, built from the layer's own linear with
    autograd-tracked ops, so d W and d bias come from autograd.  CPU or non-fp32 input or weights, and graphs with a
    dense grb_adj, run the original."""
    from .operators.spmm_residual import spmm_residual

    original = type(self)._cogdl_b200_original_forward
    lin = self.linear
    if (unsupported_operands(graph, x, init_x) is not None or lin.weight.dtype != torch.float32
            or (lin.bias is not None and lin.bias.dtype != torch.float32)):
        return original(self, graph, x, init_x)
    s = spmm_residual(graph, x, init_x, 1 - self.alpha, self.alpha)
    beta = self.beta
    eye = torch.eye(lin.weight.shape[0], dtype=lin.weight.dtype, device=lin.weight.device)
    w = beta * lin.weight + (1 - beta) * eye
    bias = beta * lin.bias if lin.bias is not None else torch.zeros(lin.weight.shape[0], dtype=s.dtype, device=s.device)
    h = torch.addmm(bias, s, w.t())
    if self.residual:
        h = h + x
    return h


def appnp_forward(self, graph):
    """PPNP.forward (cogdl/models/nn/ppnp.py:56-87) for propagation "appnp": the MLP, the edge-weight dropout in the
    reference's order (a seeded run draws the same masks), set_symmetric() as the reference does (so the backward runs
    over the dropped-weight adjacency, not its transpose), then niter cogdl_b200.spmm_residual launches of
    `(1 - alpha) * spmm(graph, preds) + alpha * local_preds`.  "ppnp" (the dense inverse), CPU or non-fp32 features
    or weights, and graphs with a dense grb_adj run the original."""
    import torch.nn.functional as F

    from .operators.spmm_residual import spmm_residual

    original = type(self)._cogdl_b200_original_forward
    x = graph.x
    if (self.propagation != "appnp" or unsupported_operands(graph, x) is not None
            or any(p.dtype != torch.float32 for p in self.nn.parameters())):
        return original(self, graph)
    graph.sym_norm()
    x = F.dropout(x, p=self.dropout, training=self.training)
    local_preds = self.nn.forward(x)
    preds = local_preds
    with graph.local_graph():
        graph.edge_weight = F.dropout(graph.edge_weight, p=self.dropout, training=self.training)
        graph.set_symmetric()
        for _ in range(self.niter):
            preds = spmm_residual(graph, preds, local_preds, 1 - self.alpha, self.alpha)
    return preds


def _correct_smooth_module():
    import cogdl.models.nn.correct_smooth as cs

    return cs


def _scalar(v):
    return isinstance(v, (int, float)) and not isinstance(v, bool)


def outcome_correlation(g, labels, alpha, nprop, post_step, alpha_term=True):
    """outcome_correlation (cogdl/models/nn/correct_smooth.py) with its loop in cogdl_b200.label_propagate, one SpMM
    launch per step, when post_step is one of the reference's two: partial(autoscale_post, lower=, upper=) with number
    bounds (the clamp), or partial(fixed_post, y=labels, nid=) (the reset of the rows nid to labels, as every reference
    call passes y).  Any other post step, CPU or non-fp32 labels, inputs requiring grad under grad mode and graphs with a
    dense grb_adj run the original."""
    import functools

    from .operators.label_prop import label_propagate

    cs = _correct_smooth_module()
    original = cs._cogdl_b200_original_outcome_correlation
    w = getattr(g, "raw_edge_weight", None)
    if (not isinstance(post_step, functools.partial) or post_step.args or not torch.is_tensor(labels)
            or unsupported_operands(g, labels) is not None
            or (torch.is_grad_enabled() and (labels.requires_grad or (w is not None and w.requires_grad)))):
        return original(g, labels, alpha, nprop, post_step, alpha_term)
    kw = post_step.keywords
    if post_step.func is cs.autoscale_post and set(kw) == {"lower", "upper"} and _scalar(kw["lower"]) and _scalar(kw["upper"]):
        return label_propagate(g, labels, alpha, nprop, lower=kw["lower"], upper=kw["upper"], alpha_term=alpha_term)
    if post_step.func is cs.fixed_post and set(kw) == {"y", "nid"} and kw["y"] is labels and torch.is_tensor(kw["nid"]):
        return label_propagate(g, labels, alpha, nprop, pinned=kw["nid"], alpha_term=alpha_term)
    return original(g, labels, alpha, nprop, post_step, alpha_term)


def diffusion(g, x, nhtop, p=1, alpha=0.5):
    """diffusion (cogdl/models/nn/correct_smooth.py) for p == 1: each step `(1 - alpha) * x + alpha * spmm(g, x)` is
    cogdl_b200.spmm_residual(g, x, x, alpha, 1 - alpha) (fp32 addition commutes, so the bits are the same) and
    `x ** 1` is x.  Any other p, CPU or non-fp32 features and graphs with a dense grb_adj run the original."""
    from .operators.spmm_residual import spmm_residual

    original = _correct_smooth_module()._cogdl_b200_original_diffusion
    if p != 1 or unsupported_operands(g, x) is not None:
        return original(g, x, nhtop, p, alpha)
    x = x ** p
    for _ in range(nhtop):
        x = spmm_residual(g, x, x, alpha, 1 - alpha)
    return x


def install_correct_smooth():
    """Rebind cogdl.models.nn.correct_smooth.outcome_correlation and diffusion (resolved as module globals at call
    time by CorrectSmooth.__call__ and CorrectSmoothMLP.forward), keeping the originals on the module."""
    cs = _correct_smooth_module()
    patched = []
    for name, new in (("outcome_correlation", outcome_correlation), ("diffusion", diffusion)):
        patched += _rebind("correct_smooth", cs, name, new, f"cogdl.models.nn.correct_smooth.{name}", keep_original=True)
    return patched


def _gin_unsupported(self, graph, x):
    eps = self.eps
    return (unsupported_operands(graph, x) is not None or not torch.is_tensor(eps) or eps.device != x.device
            or eps.dtype != torch.float32 or eps.numel() != 1 or x.dim() != 2 or x.shape[0] != graph.num_nodes)


def gin_forward(self, graph, x):
    """GINLayer.forward (cogdl/layers/gin_layer.py:34-38) with `(1 + self.eps) * x + spmm(graph, x)` in one
    cogdl_b200.gin_aggregate launch (the backward, d eps included, through its autograd Function); apply_func is the
    layer's own.  CPU or non-fp32 input or eps, and graphs with a dense grb_adj, run the original."""
    from .operators.gin import gin_aggregate

    if _gin_unsupported(self, graph, x):
        return type(self)._cogdl_b200_original_forward(self, graph, x)
    out = gin_aggregate(graph, x, self.eps)
    return self.apply_func(out) if self.apply_func is not None else out


def gine_forward(self, graph, x):
    """GINELayer.forward (cogdl/layers/gine_layer.py:30-38): `out = spmm(graph, x); out += (1 + self.eps) * x` is the
    same sum as GIN's (fp32 addition commutes), so it is one cogdl_b200.gin_aggregate launch; the fallbacks are
    gin_forward's."""
    return gin_forward(self, graph, x)


def grand_rand_prop(self, graph, x):
    """Grand.rand_prop (cogdl/models/nn/grand.py:98-104): the reference's own drop_node (the same torch.bernoulli on the
    CPU generator and `masks.to(device) * x`, so a seeded run draws the same mask; `x * (1 - p)` in eval mode), then the
    order hops in cogdl_b200.random_propagate, one SpMM launch each with the running sum and the final division in its
    store.  CPU or non-fp32 features and graphs with a dense grb_adj run the original."""
    from .operators.grand import random_propagate

    if unsupported_operands(graph, x) is not None or x.dim() != 2 or x.shape[0] != graph.num_nodes:
        return type(self)._cogdl_b200_original_rand_prop(self, graph, x)
    x = self.drop_node(x)
    return random_propagate(graph, x, self.order)


_RGCN_EYE = {}


def rgcn_forward(self, graph, x):
    """RGCNLayer.forward (cogdl/layers/rgcn_layer.py:99-150) computing the relational sum the reference's loop was
    written to compute, sum_t spmm(A_t, x W_t) with W_t = sum_b alpha[t, b] weight[b] and A_t the row-normalised graph
    restricted to the type-t edges, in one cogdl_b200.rgcn_conv (a fan-out aggregation and one GEMM).

    A deliberate divergence from the original: there, `return h_list` sits inside the per-relation loop and the
    SpMM takes the whole graph, so every edge is aggregated with the W_t of the first relation that has edges, whatever
    its type.  Both agree when there is one relation.  As in the original: graph.row_norm() is called (so the
    normalisation runs over all of a row's edges, with the same side effect on the graph), alpha is the identity when
    num_bases >= num_edge_types, and dropout, layer_norm, bias and the self-loop term follow in its order.  The masked
    graphs' padding_self_loops() (weight 0.01), which the original builds and never uses, are not reproduced.  Edge
    types held on the host are moved to x's device (LinkPredictRGCN.loss samples them there).  CPU or
    non-fp32 input or weights, a dense grb_adj, and a regularizer other than basis run the original, the single-relation
    computation above."""
    import torch.nn.functional as F

    from .operators.rgcn import rgcn_conv

    params = [self.weight] + ([self.alpha] if self.alpha is not None else [])
    if (self.regularizer != "basis" or unsupported_operands(graph, x, *params) is not None or x.dim() != 2
            or any(p.device != x.device for p in params)):
        return type(self)._cogdl_b200_original_forward(self, graph, x)
    if self.num_bases < self.num_edge_types:
        coef = self.alpha
    else:
        key = (self.num_edge_types, x.device)
        coef = _RGCN_EYE.get(key)
        if coef is None:
            coef = _RGCN_EYE[key] = torch.eye(self.num_edge_types, dtype=torch.float32, device=x.device)
    etype = graph.edge_attr
    if etype is not None and etype.device != x.device:
        # LinkPredictRGCN.loss builds its graph with host-side types (sampling_edge_uniform), on which building the
        # CSR of a graph on the GPU raises in the original; the types go to the features' device once per graph
        graph.edge_attr = etype.to(x.device)
    graph.row_norm()
    h_result = rgcn_conv(graph, x, coef, self.weight)
    h_result = F.dropout(h_result, p=self.dropout, training=self.training)
    if self.layer_norm is not None:
        h_result = self.layer_norm(h_result)
    if self.bias is not None:
        h_result = h_result + self.bias
    if self.self_loop is not None:
        h_result += F.dropout(torch.matmul(x, self.weight_self_loop), p=self.self_dropout, training=self.training)
    return h_result


def simple_hgn_forward(self, graph, x, res_attn=None):
    """myGATConv.forward of CogDL's Simple-HGN example (examples/simple_hgn/conv.py) with the attention, its dropout,
    the residual-attention blend and the aggregation in cogdl_b200.hgn_attention.  The layer's own feat_drop, x @ W,
    NaN zeroing, h_l / h_r, type table h_e = (a_e * (edge_emb @ W_e)).sum(-1), residual Linear and activation are used,
    so autograd carries d h_e to a_e, W_e and edge_emb.  The attention dropout is self.dropout.p when training.
    Returns (out, attention.detach()), the attention in the graph's CSR edge order.

    Edge types come from graph.edge_type, an attribute that building the CSR does not reorder.  They are read with
    edge_index on entry; when building the CSR reorders the edges (a stable sort by row), the types -- and a given
    res_attn -- are put through the same sort and graph.edge_type is reassigned, so this and every later call sees
    each edge with its own type.  CPU or non-fp32 input or weights, and a dropout of 1, run the original."""
    from .operators.simple_hgn import hgn_attention

    original = type(self)._cogdl_b200_original_forward
    p = self.dropout.p if self.training else 0.0
    weights = (self.W, self.W_e, self.edge_emb, self.a_l, self.a_r, self.a_e)
    if unsupported_operands(graph, x, res_attn, *weights) is not None or p >= 1.0:
        return original(self, graph, x, res_attn)
    row0 = graph.edge_index[0]
    etype = graph.edge_type
    graph_operands(graph)                       # builds the CSR if the graph has none yet
    if graph.edge_index[0] is not row0:
        order = torch.sort(row0, stable=True).indices
        etype = etype[order.to(etype.device)]
        graph.edge_type = etype
        if res_attn is not None:
            res_attn = res_attn[order]
    x = self.feat_drop(x)
    h = torch.matmul(x, self.W).view(-1, self.nhead, self.out_features)
    h[torch.isnan(h)] = 0.0
    e = torch.matmul(self.edge_emb, self.W_e).view(-1, self.nhead, self.edge_feats)
    h_l = (self.a_l * h).sum(dim=-1)
    h_r = (self.a_r * h).sum(dim=-1)
    h_e = (self.a_e * e).sum(dim=-1)
    out, attention = hgn_attention(graph, h, h_l, h_r, h_e, etype, self.leakyrelu.negative_slope, p, res_attn,
                                   self.alpha)
    out = out.view(out.shape[0], -1)
    if self.residual is not None:
        out = out + self.residual(x)
    if self.act is not None:
        out = self.act(out)
    return out, attention.detach()


def install_simple_hgn(conv_cls):
    """Rebind conv_cls.forward (the Simple-HGN example's myGATConv, which is not part of the cogdl package, so the
    caller passes the class) to simple_hgn_forward; the original stays at conv_cls._cogdl_b200_original_forward."""
    return _rebind(("simple_hgn", conv_cls), conv_cls, "forward", simple_hgn_forward,
                   f"{conv_cls.__module__}.{conv_cls.__qualname__}.forward", keep_original=True)


def uninstall_simple_hgn(conv_cls):
    _undo(("simple_hgn", conv_cls))


_READOUT_NAMES = ("batch_sum_pooling", "batch_mean_pooling", "batch_max_pooling")
_POOLING = []   # (original, replacement): built once per process, so every install rebinds the same objects


def _readout_supported(x, batch):
    """A readout the kernels take: x [N, F] fp32 and batch [N] integers, both on the GPU."""
    return (torch.is_tensor(x) and torch.is_tensor(batch) and x.is_cuda and batch.is_cuda and x.dtype == torch.float32
            and x.dim() == 2 and batch.dim() == 1 and x.shape[0] == batch.numel() and not batch.dtype.is_floating_point)


def _pooling(name, original):
    mode = name.split("_")[1]

    def pool(x, batch):
        from .operators.readout import graph_readout

        if not _readout_supported(x, batch):
            return original(x, batch)
        return graph_readout([x], batch, mode)

    pool.__name__ = pool.__qualname__ = name
    pool.__doc__ = (f"cogdl.utils.{name} (cogdl/utils/utils.py) on cogdl_b200.{name}: deterministic, and no host read "
                    "once the batch's membership is cached; B is max(batch) + 1 and a graph id without nodes pools to 0 "
                    "(the original's mean counts only the ids present).  CPU or non-fp32 input runs the original.")
    return pool


def gin_model_forward(self, batch):
    """GIN.forward (cogdl/models/nn/gin.py:95-115) with its per-layer sum pooling (a scatter_add_ per layer after a host
    read of max(batch)) as one cogdl_b200.graph_readout over the layer outputs; the layers, BatchNorm, ReLU, linears and
    dropout are the model's own, called in its order.  CPU or non-fp32 features run the original."""
    import torch.nn.functional as F

    from .operators.readout import graph_readout

    from .structure import membership_for

    h = batch.x
    if not _readout_supported(h, batch.batch):
        return type(self)._cogdl_b200_original_forward(self, batch)
    membership_for(batch.batch)     # a new batch's host reads happen here, before the layers are queued
    layer_rep = [h]
    for i in range(self.num_layers - 1):
        h = F.relu(self.batch_norm[i](self.gin_layers[i](batch, h)))
        layer_rep.append(h)
    pooled = graph_readout(layer_rep, batch.batch, "sum")
    final_score, off = 0, 0
    for i, rep in enumerate(layer_rep):
        final_score += self.dropout(self.linear_prediction[i](pooled[:, off:off + rep.shape[1]]))
        off += rep.shape[1]
    return final_score


def sortpool_forward(self, batch):
    """SortPool.forward (cogdl/models/nn/sortpool.py:105-136) with the padding to [B, max_n, F], the fill value, the
    sort of the padded rows, the cut to k and the zeroing of the fill (two host reads) replaced by cogdl_b200.sort_pool.
    The SAGE layers, the per-row h.sort(dim=-1), conv1d, the linears and dropout are the model's own.  Ties of the last
    channel go to the lower node index (the original's CUDA sort is not stable).  CPU or non-fp32 features and k above
    the kernel's maximum run the original."""
    import torch.nn.functional as F

    from .operators._raw import sort_pool_max_k
    from .operators.readout import sort_pool

    from .structure import membership_for

    h = batch.x
    if not _readout_supported(h, batch.batch) or self.k > sort_pool_max_k():
        return type(self)._cogdl_b200_original_forward(self, batch)
    membership_for(batch.batch)     # a new batch's host reads happen here, before the layers are queued
    for i in range(self.num_layers):
        h = F.relu(self.gnn_convs[i](batch, h))
    h, _ = h.sort(dim=-1)
    h = sort_pool(h, batch.batch, self.k)
    batch_size = h.shape[0]
    h = F.relu(self.conv1d(h.permute(0, 2, 1))).view(batch_size, -1)
    h = F.relu(self.fc1(h))
    h = F.dropout(h, p=self.dropout, training=self.training)
    return self.fc2(h)


def set2set_forward(self, x, batch):
    """Set2Set.forward (cogdl/layers/set2set.py:46-62) with the attention read of every step in
    cogdl_b200.set2set_attention; the LSTM and the concatenation are the layer's own.

    A deliberate divergence from the original, which cannot run: it calls `edge_softmax(e, batch)`, which is
    cogdl.utils.edge_softmax(graph, edge_val) with a tensor for the graph.  This computes what the layer's docstring
    states, a = softmax over graph g's nodes of <x_i, q_g> and r_g = sum_i a_i x_i, with B = max(batch) + 1 and 0 for a
    graph id without nodes.  CPU or non-fp32 input or LSTM weights run the original."""
    from .operators.readout import set2set_attention
    from .structure import membership_for

    if not _readout_supported(x, batch) or any(p.dtype != torch.float32 for p in self.lstm.parameters()):
        return type(self)._cogdl_b200_original_forward(self, x, batch)
    batch_size = membership_for(batch).num_graphs
    h = (x.new_zeros((self.num_layers, batch_size, self.in_channels)),
         x.new_zeros((self.num_layers, batch_size, self.in_channels)))
    q_star = x.new_zeros(batch_size, self.out_channels)
    for _ in range(self.processing_steps):
        q, h = self.lstm(q_star.unsqueeze(0), h)
        q = q.view(batch_size, self.in_channels)
        q_star = torch.cat([q, set2set_attention(x, q, batch)], dim=-1)
    return q_star


def install_readout():
    """Rebind cogdl.utils.batch_{sum,mean,max}_pooling, and every attribute of an imported cogdl.* module bound to them,
    to the cogdl_b200 readouts; GIN.forward to gin_model_forward, SortPool.forward to sortpool_forward and
    Set2Set.forward to set2set_forward.  InfoGraph and GCC take the pooling function when a model is constructed, so
    install before building models."""
    import cogdl.layers.set2set  # noqa: F401  (imported before the scan, so their bindings are rebound too)
    import cogdl.models.nn.gin  # noqa: F401
    import cogdl.models.nn.sortpool  # noqa: F401
    import cogdl.utils.utils as uu

    if not _POOLING:
        _POOLING.extend((getattr(uu, n), _pooling(n, getattr(uu, n))) for n in _READOUT_NAMES)
    return _rebind_everywhere("readout", _POOLING) + _rebind_methods("readout", (
        ("cogdl.models.nn.gin", "GIN", "forward", gin_model_forward),
        ("cogdl.models.nn.sortpool", "SortPool", "forward", sortpool_forward),
        ("cogdl.layers.set2set", "Set2Set", "forward", set2set_forward)))


_SPSPMM_MODULES = ("cogdl.models.nn.gtn", "cogdl.models.nn.srgcn", "cogdl.utils.srgcn_utils", "cogdl.models.nn.graph_unet")


def install_spspmm():
    """torch_sparse's spspmm / spmm for GTN, SRGCN and Graph U-Net.  Without a loadable torch_sparse, a module of that
    name providing exactly those two functions goes into sys.modules, so the models import; an importable torch_sparse
    is left alone.  Either way the two names are rebound in those of the four model modules already imported (models
    imported while the stand-in was there keep their binding after uninstall_spspmm())."""
    from .operators.spspmm import coo_spmm, spspmm

    patched = []
    if "torch_sparse" not in sys.modules:
        try:
            import torch_sparse  # noqa: F401
        except (ImportError, OSError):   # missing, or a binary build that does not load (undefined symbol)
            stub = types.ModuleType("torch_sparse")
            stub.__doc__ = "spspmm and spmm of cogdl_b200, seeded by cogdl_b200.install(spspmm=True)"
            stub.spspmm, stub.spmm = spspmm, coo_spmm
            patched += _rebind("spspmm", sys.modules, "torch_sparse", stub, "torch_sparse")
    for mname in _SPSPMM_MODULES:
        mod = sys.modules.get(mname)
        if mod is None:
            continue
        for attr, new in (("spspmm", spspmm), ("spmm", coo_spmm)):
            if attr == "spmm" and mname != "cogdl.utils.srgcn_utils":
                continue   # srgcn.py's `spmm` is cogdl.utils.spmm (the graph SpMM), not torch_sparse's
            if getattr(mod, attr, None) is not None:
                patched += _rebind("spspmm", mod, attr, new, f"{mname}.{attr}")
    return patched


_ACTNN_SUBMODULES = ("conf", "ops", "qscheme", "qbnscheme", "layers", "utils")
_ACTNN_NAMES = {"cogdl.operators.linear": ("quantize_activation", "dequantize_activation", "config", "empty_cache"),
                "cogdl.operators.spmm": ("quantize_activation", "dequantize_activation")}


def install_actnn():
    """The `actnn` API for CogDL's activation-compressed models.  Without an importable actnn, cogdl_b200.actnn and its
    submodules go into sys.modules as `actnn` and `actnn.<name>`, so the models' imports resolve to them; an importable
    actnn is left alone.  cogdl.operators.linear imports actnn inside a try at import time: if it was imported before,
    its names are bound here.  Modules imported while the stand-in was there keep their binding after
    uninstall_actnn()."""
    from . import actnn as stub

    patched = []
    if "actnn" not in sys.modules:
        try:
            import actnn  # noqa: F401
        except (ImportError, OSError):   # missing, or a binary build that does not load
            patched += _rebind("actnn", sys.modules, "actnn", stub, "actnn")
            for name in _ACTNN_SUBMODULES:
                _rebind("actnn", sys.modules, "actnn." + name, getattr(stub, name))
    actnn_mod = sys.modules["actnn"]
    for mname, attrs in _ACTNN_NAMES.items():
        mod = sys.modules.get(mname)
        if mod is None:
            continue
        for attr in attrs:
            src = actnn_mod.conf if attr == "config" else (actnn_mod.utils if attr == "empty_cache" else actnn_mod.ops)
            patched += _rebind("actnn", mod, attr, getattr(src, attr), f"{mname}.{attr}")
    return patched


def _host_sampler(name):
    """The reference's own host function install() found at cogdl.data.data.<name>, for CPU graphs (no CPU path in
    this package)."""
    import cogdl.data.data as ref_data

    original = getattr(ref_data, "_cogdl_b200_original_" + name)
    if original is None:
        raise RuntimeError("cogdl.operators.sample failed to load and the graph is on the CPU")
    return original


def sample_adj_c(indptr, indices, node_idx, num_neighbors=-1, replace=True):
    """cogdl.data.data.sample_adj_c (what Graph.sample_adj calls, cogdl/data/data.py:792-832; SURVEY 8f-4): CUDA graphs
    go to the device sampler, CPU graphs to the reference's own host function."""
    from . import sampling

    if not indptr.is_cuda:
        return _host_sampler("sample_adj_c")(indptr, indices, node_idx, num_neighbors, replace)
    node_idx = torch.as_tensor(node_idx, dtype=torch.int64).to(indptr.device)
    rp, ci, nodes, edges = sampling.sample_adj(indptr, indices, node_idx, num_neighbors, replace)
    # data.py:818-820 pads row_ptr for the new (edge-less) nodes with a CPU tensor; hand it over padded
    pad = nodes.numel() + 1 - rp.numel()
    if pad > 0:
        rp = torch.cat([rp, rp[-1:].expand(pad)])
    return rp, ci, nodes, edges


def subgraph_c(indptr, indices, node_idx):
    """cogdl.data.data.subgraph_c (what Graph.csr_subgraph calls, cogdl/data/data.py:856-874), routed as sample_adj_c."""
    from . import sampling

    if not indptr.is_cuda:
        return _host_sampler("subgraph_c")(indptr, indices, node_idx)
    return sampling.subgraph(indptr, indices, node_idx.to(indptr.device))


def _install_base(rebind_dispatch):
    import cogdl.utils.spmm_utils as ref_su  # raises ImportError if cogdl is not importable

    from . import operators as ops
    from .utils import spmm_utils as su

    for key, value in {
        "fast_spmm": ops.csrspmm, "csr_edge_softmax": ops.csr_edge_softmax, "csrmhspmm": ops.csrmhspmm,
        "fused_gat_func": ops.fused_gat_func,
        "spmm_flag": True, "mh_spmm_flag": True, "fused_gat_flag": True,
    }.items():
        _rebind("base", ref_su.CONFIGS, key, value)
    import cogdl.operators as ref_ops_pkg

    for mod_name, attrs in (
        ("cogdl.operators.spmm", {"csrspmm": ops.csrspmm}),
        ("cogdl.operators.edge_softmax", {"csr_edge_softmax": ops.csr_edge_softmax}),
        ("cogdl.operators.mhspmm", {"csrmhspmm": ops.csrmhspmm}),
        ("cogdl.operators.scatter_max", {"scatter_max": ops.scatter_max}),
        ("cogdl.operators.fused_gat", {"fused_gat_func": ops.fused_gat_func}),
    ):
        mod = sys.modules.get(mod_name)
        if mod is None:
            # Not imported yet: seed a module that already carries our operator, so a later
            # `from cogdl.operators.scatter_max import scatter_max` (sage_layer.py:23) resolves to it
            # and the reference's import-time JIT build of its own CUDA sources never runs.
            mod = types.ModuleType(mod_name)
            mod.__doc__ = "seeded by cogdl_b200.install()"
            _rebind("base", sys.modules, mod_name, mod)
            _rebind("base", ref_ops_pkg, mod_name.rsplit(".", 1)[1], mod)
        for k, v in attrs.items():
            _rebind("base", mod, k, v)
    import cogdl.data.data as ref_data

    patched = []
    for name, new in (("sample_adj_c", sample_adj_c), ("subgraph_c", subgraph_c)):
        patched += _rebind("base", ref_data, name, new, f"cogdl.data.data.{name}", keep_original=True)
    if rebind_dispatch:
        names = ["spmm", "edge_softmax", "mh_spmm", "fused_gat_op", "check_fused_gat", "SpMM", "EdgeSoftmax",
                 "MultiHeadSpMM", "FusedGATOp"]
        patched += _rebind_everywhere("base", [(getattr(ref_su, n), getattr(su, n)) for n in names if hasattr(ref_su, n)])
    return patched


_FEATURES = {   # install() flag -> the class methods it rebinds (module, class, attribute, replacement) or its
                # installer, in the order install() applies them
    "genconv": (("cogdl.layers.deepergcn_layer", "GENConv", "forward", genconv_forward),),
    "disengcn": (("cogdl.layers.disengcn_layer", "DisenGCNLayer", "forward", disengcn_forward),),
    "compgcn": (("cogdl.models.nn.compgcn", "CompGCNLayer", "forward", compgcn_forward),),
    "spspmm": install_spspmm,
    "gat": (("cogdl.layers.gat_layer", "GATLayer", "forward", gat_forward),),
    "actnn": install_actnn,
    "gcnii": (("cogdl.layers.gcnii_layer", "GCNIILayer", "forward", gcnii_forward),),
    "appnp": (("cogdl.models.nn.ppnp", "PPNP", "forward", appnp_forward),),
    "correct_smooth": install_correct_smooth,
    "gin": (("cogdl.layers.gin_layer", "GINLayer", "forward", gin_forward),
            ("cogdl.layers.gine_layer", "GINELayer", "forward", gine_forward)),
    "grand": (("cogdl.models.nn.grand", "Grand", "rand_prop", grand_rand_prop),),
    "rgcn": (("cogdl.layers.rgcn_layer", "RGCNLayer", "forward", rgcn_forward),),
    "readout": install_readout,
}


def _install(feature):
    how = _FEATURES[feature]
    return how() if callable(how) else _rebind_methods(feature, how)


def install(rebind_dispatch=True, genconv=False, disengcn=False, compgcn=False, spspmm=False, gat=False, actnn=False,
            gcnii=False, appnp=False, correct_smooth=False, gin=False, grand=False, rgcn=False, readout=False):
    """Register the backend in the imported cogdl package, plus each feature whose flag is set; returns the names
    rebound, in the order rebound (a repeated call rebinds nothing and returns [])."""
    flags = locals()    # the keyword arguments, by name
    patched = _install_base(rebind_dispatch)
    for feature in _FEATURES:
        if flags[feature]:
            patched += _install(feature)
    return patched


def uninstall():
    """Put back everything install() and install_simple_hgn() rebound."""
    _undo()


install_genconv, uninstall_genconv = partial(_install, "genconv"), partial(_undo, "genconv")
install_disengcn, uninstall_disengcn = partial(_install, "disengcn"), partial(_undo, "disengcn")
install_compgcn, uninstall_compgcn = partial(_install, "compgcn"), partial(_undo, "compgcn")
install_gat, uninstall_gat = partial(_install, "gat"), partial(_undo, "gat")
install_gcnii, uninstall_gcnii = partial(_install, "gcnii"), partial(_undo, "gcnii")
install_appnp, uninstall_appnp = partial(_install, "appnp"), partial(_undo, "appnp")
install_gin, uninstall_gin = partial(_install, "gin"), partial(_undo, "gin")
install_grand, uninstall_grand = partial(_install, "grand"), partial(_undo, "grand")
install_rgcn, uninstall_rgcn = partial(_install, "rgcn"), partial(_undo, "rgcn")
uninstall_spspmm, uninstall_actnn = partial(_undo, "spspmm"), partial(_undo, "actnn")
uninstall_correct_smooth, uninstall_readout = partial(_undo, "correct_smooth"), partial(_undo, "readout")
