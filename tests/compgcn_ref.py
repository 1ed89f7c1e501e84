"""fp64 torch restatement of CogDL's CompGCNLayer (cogdl/models/nn/compgcn.py:94-151), shared by the CPU golden test,
the GPU parity tests and the reference-package check.  Differentiable in every input (plain autograd, exact in fp64).
"""
import torch


def compgcn_aggregate_fp64(row, col, etype, x, rel, opn):
    """(agg_in, agg_out) [N, F]: for half h (COO edges [0, E // 2) and [E // 2, E) in the order given),
    agg_h[i] = sum_{e in h, row_e = i} phi(x[col_e], rel[t_e]) / deg_h(i), phi = x - r (sub) or x * r (mult)."""
    dev = x.device
    row, col, etype = (torch.as_tensor(t).long().reshape(-1).to(dev) for t in (row, col, etype))
    x, rel = x.double(), rel.double()
    N, E = x.shape[0], row.numel()
    outs = []
    for sl in (slice(0, E // 2), slice(E // 2, E)):
        r, c, t = row[sl], col[sl], etype[sl]
        deg = torch.bincount(r, minlength=N).double()
        phi = x[c] - rel[t] if opn == "sub" else x[c] * rel[t]
        outs.append(torch.zeros(N, x.shape[1], dtype=torch.float64, device=dev).index_add(0, r, phi / deg[r, None]))
    return outs[0], outs[1]


def compgcn_layer_fp64(p, row, col, etype, x, rel_embed, opn, activation=torch.tanh, eps=1e-5):
    """CompGCNLayer.forward with dropout 0 and BatchNorm in training mode (batch statistics, biased variance).
    p: the layer's parameters by state_dict name (weight_in / _out / _rel / _loop, loop_rel, bias or None, bn.weight,
    bn.bias and, with bases, basis_weight.alpha / .weight).  Returns (node output [N, F_out], relation output)."""
    if "basis_weight.alpha" in p:
        rel_embed = p["basis_weight.alpha"] @ p["basis_weight.weight"]
    R = torch.cat((rel_embed, p["loop_rel"]), dim=0)
    agg_in, agg_out = compgcn_aggregate_fp64(row, col, etype, x, R, opn)
    loop = x - p["loop_rel"] if opn == "sub" else x * p["loop_rel"]
    out = (agg_in @ p["weight_in"] + agg_out @ p["weight_out"] + loop @ p["weight_loop"]) / 3
    if p.get("bias") is not None:
        out = out + p["bias"]
    mean = out.mean(0)
    var = ((out - mean) ** 2).mean(0)
    out = (out - mean) / torch.sqrt(var + eps) * p["bn.weight"] + p["bn.bias"]
    return activation(out), (R @ p["weight_rel"])[:-1]
