"""install() against the reference package (oracle/_ref/pkg), each case in its own child process: install() rebinds
that package for the rest of a process, and other tests in a session run it on its own CPU path first.

Checked: the names install() returns, for every flag alone and for all of them, pinned; a second call returns [];
install -> uninstall() -> install returns the same names again; uninstall() after install(<flags>) and
uninstall_<flag>() after install() + install(<flag>=True) each give back, object for object, the attributes of every
imported cogdl.* module and of every patched class, sys.modules and CONFIGS; and every rebound method still falls
back through the original that install() keeps at <owner>._cogdl_b200_original_<name>, read at call time.
"""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FLAGS = ("genconv", "disengcn", "compgcn", "spspmm", "gat", "actnn", "gcnii", "appnp", "correct_smooth", "gin", "grand",
         "rgcn", "readout")

# what install() rebinds with no flag: the sampler and the dispatch names of the modules cogdl imports itself
BASE = [
    "cogdl.data.data.sample_adj_c", "cogdl.data.data.subgraph_c",
    "cogdl.utils.spmm_utils.check_fused_gat", "cogdl.utils.spmm_utils.spmm", "cogdl.utils.spmm_utils.SpMM",
    "cogdl.utils.spmm_utils.edge_softmax", "cogdl.utils.spmm_utils.EdgeSoftmax", "cogdl.utils.spmm_utils.mh_spmm",
    "cogdl.utils.spmm_utils.MultiHeadSpMM", "cogdl.utils.spmm_utils.fused_gat_op", "cogdl.utils.spmm_utils.FusedGATOp",
    "cogdl.utils.check_fused_gat", "cogdl.utils.spmm", "cogdl.utils.SpMM", "cogdl.utils.edge_softmax",
    "cogdl.utils.EdgeSoftmax", "cogdl.utils.mh_spmm", "cogdl.utils.MultiHeadSpMM", "cogdl.utils.fused_gat_op",
    "cogdl.utils.FusedGATOp",
]
# what each flag adds after BASE, in a process that has imported nothing of cogdl beyond the package itself
FLAG_NAMES = {
    "genconv": ["cogdl.layers.deepergcn_layer.GENConv.forward"],
    "disengcn": ["cogdl.layers.disengcn_layer.DisenGCNLayer.forward"],
    "compgcn": ["cogdl.models.nn.compgcn.CompGCNLayer.forward"],
    "spspmm": ["torch_sparse"],
    "gat": ["cogdl.layers.gat_layer.GATLayer.forward"],
    "actnn": ["actnn", "cogdl.operators.spmm.quantize_activation", "cogdl.operators.spmm.dequantize_activation"],
    "gcnii": ["cogdl.layers.gcnii_layer.GCNIILayer.forward"],
    "appnp": ["cogdl.models.nn.ppnp.PPNP.forward"],
    "correct_smooth": ["cogdl.models.nn.correct_smooth.outcome_correlation", "cogdl.models.nn.correct_smooth.diffusion"],
    "gin": ["cogdl.layers.gin_layer.GINLayer.forward", "cogdl.layers.gine_layer.GINELayer.forward"],
    "grand": ["cogdl.models.nn.grand.Grand.rand_prop"],
    "rgcn": ["cogdl.layers.rgcn_layer.RGCNLayer.forward"],
    "readout": ["cogdl.utils.utils.batch_sum_pooling", "cogdl.utils.utils.batch_mean_pooling",
                "cogdl.utils.utils.batch_max_pooling", "cogdl.utils.batch_sum_pooling", "cogdl.utils.batch_mean_pooling",
                "cogdl.utils.batch_max_pooling", "cogdl.layers.deepergcn_layer.batch_max_pooling",
                "cogdl.layers.set2set.batch_sum_pooling", "cogdl.models.nn.gin.GIN.forward",
                "cogdl.models.nn.sortpool.SortPool.forward", "cogdl.layers.set2set.Set2Set.forward"],
}

_PRELUDE = """
import importlib, json, sys
from tests.refpkg import import_reference
import_reference()
import torch
import cogdl_b200
import cogdl.utils.spmm_utils as ref_su

CLASSES = [("cogdl.layers.deepergcn_layer", "GENConv"), ("cogdl.layers.disengcn_layer", "DisenGCNLayer"),
           ("cogdl.models.nn.compgcn", "CompGCNLayer"), ("cogdl.layers.gat_layer", "GATLayer"),
           ("cogdl.layers.gcnii_layer", "GCNIILayer"), ("cogdl.models.nn.ppnp", "PPNP"),
           ("cogdl.layers.gin_layer", "GINLayer"), ("cogdl.layers.gine_layer", "GINELayer"),
           ("cogdl.models.nn.grand", "Grand"), ("cogdl.layers.rgcn_layer", "RGCNLayer"), ("cogdl.models.nn.gin", "GIN"),
           ("cogdl.models.nn.sortpool", "SortPool"), ("cogdl.layers.set2set", "Set2Set")]
"""

# The names install(**flags) returns in a fresh process, on a second call, and again after uninstall().
_NAMES = _PRELUDE + """
flags = json.loads(sys.argv[1])
names = [cogdl_b200.install(**flags), cogdl_b200.install(**flags)]
cogdl_b200.uninstall()
names.append(cogdl_b200.install(**flags))
print(json.dumps(names))
"""

# With every module a flag touches imported: uninstall() after install(<every flag>) against the state before it,
# then uninstall_<flag>() after install(<flag>=True) against the state of a bare install(), flag by flag.
_ROUND_TRIP = _PRELUDE + """
def snapshot():
    for m in ("cogdl.operators", "cogdl.models.nn.correct_smooth", "cogdl.utils.utils", "cogdl.data.data") + tuple(
            m for m, _ in CLASSES):
        importlib.import_module(m)
    state = {"sys.modules": {k: v for k, v in sys.modules.items() if not k.startswith("cogdl_b200")},
             "CONFIGS": dict(ref_su.CONFIGS)}
    state.update({k: dict(vars(m)) for k, m in list(sys.modules.items())
                  if m is not None and (k == "cogdl" or k.startswith("cogdl."))})
    state.update({f"{m}.{c}": dict(vars(getattr(sys.modules[m], c))) for m, c in CLASSES})
    return state


def changed(a, b, absent=object()):
    return sorted(f"{k}.{n}" for k in a.keys() | b.keys() for n in a.get(k, {}).keys() | b.get(k, {}).keys()
                  if a.get(k, {}).get(n, absent) is not b.get(k, {}).get(n, absent))


flags = json.loads(sys.argv[1])
before = snapshot()
cogdl_b200.install(**{f: True for f in flags})
cogdl_b200.uninstall()
result = {"uninstall": changed(before, snapshot())}
cogdl_b200.install()
before = snapshot()
for flag in flags:
    cogdl_b200.install(**{flag: True})
    getattr(cogdl_b200, "uninstall_" + flag)()
    result[flag] = changed(before, snapshot())
print(json.dumps(result))
"""

# Every rebound method, fed CPU tensors, calls <owner>._cogdl_b200_original_<name> as it is when called; each, and
# each readout pooling function, carries the _cogdl_b200 mark.
_FALLBACK = _PRELUDE + """
from types import SimpleNamespace

from cogdl.data import Graph

cogdl_b200.install(**{f: True for f in json.loads(sys.argv[1])})
mod = {m: importlib.import_module(m) for m, _ in CLASSES}
cls = {c: getattr(mod[m], c) for m, c in CLASSES}
g = Graph(x=torch.randn(6, 8), edge_index=torch.tensor([[0, 1, 2, 3, 4, 5], [1, 2, 3, 4, 5, 0]]))
x = torch.randn(6, 8)
batch = SimpleNamespace(x=x, batch=torch.tensor([0, 0, 0, 1, 1, 1]))
calls = [
    (cls["GENConv"](8, 8), "forward", (g, x)),
    (cls["DisenGCNLayer"](8, 8, 2, 1), "forward", (g, x)),
    (cls["CompGCNLayer"](8, 8, 2), "forward", (g, x, torch.randn(4, 8))),
    (cls["GATLayer"](8, 8), "forward", (g, x)),
    (cls["GCNIILayer"](8), "forward", (g, x, x)),
    (cls["PPNP"](8, 8, 3, 2, 0.0, "appnp", 0.1, 2), "forward", (g,)),
    (cls["GINLayer"](), "forward", (g, x)),
    (cls["GINELayer"](), "forward", (g, x)),
    (cls["Grand"](8, 8, 3, 0.0, 0.0, False, 0.5, 2, 0.5), "rand_prop", (g, x)),
    (cls["RGCNLayer"](8, 8, 2, num_bases=2), "forward", (g, x)),
    (cls["GIN"](2, 8, 3, 8, 2), "forward", (batch,)),
    (cls["SortPool"](8, 8, 3, 2, 8, 3), "forward", (batch,)),
    (cls["Set2Set"](8, 2), "forward", (x, batch.batch)),
]
cs = importlib.import_module("cogdl.models.nn.correct_smooth")
calls += [(cs, "outcome_correlation", (g, x, 0.5, 2, None)), (cs, "diffusion", (g, x, 2))]
routed = []
for obj, name, args in calls:
    owner = obj if obj is cs else type(obj)
    key = "_cogdl_b200_original_" + name
    original, seen = getattr(owner, key), []
    setattr(owner, key, lambda *a: seen.append(a) or "spy")
    try:
        marked = getattr(getattr(owner, name), "_cogdl_b200", False)
        if marked and getattr(obj, name)(*args) == "spy" and len(seen) == 1:
            routed.append(f"{owner.__name__}.{name}")
    finally:
        setattr(owner, key, original)


class Conv(torch.nn.Module):     # stands in for the Simple-HGN example's layer, which install() cannot import
    def forward(self, graph, x, res_attn=None):
        return x


before = dict(vars(Conv))
rebound = cogdl_b200.install_simple_hgn(Conv) + cogdl_b200.install_simple_hgn(Conv)
cogdl_b200.uninstall_simple_hgn(Conv)
uu = importlib.import_module("cogdl.utils.utils")
routed += [n for n in ("batch_sum_pooling", "batch_mean_pooling", "batch_max_pooling")
           if getattr(getattr(uu, n), "_cogdl_b200", False)]
print(json.dumps({"routed": routed, "simple_hgn": rebound, "simple_hgn_restored": dict(vars(Conv)) == before}))
"""


def _child(code, arg):
    r = subprocess.run([sys.executable, "-c", code, json.dumps(arg)], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def runs():
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.skip("reference package not built (oracle/_ref/pkg)")
    cases = {"all": {f: True for f in FLAGS}, **{f: {f: True} for f in FLAGS}}
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        names = {k: ex.submit(_child, _NAMES, v) for k, v in cases.items()}
        round_trip = ex.submit(_child, _ROUND_TRIP, list(FLAGS))
        fallback = ex.submit(_child, _FALLBACK, list(FLAGS))
        return {k: j.result() for k, j in names.items()}, round_trip.result(), fallback.result()


@pytest.mark.parametrize("case", ("all",) + FLAGS)
def test_install_returns_the_pinned_names(runs, case):
    """Fresh install, second install ([]), install after uninstall()."""
    flags = FLAGS if case == "all" else (case,)
    expected = BASE + [n for f in flags for n in FLAG_NAMES[f]]
    assert runs[0][case] == [expected, [], expected]


@pytest.mark.parametrize("case", ("uninstall",) + FLAGS)
def test_uninstall_gives_back_every_object(runs, case):
    """uninstall() after install(<every flag>), or uninstall_<flag>() after install() + install(<flag>=True)."""
    assert runs[1][case] == [], f"{case} left these changed"


def test_rebound_methods_fall_back_through_the_kept_original(runs):
    assert runs[2]["routed"] == ["GENConv.forward", "DisenGCNLayer.forward", "CompGCNLayer.forward", "GATLayer.forward",
                       "GCNIILayer.forward", "PPNP.forward", "GINLayer.forward", "GINELayer.forward",
                       "Grand.rand_prop", "RGCNLayer.forward", "GIN.forward", "SortPool.forward", "Set2Set.forward",
                       "cogdl.models.nn.correct_smooth.outcome_correlation", "cogdl.models.nn.correct_smooth.diffusion",
                       "batch_sum_pooling", "batch_mean_pooling", "batch_max_pooling"]


def test_simple_hgn_installs_once_and_uninstalls(runs):
    assert runs[2]["simple_hgn"] == ["__main__.Conv.forward"]
    assert runs[2]["simple_hgn_restored"]
