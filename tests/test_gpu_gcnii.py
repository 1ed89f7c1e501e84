"""The reference GCNII and APPNP through cogdl_b200.install(gcnii=True, appnp=True), in a child process
(tests/gcnii_refpkg_check.py)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_gcnii_and_appnp_through_install():
    """Eval logits vs the reference's golden CPU logits and parameter gradients vs the fp64 restatement, for a
    CSR-built and an edge_index-built graph; a seeded training step equal to the unfused GPU path (same dropout
    masks); install() without the flags and uninstall leave the originals in charge."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.gcnii_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"] and res["rebound"] and res["restored"], res
    assert res["patched"] == ["cogdl.layers.gcnii_layer.GCNIILayer.forward", "cogdl.models.nn.ppnp.PPNP.forward"], res
    assert len(res["logits_vs_golden"]) == 6, res
    assert max(res["logits_vs_golden"].values()) <= 1e-5, res
    assert max(res["grads_vs_fp64"].values()) <= 1e-5, res
    assert max(res["train_logits"].values()) <= 1e-5, res
    assert max(res["train_grads"].values()) <= 1e-4, res
