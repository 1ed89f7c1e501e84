"""The reference Correct & Smooth through cogdl_b200.install(correct_smooth=True), in a child process
(tests/correct_smooth_refpkg_check.py)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_correct_smooth_through_install():
    """postprocess and diffusion bit-identical to the unfused reference loops on this package's spmm and within 1e-5
    of the reference's CPU results; the fallback cases and uninstall leave the originals in charge."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.correct_smooth_refpkg_check"], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"] and res["rebound"] and res["restored"], res
    assert res["patched"] == ["cogdl.models.nn.correct_smooth.outcome_correlation",
                              "cogdl.models.nn.correct_smooth.diffusion"], res
    assert len(res["bit_identical"]) == 9 and all(res["bit_identical"].values()), res
    assert max(res["vs_golden"].values()) <= 1e-5, res
    assert "labelprop_kernel" in res["last_kernel"], res
    assert all(res["fallbacks"].values()), res
    assert res["fallback_calls"] == ["outcome_correlation"] * 5 + ["diffusion"] * 2, res
