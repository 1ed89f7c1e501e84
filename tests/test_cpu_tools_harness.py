"""The timing scripts under tools/ measure through one module, tools/gpu_timing.py: no other script times with its own
CUDA events, queries the card, allocates an L2-flush buffer or hashes outputs itself."""
import glob
import hashlib
import importlib
import os
import py_compile
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
SCRIPTS = sorted(glob.glob(os.path.join(TOOLS, "*.py")))
OWNED_BY_HARNESS = ("torch.cuda.Event(", "nvidia-smi", "512 << 20", "hashlib")


@pytest.fixture(scope="module")
def gpu_timing():
    sys.path.insert(0, TOOLS)
    try:
        yield importlib.import_module("gpu_timing")
    finally:
        sys.path.remove(TOOLS)


@pytest.mark.parametrize("path", SCRIPTS, ids=os.path.basename)
def test_every_tool_compiles(path, tmp_path):
    py_compile.compile(path, cfile=str(tmp_path / "out.pyc"), doraise=True)


def test_only_the_harness_times_flushes_queries_the_card_or_hashes():
    offenders = []
    for path in SCRIPTS:
        if os.path.basename(path) == "gpu_timing.py":
            continue
        with open(path) as f:
            text = f.read()
        offenders += [f"{os.path.basename(path)}: {s}" for s in OWNED_BY_HARNESS if s in text]
    assert not offenders, offenders


def test_harness_imports_without_cuda_or_the_package():
    code = ("import sys; import gpu_timing; "
            "assert not any(m == 'cogdl_b200' or m.startswith('cogdl_b200.') for m in sys.modules), 'imports cogdl_b200'")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    subprocess.run([sys.executable, "-c", code], env=env, cwd=TOOLS, check=True, timeout=300)


def test_timers_refuse_to_run_without_cuda(gpu_timing, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    for call in (lambda: gpu_timing.event_times(lambda: None, 1, 0, False),
                 lambda: gpu_timing.host_times(lambda: None, 1, 0),
                 lambda: gpu_timing.alternate({"a": lambda: None}, 1, 1, 0, False),
                 gpu_timing.flush_l2):
        with pytest.raises(RuntimeError):
            call()


def test_digest_matches_the_inline_formula_and_hashes_in_order(gpu_timing):
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(37, 5, generator=g), torch.randint(0, 100, (11,), generator=g, dtype=torch.int32)
    at = a.t()                                                      # non-contiguous: hashed in logical order
    inline = lambda t: hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()[:16]  # noqa: E731
    for t in (a, b, at):
        assert gpu_timing.digest(t) == inline(t)
    both = hashlib.sha256(a.numpy().tobytes() + b.numpy().tobytes()).hexdigest()[:16]
    assert gpu_timing.digest(a, b) == both
    assert gpu_timing.digest(b, a) != both
