"""How the scripts under tools/ measure: the CUDA-event and host timers, the L2 flush, the card line, output hashes,
peak memory and the result file.  Every speed figure these scripts print is taken with the functions here.

This module does not import cogdl_b200: time_spmm_l2.py's workers load the package from other trees.  Without a CUDA
device the timers raise; they never fall back to host timing.
"""
import hashlib
import json
import os
import statistics
import subprocess
import time

import torch

FLUSH_BYTES = 512 << 20      # ten times the H100's 50 MB L2
_flush = None


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("gpu_timing: no CUDA device")


def card(fields="name,power.limit,clocks.max.sm"):
    """One `nvidia-smi --query-gpu` line for the current CUDA device (selected by UUID), or why the query failed."""
    try:
        uuid = str(torch.cuda.get_device_properties(torch.cuda.current_device()).uuid)
        q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader",
                            "-i", uuid if uuid.startswith("GPU-") else "GPU-" + uuid],
                           capture_output=True, text=True, timeout=30)
    except Exception as ex:  # noqa: BLE001
        return f"nvidia-smi query failed ({ex})"
    if q.returncode != 0:
        return f"nvidia-smi query failed ({(q.stderr or q.stdout).strip()})"
    return q.stdout.strip()


def flush_l2():
    """Zero a 512 MiB device buffer, so no operand of the next call is left in the L2."""
    global _flush
    if _flush is None:
        _require_cuda()
        _flush = torch.empty(FLUSH_BYTES, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def event_times(fn, reps, warmup, flush, sync_each=True):
    """CUDA-event time of each of `reps` calls of fn, in us, after `warmup` untimed calls.  With `flush`, flush_l2()
    runs before each timed call, outside the interval.  With `sync_each`, each timed call ends in a device synchronise,
    so the host cannot queue the next call early; without it the calls are queued back to back, as bench.py does."""
    _require_cuda()
    for _ in range(warmup):
        fn()
    evs = []
    for _ in range(reps):
        if flush:
            flush_l2()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        if sync_each:
            torch.cuda.synchronize()
        evs.append((a, b))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) * 1e3 for a, b in evs]


def host_times(fn, reps, warmup):
    """perf_counter time of each of `reps` calls of fn, in us, each ended by a device synchronise, after `warmup`
    untimed calls."""
    _require_cuda()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e6)
    return ts


def alternate(variants, rounds, steps, warmup, flush, sync_each=True):
    """{name: (all us, per-round medians)} for variants {name: fn}: `warmup` untimed calls of each, then `rounds`
    rounds in which the variants take turns, each timed over `steps` calls by event_times."""
    _require_cuda()
    for fn in variants.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    out = {name: ([], []) for name in variants}
    for _ in range(rounds):
        for name, fn in variants.items():
            ts = event_times(fn, steps, 0, flush, sync_each)
            out[name][0].extend(ts)
            out[name][1].append(statistics.median(ts))
    return out


def peak_above(fn):
    """Peak bytes allocated while fn runs, above what was allocated before it."""
    _require_cuda()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def digest(*tensors):
    """The first 16 hex digits of the SHA-256 of the tensors' bytes, in order."""
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def write_result(out_dir, name, res):
    """Set res["card"], print the card line and write res to out_dir/name.json."""
    res["card"] = card()
    print("card:", res["card"], flush=True)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, name + ".json"), "w") as f:
        json.dump(res, f, indent=1)
