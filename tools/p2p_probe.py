"""Probe (torchrun, >= 2 GPUs): can a kernel of libcogdl_b200 read a peer GPU's memory directly
(NVLink P2P through torch symmetric memory)?  Prints what works; used to decide the multi-GPU design."""
import ctypes
import os
import sys

import torch
import torch.distributed as dist
from gpu_timing import event_times

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from cogdl_b200 import _cabi
    from cogdl_b200.structure import _ptr, _stream

    try:
        import torch.distributed._symmetric_memory as symm

        n, F = 1 << 20, 128
        buf = symm.empty((n, F), dtype=torch.float32, device=dev)
        buf.fill_(float(rank + 1))
        hdl = symm.rendezvous(buf, dist.group.WORLD)
        print(f"[rank {rank}] symm ok: world={hdl.world_size} ptrs={[hex(p) for p in hdl.buffer_ptrs]}", flush=True)
        hdl.barrier()
        peer = (rank + 1) % world
        idx = torch.randint(0, n, (1 << 18,), device=dev, dtype=torch.int32)
        out = torch.empty((idx.numel(), F), device=dev)

        def gather(times):
            for _ in range(times):
                _cabi.call("cogdl_b200_gather_rows_f32", _ptr(idx), ctypes.c_void_p(hdl.buffer_ptrs[peer]), _ptr(out),
                           idx.numel(), F, _stream(dev))
        gather(3)
        torch.cuda.synchronize()
        ms = event_times(lambda: gather(5), 1, 0, flush=False)[0] / 1e3 / 5
        ok = bool((out == float(peer + 1)).all())
        print(f"[rank {rank}] peer gather of {idx.numel()} x 512 B rows from rank {peer}: correct={ok} {ms:.3f} ms "
              f"= {idx.numel() * 512 / ms / 1e6:.1f} GB/s", flush=True)
        hdl.barrier()
    except Exception as ex:  # noqa: BLE001
        print(f"[rank {rank}] symmetric memory probe FAILED: {type(ex).__name__}: {ex}", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
