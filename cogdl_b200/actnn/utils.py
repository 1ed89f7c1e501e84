"""actnn.utils: the helpers CogDL imports (empty_cache) and the reference's byte counters."""
import numpy as np
import torch


def get_memory_usage(print_info=False):
    """Allocated bytes of device 0, from torch's allocator."""
    allocated = torch.cuda.memory_allocated(0)
    reserved = torch.cuda.memory_reserved(0)
    if print_info:
        print("allocated: %.2f MB" % (allocated / 1024 / 1024), flush=True)
        print("reserved:  %.2f MB" % (reserved / 1024 / 1024), flush=True)
    return allocated


def compute_tensor_bytes(tensors):
    """Bytes held by a tensor or a list of tensors (non-tensors count 0)."""
    if not isinstance(tensors, (list, tuple)):
        tensors = [tensors]
    return int(sum(np.prod(x.size()) * x.element_size() for x in tensors if isinstance(x, torch.Tensor)))


def empty_cache(ratio):
    """Release the allocator's cached blocks when less than `ratio` of the reserved memory is in use."""
    if ratio is None:
        return
    allocated = torch.cuda.memory_allocated(0)
    reserved = torch.cuda.memory_reserved(0)
    if reserved > 0 and allocated / reserved < ratio:
        torch.cuda.empty_cache()
