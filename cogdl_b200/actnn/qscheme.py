"""actnn.qscheme.QScheme: the reference's per-layer adaptive scheme (third_party/actnn/actnn/actnn/qscheme.py) with
the per-row bit allocation on the device.  C is computed with the reference's torch ops and never leaves the device;
kernels.allocate_bits gives the reference greedy's result bit for bit.  allocate_perlayer (one entry per layer, or
per (layer, row) when the group's width differs from initial_bits) runs on the host, as calc_precision does."""
import numpy as np
import torch

from . import kernels
from .conf import config


def calc_precision_host(b, C, w, target):
    """The reference greedy (calc_precision.cc:9-50) on the host: while sum(b * w) > target, take the entry of the
    largest (float)(C_i * (1 / (2^b_i - 1)^2 - 1 / (2^(b_i - 1) - 1)^2) / w_i), ties to the larger index, and lower
    its b by one; an entry at b = 1 leaves the queue.  b: int32 [N] (changed in place and returned), C float32 [N]
    (finite, >= 0), w int32 [N] (> 0).

    An entry's keys fall as its b falls, so the greedy takes all keys in one descending (key, index) order: the keys
    are sorted once and the pops are the shortest prefix whose weights bring sum(b * w) to the target."""
    b_data = b.numpy()
    C_data = C.to(torch.float32).numpy().astype(np.float64)
    w_data = w.numpy().astype(np.int64)
    b_sum = int(np.dot(b_data.astype(np.int64), w_data))
    if b_sum <= target:
        return b
    reps = np.maximum(b_data.astype(np.int64) - 1, 0)
    idx = np.repeat(np.arange(len(b_data), dtype=np.int64), reps)
    first = np.repeat(np.cumsum(reps) - reps, reps)
    bb = np.repeat(b_data.astype(np.int64), reps) - (np.arange(len(idx)) - first)   # b_i, b_i - 1, ..., 2
    c1 = ((1 << bb) - 1) ** 2
    c2 = ((1 << (bb - 1)) - 1) ** 2
    key = (C_data[idx] * (1.0 / c1 - 1.0 / c2) / w_data[idx]).astype(np.float32)
    order = np.lexsort((-bb, -idx, -key.astype(np.float64)))
    popped = np.cumsum(w_data[idx[order]])
    k = int(np.searchsorted(popped, b_sum - target, side="left")) + 1   # first prefix with b_sum - popped <= target
    b_data -= np.bincount(idx[order[:k]], minlength=len(b_data)).astype(b_data.dtype)
    return b


class QScheme(object):
    num_samples = 1
    num_layers = 0
    batch = None
    update_scale = True
    layers = []
    prev_layer = None

    def __init__(self, layer, group=0, num_locations=1, depthwise_groups=1):
        self.initial_bits = config.initial_bits
        self.bits = config.activation_compression_bits[group]
        if config.use_gradient:
            assert QScheme.num_samples > 1
            self.scales = torch.zeros(QScheme.num_samples)
        else:
            self.scales = torch.tensor([0.0])
        QScheme.layers.append(self)
        self.C = None
        self.dim = None
        self.num_locations = num_locations
        self.depthwise_groups = depthwise_groups
        self.layer = layer
        self.group = group
        self.name = "layer_{}".format(QScheme.num_layers)
        QScheme.num_layers += 1

    def get_scale(self):
        if config.use_gradient:
            assert QScheme.batch is not None
            scale = self.scales[QScheme.batch].clone()
            avg_scale = scale.mean()
            scale[scale == 0] = avg_scale + 1e-9
            return scale
        return self.scales

    def set_scale(self, grad):
        if QScheme.update_scale:
            if config.use_gradient:
                assert QScheme.batch is not None
                scale = grad.view(grad.shape[0], -1).float().norm(dim=1).square().cpu()
                self.scales[QScheme.batch] = self.scales[QScheme.batch] * 0.5 + scale * 0.5
            else:
                scale = grad.view(grad.shape[0], -1).float().norm(dim=1).square()
                self.scales = scale.mean()

    def range_sqr(self, input):
        """G * ||R_n||^2 / I of the reference (qscheme.py:59-80), on the device."""
        N = input.shape[0]
        num_pixels = input.reshape(N, -1).shape[1] // input.shape[1]
        mn, mx = kernels.group_minmax(input, config.group_size)
        if not config.pergroup:
            mn = torch.ones_like(mn) * mn.min()
            mx = torch.ones_like(mx) * mx.max()
        return torch.norm((mx - mn).view(N, -1), dim=1).float().square() * (config.group_size / num_pixels), mn, mx

    def compute_quantization_bits(self, input):
        """(input, bits int32 [N] on the device, mn [N, G], mx [N, G])."""
        QScheme.prev_layer = self
        N = input.shape[0]
        Range_sqr, mn, mx = self.range_sqr(input)
        grad_sum = self.get_scale().to(input.device)
        C = (self.num_locations / 4 / self.depthwise_groups * Range_sqr * grad_sum).to(torch.float32)
        b = kernels.allocate_bits(C, int(self.bits * N), int(self.initial_bits))
        self.C = C
        self.dim = input.numel() // N
        self.b = b
        return input, b, mn, mx

    @staticmethod
    def allocate_perlayer():
        num_groups = len(config.activation_compression_bits)
        for g in range(num_groups):
            layers = [layer for layer in QScheme.layers if layer.group == g]
            L = len(layers)
            if L == 0:
                continue
            if config.activation_compression_bits[g] == config.initial_bits:
                C = torch.tensor([float(layer.C.sum()) for layer in layers], dtype=torch.float32)
                w = torch.tensor([layer.dim for layer in layers], dtype=torch.int)
                total_bits = w.sum() * config.activation_compression_bits[g]
                b = torch.ones(L, dtype=torch.int32) * 8
                b = calc_precision_host(b, C, w, float(total_bits))
                for i in range(L):
                    layers[i].bits = layers[i].initial_bits = int(b[i])
            else:
                C = torch.cat([layer.C.detach().float().cpu() for layer in layers], 0)
                N = layers[0].C.shape[0]
                w = torch.cat([torch.ones(N, dtype=torch.int32) * layer.dim for layer in layers], 0)
                total_bits = w.sum() * config.activation_compression_bits[g]
                b = torch.ones(N * L, dtype=torch.int32) * config.initial_bits
                b = calc_precision_host(b, C, w, float(total_bits))
                for i in range(L):
                    layers[i].bits = b[i * N:(i + 1) * N].float().mean()

    def if_allocate_perlayer(self):
        if not config.perlayer:
            return
        for layer in QScheme.layers:
            if layer.C is None:
                return
        first_layer = None
        for layer in QScheme.layers:
            if layer.layer.weight.requires_grad:
                first_layer = layer
                break
        if config.compress_activation and config.training:
            if self == first_layer:
                from .qbnscheme import QBNScheme

                QScheme.allocate_perlayer()
                QBNScheme.allocate_perlayer()
