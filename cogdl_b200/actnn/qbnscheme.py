"""actnn.qbnscheme.QBNScheme: the reference's batch-norm scheme (third_party/actnn/actnn/actnn/qbnscheme.py) with the
per-row bit allocation on the device."""
import torch

from . import kernels
from .conf import config
from .qscheme import QScheme


class QBNScheme(QScheme):
    layers = []

    def __init__(self, group=0):
        self.initial_bits = config.initial_bits
        self.bits = config.activation_compression_bits[group]
        QBNScheme.layers.append(self)
        if len(QScheme.layers) > 0:
            self.prev_linear = QScheme.layers[-1]
        else:
            self.prev_linear = None

    def compute_quantization_bits(self, input):
        self.prev_linear = QScheme.prev_layer
        N = input.shape[0]
        Range_sqr, mn, mx = self.range_sqr(input)
        C = Range_sqr.to(torch.float32)
        b = kernels.allocate_bits(C, int(self.bits * N), int(self.initial_bits))
        return input, b, mn, mx

    @staticmethod
    def allocate_perlayer():
        for layer in QBNScheme.layers:
            if layer.prev_linear is not None:
                layer.bits = layer.prev_linear.bits
            else:
                layer.bits = 8
