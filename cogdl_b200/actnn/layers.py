"""actnn.layers: QLinear, QReLU, QDropout and QBatchNorm1d (third_party/actnn/actnn/actnn/layers.py:194-380).
QReLU and QDropout save a 1-bit mask instead of their input; QDropout's mask is drawn in the kernel from a fresh
64-bit seed taken from torch's CPU generator on every call."""
import torch
import torch.nn as nn

from . import kernels
from .conf import config
from .ops import batch_norm, linear
from .qbnscheme import QBNScheme
from .qscheme import QScheme


class QLinear(nn.Linear):
    num_layers = 0

    def __init__(self, input_features, output_features, bias=True, group=0):
        super(QLinear, self).__init__(input_features, output_features, bias)
        if config.adaptive_conv_scheme:
            self.scheme = QScheme(self, group=group)
        else:
            self.scheme = None

    def forward(self, input):
        if config.training:
            return linear.apply(input, self.weight, self.bias, self.scheme)
        return super(QLinear, self).forward(input)


class QBatchNorm1d(nn.BatchNorm1d):
    def __init__(self, num_features, eps=1e-05, momentum=0.1, affine=True, track_running_stats=True, group=0):
        super(QBatchNorm1d, self).__init__(num_features, eps, momentum, affine, track_running_stats)
        if config.adaptive_bn_scheme:
            self.scheme = QBNScheme(group=group)
        else:
            self.scheme = None

    def forward(self, input):
        if not config.training:
            return super(QBatchNorm1d, self).forward(input)
        self._check_input_dim(input)
        exponential_average_factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats:
            if self.num_batches_tracked is not None:
                self.num_batches_tracked = self.num_batches_tracked + 1
                if self.momentum is None:
                    exponential_average_factor = 1.0 / float(self.num_batches_tracked)
                else:
                    exponential_average_factor = self.momentum
        if self.training:
            bn_training = True
        else:
            bn_training = (self.running_mean is None) and (self.running_var is None)
        return batch_norm.apply(
            input,
            self.running_mean if not self.training or self.track_running_stats else None,
            self.running_var if not self.training or self.track_running_stats else None,
            self.weight, self.bias, bn_training, exponential_average_factor, self.eps, self.scheme)


class _QReLUFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input):
        y, mask = kernels.relu_fwd(input)
        ctx.save_for_backward(mask)
        return y

    @staticmethod
    def backward(ctx, grad_output):
        (mask,) = ctx.saved_tensors
        return kernels.relu_bwd(grad_output, mask)


class _QDropoutFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, p, seed):
        y, mask = kernels.dropout_fwd(input, p, seed)
        ctx.p = p
        ctx.save_for_backward(mask)
        return y

    @staticmethod
    def backward(ctx, grad_output):
        (mask,) = ctx.saved_tensors
        return kernels.dropout_bwd(grad_output, mask, ctx.p), None, None


def act_quantized_relu(input):
    return _QReLUFunction.apply(input)


def act_quantized_dropout(input, p, seed=None):
    return _QDropoutFunction.apply(input, p, kernels.draw_seed() if seed is None else seed)


class QReLU(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, input):
        return act_quantized_relu(input)


class QDropout(nn.Dropout):
    def __init__(self, p=0.5):
        super().__init__(p=p)

    def forward(self, input):
        if self.training:
            return act_quantized_dropout(input, self.p)
        return super(QDropout, self).forward(input)
