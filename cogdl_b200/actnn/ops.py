"""actnn.ops: quantize_activation / dequantize_activation and the linear and batch-norm autograd functions, with the
reference's semantics (third_party/actnn/actnn/actnn/ops.py:77-139, 386-502) on the sm_90a kernels of actnn.cu.

quantize_activation(input, scheme) returns (packed, bits, scale, mn) like the reference: packed is a uint8 bitstream
(our layout), bits an int or an int32 [N] tensor, scale and mn bf16 per group.  With config.stochastic the rounding
noise comes from a fresh 64-bit seed drawn from torch's CPU generator, so torch.manual_seed reproduces it."""
import numpy as np
import torch
import torch.nn.functional as F

from . import kernels
from .conf import config
from .utils import empty_cache


def _check_config():
    if config.simulate or config.swap:
        raise NotImplementedError("actnn config.simulate / config.swap are not supported by cogdl_b200")


def no_scheme_compute_quantization_bits(input):
    """The reference's scheme-less path (ops.py:77-96): one width, config.activation_compression_bits[0]."""
    return config.activation_compression_bits[0]


def quantize_activation(input, scheme):
    if not config.compress_activation:
        return input, None, None, None
    _check_config()
    if scheme:
        q_bits = scheme.compute_quantization_bits(input)[1]
    else:
        q_bits = no_scheme_compute_quantization_bits(input)
    seed = kernels.draw_seed() if config.stochastic else 0
    packed, scale, mn = kernels.pack(input, q_bits, config.group_size, config.stochastic, seed)
    return packed, q_bits, scale, mn


def dequantize_activation(quantized, q_input_shape):
    if not config.compress_activation:
        return quantized[0]
    packed, q_bits, q_scale, q_min = quantized
    N = q_input_shape[0]
    D = int(np.prod(q_input_shape[1:]))
    # the group size in force now, as the reference's dequantize_and_unpack (ops.py:64-66) reads it
    out = kernels.unpack(packed, q_bits, q_scale, q_min, N, D, config.group_size)
    return out.view(*q_input_shape)


class linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, weight, bias=None, scheme=None):
        quantized = quantize_activation(input, scheme)
        empty_cache(config.empty_cache_threshold)
        ctx.scheme = scheme
        ctx.saved = quantized, weight, bias
        ctx.other_args = input.shape
        return F.linear(input, weight, bias)

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.scheme:
            ctx.scheme.set_scale(grad_output)
        quantized, weight, bias = ctx.saved
        input = dequantize_activation(quantized, ctx.other_args)
        del quantized, ctx.saved
        empty_cache(config.empty_cache_threshold)
        C_in = input.shape[-1]
        C_out = grad_output.shape[-1]
        grad_output_flatten = grad_output.reshape(-1, C_out)
        input_flatten = input.reshape(-1, C_in)
        grad_input = grad_output_flatten.mm(weight)
        grad_weight = grad_output_flatten.t().mm(input_flatten)
        grad_bias = grad_output_flatten.sum(0) if bias is not None else None
        if ctx.scheme:
            ctx.scheme.if_allocate_perlayer()
        return grad_input, grad_weight, grad_bias, None


class batch_norm(torch.autograd.Function):
    """BN on the full-precision input; the input is saved quantized, and the backward runs torch's
    native_batch_norm_backward on its dequantized copy."""

    @staticmethod
    def forward(ctx, input, running_mean, running_var, weight, bias, training, exponential_average_factor, eps,
                scheme):
        quantized = quantize_activation(input, scheme)
        empty_cache(config.empty_cache_threshold)
        output, save_mean, save_var = torch.native_batch_norm(input, weight, bias, running_mean, running_var, training,
                                                              exponential_average_factor, eps)
        ctx.scheme = scheme
        ctx.other_args = input.shape
        ctx.saved = (quantized, weight, running_mean, running_var, save_mean, save_var, training, eps)
        return output

    @staticmethod
    def backward(ctx, grad_output):
        quantized, weight, running_mean, running_var, save_mean, save_var, training, eps = ctx.saved
        input = dequantize_activation(quantized, ctx.other_args)
        del quantized, ctx.saved
        empty_cache(config.empty_cache_threshold)
        grad_input, grad_weight, grad_bias = torch.ops.aten.native_batch_norm_backward(
            grad_output.contiguous(), input, weight, running_mean, running_var, save_mean, save_var, training, eps,
            [ctx.needs_input_grad[0], ctx.needs_input_grad[3], ctx.needs_input_grad[4]])
        if ctx.scheme:
            ctx.scheme.if_allocate_perlayer()
        return grad_input, None, None, grad_weight, grad_bias, None, None, None, None
