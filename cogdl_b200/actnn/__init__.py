"""The `actnn` API that CogDL imports (activation-compressed training, third_party/actnn), on the sm_90a kernels of
actnn.cu: set_optimization_level and config (actnn.conf), quantize_activation / dequantize_activation (actnn.ops),
QScheme and QBNScheme with the per-row bit allocation on the device, QLinear / QReLU / QDropout / QBatchNorm1d
(actnn.layers) and empty_cache (actnn.utils).  Convolutions, pooling, SyncBN, the data loader and host swapping are
not provided.  cogdl_b200.install(actnn=True) puts this package into sys.modules as `actnn` when no real actnn
imports."""
from . import conf, kernels, layers, ops, qbnscheme, qscheme, utils  # noqa: F401
from .conf import config, set_optimization_level  # noqa: F401
from .layers import QBatchNorm1d, QDropout, QLinear, QReLU  # noqa: F401
from .qbnscheme import QBNScheme  # noqa: F401
from .qscheme import QScheme  # noqa: F401
from .utils import compute_tensor_bytes, empty_cache, get_memory_usage  # noqa: F401
