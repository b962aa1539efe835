"""visdial_b200 — H100-native engine for the per-batch hot path of batra-mlp-lab/visdial.

Host-side mirror (Python, because no Lua runtime exists in this image) of the reference's plugin
surface: `encoders/<name>` + `decoders/<name>` modules loaded by name (model.lua:19-26), the `Model`
class (model.lua:8-430) and the `utils` rank helpers, all calling libvisdial_b200.so through the
C ABI of include/visdial_b200.h.  The same ABI is what lua/*.lua binds with LuaJIT FFI."""
from .engine import Engine, Batch, DeviceTensor, init_parameters, split_parameters, layout, DEFAULT_PARAMS  # noqa: F401
from .model import Model  # noqa: F401
from ._lib import VdError, VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16  # noqa: F401
