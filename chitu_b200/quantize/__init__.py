from .fp8 import Fp8Linear, quant_act_fp8  # noqa: F401
from .w4a16 import W4A16Linear  # noqa: F401
from .w8a8 import W8A8Linear, quant_act, quant_weight  # noqa: F401
