"""`import quant_cuda` drop-in: the reference's modeling_llama.py:53 does exactly this import.
Putting the repo root (or an installed kvquant_b200) on sys.path makes the reference's QuantK/QuantV run on the
H100-native kernels unchanged.  See INTEGRATION.md."""
from kvquant_b200.quant_cuda import *  # noqa: F401,F403
from kvquant_b200.quant_cuda import OP_NAMES, rope_table  # noqa: F401
