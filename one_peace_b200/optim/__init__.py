from .adam import Adam, AdjustAdam  # noqa: F401
from .adan import Adan, FairseqAdan  # noqa: F401
from .fp16_optimizer_memory_efficent import MemoryEfficientBF16Optimizer  # noqa: F401
