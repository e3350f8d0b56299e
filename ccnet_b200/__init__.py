"""ccnet_b200 -- Hopper-native (sm_90a) criss-cross attention (CCNet's hot path) behind the reference API."""
from .module import CrissCrossAttention, RCCA  # noqa: F401
from .functional import cca, cca_forward, cca_backward  # noqa: F401
from . import ops  # noqa: F401  (registers torch.ops.cca.forward / backward / forward_residual)

__all__ = ["CrissCrossAttention", "RCCA", "cca", "cca_forward", "cca_backward"]
