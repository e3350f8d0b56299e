"""ccnet_b200 -- Hopper-native (sm_90a) criss-cross attention (CCNet's hot path) behind the reference API."""
from .module import CrissCrossAttention, CrissCrossAttention3D, RCCA, RingState  # noqa: F401
from .functional import (cca, cca3d, cca3d_attention, cca3d_backward, cca3d_forward, cca3d_step, cca_attention,  # noqa: F401
                         cca_backward, cca_forward)
from . import ops  # noqa: F401  (registers torch.ops.cca.forward / backward / forward_residual / attention / 3D ops)

__all__ = ["CrissCrossAttention", "CrissCrossAttention3D", "RCCA", "cca", "cca_forward", "cca_backward", "cca_attention",
           "cca3d", "cca3d_forward", "cca3d_backward", "cca3d_attention", "cca3d_step", "RingState"]
