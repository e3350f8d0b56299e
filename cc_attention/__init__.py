"""Drop-in replacement of the reference package ``cc_attention`` (cc_attention/__init__.py:1).

Put this repository ahead of the reference on ``sys.path`` and ``networks/ccnet.py:13``
(``from cc_attention import CrissCrossAttention``) picks up this repository's operator unchanged.
"""
from ccnet_b200.module import CrissCrossAttention, CrissCrossAttention3D  # noqa: F401
