"""Row (b) of the scope table: the reference's networks/ccnet.py imports ``CrissCrossAttention`` from the ``cc_attention``
package (networks/ccnet.py:13) and builds its RCCA head around it (networks/ccnet.py:105).  What that network and the
reference's own module expect of the operator -- state-dict keys and shapes -- was taken from the reference itself and stored
in tests/golden/reference_state_maps.json (tests/golden/make_reference_maps.py); these tests hold this repository to it."""
import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAPS = os.path.join(ROOT, "tests", "golden", "reference_state_maps.json")


def _maps():
    with open(MAPS) as f:
        return json.load(f)


def test_reference_network_builds_on_the_b200_operator():
    import cc_attention
    import ccnet_b200
    assert cc_attention.CrissCrossAttention is ccnet_b200.CrissCrossAttention     # what networks/ccnet.py:13 imports
    assert cc_attention.__file__.startswith(ROOT)
    seg = _maps()["seg_model"]
    keys = {k for k in seg if k.startswith("head.cca.")}
    assert keys == {"head.cca." + n for n in ("gamma", "query_conv.weight", "query_conv.bias", "key_conv.weight",
                                               "key_conv.bias", "value_conv.weight", "value_conv.bias")}
    assert tuple(seg["head.cca.query_conv.weight"]) == (64, 512, 1, 1)
    assert tuple(seg["head.cca.value_conv.weight"]) == (512, 512, 1, 1)
    assert _maps()["seg_model_recurrence"] == 2
    with torch.device("meta"):
        head = ccnet_b200.CrissCrossAttention(512)
    ours = {"head.cca." + k: list(v.shape) for k, v in head.state_dict().items()}
    assert ours == {k: seg[k] for k in keys}


def test_released_checkpoint_keys_load_into_the_module():
    """A checkpoint with the reference module's head.cca.* entries (keys and shapes of the reference's CrissCrossAttention(512))
    restores the module's parameters through the non-strict load the reference's utils/pyt_utils.py:47-85 load_model does."""
    import ccnet_b200
    ref_map = _maps()["criss_cross_attention_512"]
    gen = torch.Generator().manual_seed(0)
    ref_sd = {k: torch.randn(*shape, generator=gen) for k, shape in ref_map.items()}
    ref_sd["gamma"].fill_(0.37)
    ckpt = {"head.cca." + k: v for k, v in ref_sd.items()}
    head = ccnet_b200.CrissCrossAttention(512)
    wrapper = torch.nn.Module()
    wrapper.head = torch.nn.Module()
    wrapper.head.cca = head
    missing, unexpected = wrapper.load_state_dict(ckpt, strict=False)
    assert not missing and not unexpected
    for k, v in ref_sd.items():
        assert torch.equal(head.state_dict()[k], v), k
