"""The harness network (harness/ccnet_model.py, used for BASELINE configs[2] / [3]) names and shapes every tensor exactly like
the reference's Seg_Model (networks/ccnet.py with the inplace_abn stand-in), whose state-dict key -> shape map is stored in
tests/golden/reference_state_maps.json (tests/golden/make_reference_maps.py)."""
import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_harness_network_matches_reference_state_dict():
    with open(os.path.join(ROOT, "tests", "golden", "reference_state_maps.json")) as f:
        maps = json.load(f)
    from harness.ccnet_model import CCNet
    with torch.device("meta"):
        ours = CCNet(num_classes=19, recurrence=2)
    a = {k: tuple(v) for k, v in maps["seg_model"].items()}
    b = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    assert a == b, (sorted(set(a) ^ set(b))[:20], [k for k in a if k in b and a[k] != b[k]][:10])
    assert sum(p.numel() for p in ours.parameters()) == maps["seg_model_params"]


def test_harness_network_forward_shapes_on_cpu_fallback_free():
    """Tiny structural check without the operator: the head's attention needs CUDA, so only the backbone + dsn run here."""
    from harness.ccnet_model import CCNet
    net = CCNet(num_classes=5, layers=(1, 1, 1, 1), recurrence=1).eval()
    x = torch.randn(1, 3, 65, 65)
    with torch.no_grad():
        y = torch.relu(net.bn1(net.conv1(x)))
        y = torch.relu(net.bn2(net.conv2(y)))
        y = net.maxpool(torch.relu(net.bn3(net.conv3(y))))
        y = net.layer3(net.layer2(net.layer1(y)))
        assert y.shape == (1, 1024, 9, 9)                # 65 -> 33 -> 17 -> 9: output stride 8
        assert net.dsn(y).shape == (1, 5, 9, 9)
        assert net.layer4(y).shape == (1, 2048, 9, 9)
