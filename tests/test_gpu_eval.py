"""GPU side of SURVEY.md 8(f) N4: sliding-window inference through the harness network with this repository's operator in its head
against the SAME weights with the CPU oracle module in the head (logit difference on synthetic tiles), and a checkpoint round
trip in the reference's on-disk format (utils/pyt_utils.py:47-85)."""
import copy
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _networks():
    from harness.ccnet_model import CCNet
    from oracle.cca_oracle import CrissCrossAttentionOracle
    torch.manual_seed(21)
    net = CCNet(num_classes=7, layers=(1, 1, 1, 1), recurrence=2).eval()
    with torch.no_grad():
        net.head.cca.gamma.fill_(0.7)
        for m in net.modules():                                   # non-trivial running statistics
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.1)
                m.running_var.uniform_(0.5, 1.5)
    ref = copy.deepcopy(net)
    oracle = CrissCrossAttentionOracle(512)
    oracle.load_state_dict(net.head.cca.state_dict())
    ref.head.cca = oracle.eval()
    return net, ref


def test_sliding_window_logits_match_cpu_oracle_network(tmp_path):
    from harness import eval_synth as ev
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    net, ref = _networks()
    # through the reference's checkpoint format: saved from a wrapper ('module.' keys) under 'model', loaded non-strictly
    torch.save({"model": {"module." + k: v for k, v in net.state_dict().items()}}, tmp_path / "snap.pth")
    from harness.ccnet_model import CCNet
    gpu_net = CCNet(num_classes=7, layers=(1, 1, 1, 1), recurrence=2).eval()
    gpu_net, missing, unexpected = ev.load_model(gpu_net, str(tmp_path / "snap.pth"))
    assert not missing and not unexpected
    gpu_net = gpu_net.cuda()
    image = torch.randn(1, 3, 161, 225, generator=torch.Generator().manual_seed(4))
    tile = (129, 129)                                             # 17 x 17 feature map per window, 2 x 3 windows
    want = ev.predict_sliding(ref, image, tile, 7)
    got = ev.predict_sliding(gpu_net, image.cuda(), tile, 7).cpu()
    scale = want.abs().max().item()
    assert (got - want).abs().max().item() <= 2e-4 * scale, ((got - want).abs().max().item(), scale)
    got3 = ev.predict_sliding(gpu_net, image.cuda(), tile, 7, tile_batch=3).cpu()      # windows stacked into one forward
    assert (got3 - want).abs().max().item() <= 2e-4 * scale
    # the operator matters for the result: without it (gamma = 0) the logits move by much more than the tolerance
    with torch.no_grad():
        gpu_net.head.cca.gamma.zero_()
    off = ev.predict_sliding(gpu_net, image.cuda(), tile, 7).cpu()
    assert (off - want).abs().max().item() > 50 * 2e-4 * scale
    label = torch.randint(0, 7, (1, 161, 225), generator=torch.Generator().manual_seed(5))
    cm_ref = ev.get_confusion_matrix(label, want.argmax(3), 7)
    cm_got = ev.get_confusion_matrix(label.cuda(), got.cuda().argmax(3), 7).cpu()
    assert (cm_ref - cm_got).abs().sum().item() <= 4              # argmax ties at the tolerance may flip a pixel or two
