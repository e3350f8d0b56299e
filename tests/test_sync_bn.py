"""harness/sync_bn.py on the CPU: the conversion keeps parameter / buffer names and values, evaluation mode and single-process
training mode are plain batch norm (the all-rank statistics path needs CUDA + NCCL: tools/r2_gpu_syncbn.py under torch.distributed.run)."""
import torch
import torch.nn as nn

from harness.sync_bn import SyncBatchNorm2d, convert_sync_batchnorm


def test_conversion_shares_parameters_and_keeps_the_state_dict_keys():
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Sequential(nn.Conv2d(8, 4, 1), nn.BatchNorm2d(4)))
    keys = list(net.state_dict().keys())
    conv = convert_sync_batchnorm(net)
    assert list(conv.state_dict().keys()) == keys
    assert isinstance(conv[1], SyncBatchNorm2d) and isinstance(conv[3][1], SyncBatchNorm2d)
    assert conv[1].weight is net[1].weight or torch.equal(conv[1].weight, net[1].weight)
    x = torch.randn(2, 3, 9, 9)
    ref = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Sequential(nn.Conv2d(8, 4, 1), nn.BatchNorm2d(4)))
    ref.load_state_dict(conv.state_dict())
    for mode in (True, False):
        conv.train(mode); ref.train(mode)
        assert torch.allclose(conv(x), ref(x), atol=1e-6)


def test_harness_network_converts_every_batchnorm():
    from harness.ccnet_model import CCNet
    net = CCNet(num_classes=19, recurrence=1)
    n_bn = sum(1 for m in net.modules() if type(m) is nn.BatchNorm2d)
    keys = list(net.state_dict().keys())
    conv = convert_sync_batchnorm(net)
    assert sum(1 for m in conv.modules() if type(m) is nn.BatchNorm2d) == 0
    assert sum(1 for m in conv.modules() if isinstance(m, SyncBatchNorm2d)) == n_bn and n_bn > 90
    assert list(conv.state_dict().keys()) == keys
