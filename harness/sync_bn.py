"""Synchronised BatchNorm for the synthetic DDP train step (BASELINE configs[3]) without the per-layer host synchronisation.

`torch.nn.SyncBatchNorm` filters the gathered statistics of ranks with an empty batch through a boolean mask
(`count_all[mask]`, torch/nn/modules/_functions.py), which copies the mask to the host in EVERY layer's forward.  With ~100
normalisation layers in ResNet101+RCCA that serialises the CPU with the GPU a hundred times per step.  The reference's
own `InPlaceABNSync` (networks/ccnet.py:16) has no such stall.  Every rank of this harness always holds a non-empty batch, so the
mask is dropped; everything else is torch's SyncBatchNorm function: the same ATen kernels (batch_norm_stats, ..._gather_stats_with_counts,
..._elemt, ..._backward_reduce, ..._backward_elemt), one all-gather of [2C+1] in forward, one all-reduce of [2C] in backward."""
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F


class _SyncBNFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum, group, world):
        if not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous()
        C = x.shape[1]
        mean, invstd = torch.batch_norm_stats(x, eps)
        count = torch.full((1,), x.numel() // C, dtype=mean.dtype, device=mean.device)
        combined = torch.cat([mean, invstd, count], dim=0)                       # 2C + 1
        flat = torch.empty(1, combined.numel() * world, dtype=combined.dtype, device=combined.device)
        dist.all_gather_into_tensor(flat, combined, group, async_op=False)
        mean_all, invstd_all, count_all = torch.split(flat.view(world, -1), C, dim=1)
        counts = count_all.reshape(-1)                                           # (no empty-rank mask: no device -> host copy)
        if running_mean is not None and counts.dtype != running_mean.dtype:
            counts = counts.to(running_mean.dtype)
        mean_g, invstd_g = torch.batch_norm_gather_stats_with_counts(x, mean_all, invstd_all, running_mean, running_var,
                                                                     momentum, eps, counts)
        ctx.save_for_backward(x, weight, mean_g, invstd_g, count_all.reshape(-1).to(torch.int32))
        ctx.group = group
        return torch.batch_norm_elemt(x, weight, bias, mean_g, invstd_g, eps)

    @staticmethod
    def backward(ctx, dy):
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous()
        x, weight, mean, invstd, count_tensor = ctx.saved_tensors
        sum_dy, sum_dy_xmu, gw, gb = torch.batch_norm_backward_reduce(dy, x, mean, invstd, weight, ctx.needs_input_grad[0],
                                                                      ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        gx = None
        if ctx.needs_input_grad[0]:
            C = sum_dy.shape[0]
            combined = torch.cat([sum_dy, sum_dy_xmu], dim=0)
            dist.all_reduce(combined, dist.ReduceOp.SUM, ctx.group, async_op=False)
            sum_dy, sum_dy_xmu = torch.split(combined, C)
            gx = torch.batch_norm_backward_elemt(dy, x, mean, invstd, weight, sum_dy, sum_dy_xmu, count_tensor)
        if weight is None or not ctx.needs_input_grad[1]:
            gw = None
        if weight is None or not ctx.needs_input_grad[2]:
            gb = None
        return gx, gw, gb, None, None, None, None, None, None


class SyncBatchNorm2d(nn.BatchNorm2d):
    """BatchNorm2d whose training-mode statistics are taken over all ranks of `process_group` (default group); evaluation mode
    and single-process runs are plain batch norm.  Parameter / buffer names are those of BatchNorm2d (checkpoint compatible)."""

    process_group = None

    def forward(self, x):
        world = dist.get_world_size(self.process_group) if dist.is_available() and dist.is_initialized() else 1
        if not self.training or world == 1 or not x.is_cuda:
            return super().forward(x)
        if self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        momentum = 0.0 if self.momentum is None else self.momentum
        group = self.process_group if self.process_group is not None else dist.group.WORLD
        return _SyncBNFunction.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps, momentum, group, world)


def convert_sync_batchnorm(module: nn.Module, process_group=None) -> nn.Module:
    """Like nn.SyncBatchNorm.convert_sync_batchnorm: every nn.BatchNorm2d (exactly that type) becomes a SyncBatchNorm2d that
    shares its parameters and buffers."""
    out = module
    if type(module) is nn.BatchNorm2d:
        out = SyncBatchNorm2d(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats)
        out.process_group = process_group
        if module.affine:
            out.weight, out.bias = module.weight, module.bias
        out.running_mean, out.running_var, out.num_batches_tracked = module.running_mean, module.running_var, module.num_batches_tracked
        out.training = module.training
    for name, child in module.named_children():
        out.add_module(name, convert_sync_batchnorm(child, process_group))
    return out
