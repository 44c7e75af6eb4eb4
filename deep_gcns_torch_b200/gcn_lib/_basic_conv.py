"""The BasicConv lowering of the dense and sparse graph convolutions: their `nn` (a Linear or 1x1 conv, then any of
BatchNorm and one activation) read into _native.ConvParams, and torch's BatchNorm training bookkeeping after the
fused forward."""
import torch
from torch import nn

from .. import _native


class BasicConvLowering:
    """Mixin of a module whose `nn` the kernels run as one dgcn_basic_conv."""

    def _parts(self):
        """(linear_or_conv, act, prelu_weight, bn) of self.nn; NotImplementedError for a layer the kernels do not
        run."""
        lin, act, prelu, bn = self.nn[0], None, None, None
        for m in list(self.nn)[1:]:
            if isinstance(m, nn.ReLU):
                act = "relu"
            elif isinstance(m, nn.LeakyReLU):
                act = "leakyrelu"
            elif isinstance(m, nn.PReLU):
                act, prelu = "prelu", m.weight
            elif isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d, nn.SyncBatchNorm)):    # (convert_sync_batchnorm)
                bn = m
            else:
                raise NotImplementedError("{}: a {} layer in nn is not supported".format(type(self).__name__,
                                                                                       type(m).__name__))
        if prelu is not None and prelu.numel() != 1:
            raise NotImplementedError("{}: PReLU with one weight per channel is not supported".format(
                type(self).__name__))
        return lin, act, prelu, bn

    def _conv_params(self, parts=None):
        """ConvParams of self.nn (parts: _parts(), when the caller has it): batch statistics in training mode or
        without running statistics, the running ones otherwise."""
        lin, act, prelu, bn = self._parts() if parts is None else parts
        norm, kw = _native.NORM_NONE, {}
        if bn is not None:
            use_batch = self.training or bn.running_mean is None
            norm = _native.NORM_BATCH_TRAIN if use_batch else _native.NORM_BATCH_EVAL
            kw = dict(bn_weight=bn.weight, bn_bias=bn.bias, bn_mean=bn.running_mean, bn_var=bn.running_var,
                      bn_eps=bn.eps, sync_group=_native.sync_group(bn))
        return _native.ConvParams(lin.weight, lin.bias, act, prelu, norm, **kw)


def update_running_stats(bn, prm, count):
    """BatchNorm training bookkeeping (running statistics, momentum, unbiased variance, num_batches_tracked) exactly
    as torch does it, after a forward with prm over `count` positions.  An empty batch leaves the running statistics
    as torch does.  With synced statistics the variance is unbiased with the global count, read on the device, and a
    rank without positions updates its running statistics from the global ones like its peers."""
    if bn is None or prm.norm != _native.NORM_BATCH_TRAIN or not bn.track_running_stats:
        return
    with torch.no_grad():
        bn.num_batches_tracked += 1
        if prm.moments is None and count == 0:
            return
        mom = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)
        if prm.moments is not None:
            count = prm.moments[-1]
            unbiased = prm.batch_var * (count / (count - 1).clamp_min(1)).float()
        else:
            unbiased = prm.batch_var * (count / max(count - 1, 1))
        bn.running_mean.mul_(1 - mom).add_(prm.batch_mean, alpha=mom)
        bn.running_var.mul_(1 - mom).add_(unbiased, alpha=mom)
