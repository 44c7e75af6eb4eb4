"""nn.SyncBatchNorm.convert_sync_batchnorm on the sparse-layout EdgeConv, without a GPU: the converted layers hand
their SyncBatchNorm to the kernel, and with no process group it shares nothing."""
import pytest
import torch
from torch import nn


def _sync_bn(mod):
    return [m for m in mod.modules() if isinstance(m, nn.SyncBatchNorm)]


def test_converted_edgconv_parts_return_sync_batchnorm():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(S.EdgConv(6, 16, "prelu", "batch"))
    lin, act, prelu, bn = conv._parts()
    assert isinstance(bn, nn.SyncBatchNorm) and bn.num_features == 16
    assert lin is conv.nn[0] and act == "prelu" and prelu is conv.nn[2].weight


@pytest.mark.parametrize("make", [
    lambda S: S.GraphConv(6, 16, "edge", "relu", "batch"),
    lambda S: S.ResDynBlock(16, 9, 2, "edge", "leakyrelu", "batch"),
], ids=["GraphConv-edge", "ResDynBlock-edge"])
def test_edge_blocks_convert(make):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    mod = nn.SyncBatchNorm.convert_sync_batchnorm(make(S))
    edge = [m for m in mod.modules() if isinstance(m, S.EdgConv)]
    assert len(edge) == 1 and len(_sync_bn(mod)) == 1
    assert edge[0]._parts()[3] is _sync_bn(mod)[0]


def test_no_process_group_means_local_statistics():
    import torch.distributed as dist
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    assert not (dist.is_available() and dist.is_initialized())
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(S.EdgConv(6, 16, "relu", "batch")).train()
    bn = conv._parts()[3]
    assert _native.sync_group(bn) is None
    prm = conv._conv_params()
    assert prm.norm == _native.NORM_BATCH_TRAIN and prm.sync_group is None


def test_cpu_tensors_raise_not_implemented_with_cuda_in_message():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    x, ei = torch.randn(5, 4), torch.zeros((2, 3), dtype=torch.long)
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(S.EdgConv(4, 8, "relu", "batch"))
    with pytest.raises(NotImplementedError, match="SyncBatchNorm needs CUDA tensors"):
        conv(x, ei)
    with pytest.raises(RuntimeError, match="CUDA") as e:       # the unconverted layer keeps its RuntimeError
        S.EdgConv(4, 8, "relu", "batch")(x, ei)
    assert not isinstance(e.value, NotImplementedError)
