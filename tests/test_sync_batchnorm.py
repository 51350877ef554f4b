"""nn.SyncBatchNorm on the ResNet-18 and PPM encoders, without a GPU: the split entry points of libdva_resnet.so
reject bad arguments through dva_last_error() without a launch, nn.SyncBatchNorm.convert_sync_batchnorm gives each
family and the PPM head the module tree the trunk walk and the head expect, and nothing is synchronised without a
process group.  tests/test_gpu_sync_batchnorm.py runs them over ranks."""
import pytest
import torch
from torch import nn

from deepviewagg_b200 import _lib, ops
from deepviewagg_b200.core.common_modules import MLP, FastBatchNorm1d
from deepviewagg_b200.modules.multimodal.modalities import image as I

FAMILIES = ["ADE20KResNet18TruncatedLayer4", "ADE20KResNet18Pyramid", "ADE20KResNet18Layer0",
            "ResNet18TruncatedLayer4", "ResNet18Pyramid", "CityscapesResNet18TruncatedLayer2", "CityscapesResNet18"]
DROPPED = ("_tmp_running_mean", "_tmp_running_var", "_running_iter")


def test_split_entry_points_reject_bad_arguments_without_a_launch():
    lib = _lib.load_resnet()
    n0 = _lib.launch_count()
    rc = lib.dva_resnet_conv_bn_fwd_sums(None, 1, 8, 8, 3, None, 64, 3, 2, 2, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and "unsupported shape (T 3, stride 2, dilation 2)" in _lib.last_error()
    rc = lib.dva_resnet_conv_bn_fwd_sums(None, 1, 8, 8, 3, None, 64, 3, 1, 1, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_conv_bn_fwd_sums: null pointer"
    rc = lib.dva_resnet_bn_sync_stats(None, 8, 1, 0.1, 1e-5, None, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and "more than 1 value per channel" in _lib.last_error()
    rc = lib.dva_resnet_bn_sync_stats(None, 0, 4, 0.1, 1e-5, None, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_sync_stats: bad sizes"
    rc = lib.dva_resnet_bn_sync_stats(None, 8, 4, 0.1, 1e-5, None, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_sync_stats: null pointer"
    rc = lib.dva_resnet_bn_bwd_sums(None, None, None, 0, 8, None, None, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_bwd_sums: bad sizes"
    rc = lib.dva_resnet_bn_bwd_sums(None, None, None, 16, 8, None, None, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_bwd_sums: null pointer"
    rc = lib.dva_resnet_bn_sync_bwd(None, None, None, 16, 8, None, None, None, None, 8, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_sync_bwd: bad global count"
    rc = lib.dva_resnet_bn_sync_bwd(None, None, None, 16, 8, None, None, None, None, 32, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_bn_sync_bwd: null pointer"
    assert _lib.launch_count() == n0


def _bns(m):
    return [b for b in m.modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]


def _converted(m):
    before = m.state_dict()
    c = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    after = c.state_dict()
    assert set(after) == {k for k in before if not k.endswith(DROPPED)}
    assert all(torch.equal(after[k], before[k]) for k in after)
    assert _bns(c) and all(type(b) is nn.SyncBatchNorm for b in _bns(c))
    return c


@pytest.mark.parametrize("name", FAMILIES)
def test_conversion_gives_the_trunk_walk_every_batchnorm(name):
    m = getattr(I, name)()
    momenta = [b.momentum for b in _bns(m)]
    c = _converted(m)
    assert [b.momentum for b in _bns(c)] == momenta
    walked = [bn for bn, _, _ in c._bn_sizes(64, 64)]
    assert len(walked) == len(_bns(c)) and {id(b) for b in walked} == {id(b) for b in _bns(c)}
    for layer in c._trunk():
        if isinstance(layer, list):
            assert all(isinstance(bn, nn.SyncBatchNorm) and isinstance(conv, nn.Conv2d) for conv, bn in layer)


def test_conversion_of_the_ppm_encoder():
    c = _converted(I.ADE20KResNet18PPM())
    enc, dec = c.encoder, c.decoder
    assert all(isinstance(bn, nn.SyncBatchNorm) for bn in (enc.bn1, enc.bn2, enc.bn3, dec.conv_last[1]))
    assert all(isinstance(m[2], nn.SyncBatchNorm) and m[2].momentum == 0.001 for m in dec.ppm)
    walked = [bn for bn, _, _ in I._trunk_bn_sizes(enc._trunk(), 64, 64)]
    assert {id(b) for b in walked} == {id(b) for b in _bns(enc)} and len(walked) == len(_bns(enc)) == 23
    # the Prudent batch-size-1 rule goes with the conversion: the scale-1 branch trains on one image
    assert ops.ppm_branch_training(dec.ppm[0][2], 1, 1)
    assert not ops.ppm_branch_training(I.PPMFeatMap(fc_dim=8).ppm[0][2], 1, 1)


def test_nothing_is_synchronised_without_a_process_group():
    assert not torch.distributed.is_initialized()
    bn = nn.SyncBatchNorm(4)
    assert ops.bn_sync_group(bn) is None
    with ops.sync_batchnorm_split_at_one_rank():
        assert ops.bn_sync_group(bn) is None
    # torch's bookkeeping, and the size check before any launch on the local count
    assert ops._rn_bn_cfg(bn) == (True, 0.1, 1e-5, None) and int(bn.num_batches_tracked) == 1
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        I._check_bn_values(bn, True, 1, 1, 1)


def test_conversion_of_a_pool_mlp():
    mlp = nn.SyncBatchNorm.convert_sync_batchnorm(MLP([8, 16, 4], bias=False))
    for layer in mlp:
        assert isinstance(layer[1], FastBatchNorm1d) and isinstance(layer[1].batch_norm, nn.SyncBatchNorm)
    assert set(mlp.state_dict()) == set(MLP([8, 16, 4], bias=False).state_dict())
