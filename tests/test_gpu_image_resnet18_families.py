"""The ImageNet and Cityscapes ResNet-18 encoders (ResNet18*, CityscapesResNet18* on libdva_resnet.so) on the GPU,
against the float64 restatement oracle/image_resnet18_families_oracle.py on the same parameters and on the kernels'
own ReLU masks and max-pool indices, with the bounds of tests/test_gpu_image_resnet18.py: outputs max |got - ref| /
max |ref| <= max(L * K_max * u32, 4 e32), gradients normwise <= 4 times that, with L the convolution count, K_max =
T^2 * C_in of the widest convolution (at least 147 for the 7x7 stem) and e32 the same restatement in fp32 on cuDNN
with TF32 off.  Running stats under the same rule (momentum 0.1 passes a tenth of the batch statistics' error on);
num_batches_tracked exact."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import torch.utils.checkpoint

from conftest import GOLDEN
from deepviewagg_b200 import _lib, ops
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_resnet18_families_oracle as O
from test_gpu_image_encoder import l2rel, maxrel
from test_gpu_image_resnet18 import _bn_training, _branch_run, _running, bounds, run
from test_gpu_kernel_matrix import record

pytestmark = pytest.mark.gpu


def make(cls, seed=0, **kw):
    m = cls(**kw)
    m.load_state_dict(O.hashed_state(m.state_dict(), seed + 30), strict=True)
    return m.cuda()


def kernel_branches(m, x):
    """The ReLU masks and max-pool indices of the kernels' forward of m on x, in the oracle's order (the module's
    state, running stats and counters included, is left as it was)."""
    st = {k: v.clone() for k, v in m.state_dict().items()}
    out = []
    with torch.no_grad():
        h = I._rows(x)
        for layer in m._trunk():
            if isinstance(layer, list):
                for conv, bn in layer:
                    h = ops.rn_conv_bn_relu(h, conv, bn)
                    out.append(h > 0)
                pad = layer.pool_padding
                out.append(F.max_pool2d(h.permute(0, 3, 1, 2), 3, 2, pad, return_indices=True)[1].permute(0, 2, 3, 1))
                h = ops.rn_maxpool(h, pad)
            else:
                for blk in layer:
                    out.append(ops.rn_conv_bn_relu(h, blk.conv1, blk.bn1) > 0)
                    h = ops.rn_basic_block(h, blk)
                    out.append(h > 0)
    m.load_state_dict(st)
    return [t.permute(0, 3, 1, 2).contiguous().cpu() for t in out]


def _oracle_args(m):
    fam = "cityscapes" if type(m).__name__.startswith("Cityscapes") else "imagenet"
    if isinstance(m, I.CityscapesResNet18):
        return fam, list(I._TRUNK_LAYERS), list(I._TRUNK_LAYERS)
    return fam, list(m._LAYERS), None


def _momentum(m):
    return next(b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)).momentum


def oracle(m, x, gy, dtype=torch.float64, device="cpu", masks=None):
    """(y, gx, {param: grad}, {buffer: value after the step}) of the restatement in `dtype` on `device`."""
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    p = {k: v.detach().to(device, dtype if v.is_floating_point() else v.dtype).clone()
         for k, v in m.state_dict().items()}
    for k in names:
        p[k].requires_grad_(True)
    xo = x.detach().to(device, dtype).requires_grad_(True)
    fam, layers, prefixes = _oracle_args(m)
    pyramid = isinstance(m, I._Pyramid)
    y = O.forward(xo, p, fam, layers, _bn_training(m), m.scale_factor, pyramid, _momentum(m), masks, prefixes)
    g = torch.autograd.grad(y, [xo] + [p[k] for k in names], gy.to(device, dtype))
    return y.detach(), g[0], dict(zip(names, g[1:])), {k: v for k, v in p.items() if "running" in k or "num_b" in k}


def cudnn_fp32(m, x, gy, masks):
    tf = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return oracle(m, x, gy, torch.float32, "cuda", masks)
    finally:
        torch.backends.cudnn.allow_tf32 = tf


def check(m, x, gy):
    """One forward + backward of m against the float64 oracle; returns (y, gx, {param: grad})."""
    before = _running(m)
    y, gx, gp = run(m, x, gy)
    after = _running(m)
    with torch.no_grad():
        for k, v in before.items():
            m.state_dict()[k].copy_(v)
    masks = kernel_branches(m, x)
    ry, rgx, rgp, rrun = oracle(m, x, gy, masks=masks)
    cy, cgx, cgp, crun = cudnn_fp32(m, x, gy, masks)
    with torch.no_grad():
        for k, v in after.items():
            m.state_dict()[k].copy_(v)
    assert y.shape == ry.shape and y.is_contiguous(memory_format=torch.channels_last)
    bo, bg = bounds(m)
    assert maxrel(y.detach(), ry) <= max(bo, 4 * maxrel(cy, ry)), (maxrel(y.detach(), ry), maxrel(cy, ry))
    assert l2rel(gx, rgx) <= max(bg, 4 * l2rel(cgx, rgx)), (l2rel(gx, rgx), l2rel(cgx, rgx))
    assert set(gp) == set(rgp)
    for k in gp:
        assert l2rel(gp[k], rgp[k]) <= max(bg, 4 * l2rel(cgp[k], rgp[k])), (k, l2rel(gp[k], rgp[k]))
    for k, v in rrun.items():
        got = after[k].cpu()
        if "num_batches_tracked" in k:
            assert torch.equal(got, v), k
            continue
        # momentum 0.1 carries a tenth of the batch statistics' error into the running stats: the output bound on
        # them, or 4 times cuDNN's fp32 error, or a few fp32 ulps
        err, cerr = float((got.double() - v).abs().max()), float((crun[k].double().cpu() - v).abs().max())
        scale = float(v.abs().max())
        assert err <= max(bo * scale, 4 * cerr, 4 * 2.0 ** -23 * scale), (k, err, cerr, bo * scale)
    return y, gx, gp


@pytest.mark.parametrize("B,H,W", [(2, 61, 45), (1, 64, 97)])
def test_imagenet_truncated_layer4_train_step(B, H, W):
    m = make(I.ResNet18TruncatedLayer4).train()
    x = torch.randn(B, 3, H, W, device="cuda")
    side = lambda n: ops.rn_out(ops.rn_out(ops.rn_out(ops.rn_out(ops.rn_pool_out(ops.rn_out(n, 2)), 2), 2), 2), 1)
    gy = torch.randn(B, 512, side(H), side(W), device="cuda")
    y, _, gp = check(m, x, gy)
    assert y.shape == (B, 512, side(H), side(W)) and len(gp) == len(list(m.parameters())) == 60
    assert all(int(b.num_batches_tracked) == 1 for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))


@pytest.mark.parametrize("B,H,W", [(2, 60, 44), (2, 61, 47)])
def test_cityscapes_truncated_layer4_train_step(B, H, W):
    """60 x 44: the stem's 30 x 22 map loses its last row and column to the unpadded pool; 61 x 47: it does not."""
    m = make(I.CityscapesResNet18TruncatedLayer4, seed=1).train()
    x = torch.randn(B, 3, H, W, device="cuda")
    side = lambda n: ops.rn_out(ops.rn_out(ops.rn_out(ops.rn_pool_out(ops.rn_out(n, 2), 0), 2), 2), 2)
    y, _, _ = check(m, x, torch.randn(B, 512, side(H), side(W), device="cuda"))
    assert y.shape == (B, 512, side(H), side(W))


@pytest.mark.parametrize("cls,shape", [("ResNet18Layer2", (1, 64, 15, 18)), ("CityscapesResNet18Layer1", (2, 128, 9, 11)),
                                       ("ResNet18Layer0", (2, 3, 33, 20)), ("CityscapesResNet18Layer4", (2, 256, 5, 6))])
def test_layers_alone(cls, shape):
    m = make(getattr(I, cls), seed=2).train()
    y = m(torch.randn(*shape, device="cuda"))
    check(m, torch.randn(*shape, device="cuda"), torch.randn(*y.shape, device="cuda"))


def test_cityscapes_full_and_pyramids():
    m = make(I.CityscapesResNet18, seed=3).train()
    check(m, torch.randn(2, 3, 50, 66, device="cuda"), torch.randn(2, 512, 2, 2, device="cuda"))
    for cls, c, seed in ((I.ResNet18Pyramid, 1024, 4), (I.CityscapesResNet18Pyramid, 1088, 5)):
        p = make(cls, seed=seed).train()
        y, _, _ = check(p, torch.randn(2, 3, 40, 56, device="cuda"), torch.randn(2, c, 40, 56, device="cuda"))
        assert y.shape == (2, c, 40, 56)


@pytest.mark.parametrize("fam", ["imagenet", "cityscapes"])
@pytest.mark.parametrize("training", [False, True])
def test_truncated_layer0_on_the_pretrained_stem(fam, training):
    g = np.load(f"{GOLDEN}/image_resnet18_families_{fam}_layer0.npz")
    m = (I.ResNet18TruncatedLayer0 if fam == "imagenet" else I.CityscapesResNet18TruncatedLayer0)()
    m.load_state_dict({k: torch.from_numpy(g[k]) for k in m.state_dict()}, strict=True)
    m = m.cuda().train(training)
    x = torch.randn(2, 3, 50, 66, device="cuda")
    y = m(x.clone())
    m.load_state_dict({k: torch.from_numpy(g[k]) for k in m.state_dict()}, strict=True)
    check(m, x, torch.randn(*y.shape, device="cuda"))


def test_eval_mode_frozen_and_momentum_none():
    m = make(I.ResNet18TruncatedLayer2, seed=6).eval()
    x = torch.randn(2, 3, 40, 52, device="cuda")
    gy = torch.randn(2, 128, 5, 7, device="cuda")
    before = _running(m)
    check(m, x, gy)
    assert all(torch.equal(v, _running(m)[k]) for k, v in before.items())
    f = make(I.CityscapesResNet18TruncatedLayer2, seed=6, frozen=True)
    f.train()
    assert not f.training and not _bn_training(f)
    xg = x.clone().requires_grad_(True)
    n0 = _lib.launch_count()
    before = _running(f)
    gf = torch.randn_like(f(x))
    _, names = record(lambda: torch.autograd.grad(f(xg), [xg], gf), canon=lambda n: n, seen=set())
    assert not any("rn_conv_wgrad_kernel" in n for n in names) and any("rn_conv_gemm_kernel" in n for n in names)
    assert all(p.grad is None for p in f.parameters()) and _lib.launch_count() > n0
    assert all(torch.equal(v, _running(f)[k]) for k, v in before.items())
    # momentum None: the cumulative average, 1 / num_batches_tracked, over two steps
    c = make(I.CityscapesResNet18Layer0, seed=7).train()
    for b in c.modules():
        if isinstance(b, torch.nn.BatchNorm2d):
            b.momentum = None
    for _ in range(2):
        check(c, torch.randn(2, 3, 26, 30, device="cuda"), torch.randn(2, 128, 6, 7, device="cuda"))
    assert all(int(b.num_batches_tracked) == 2 for b in c.modules() if isinstance(b, torch.nn.BatchNorm2d))


@pytest.mark.parametrize("pad", [0, 1])
def test_maxpool_ties_nan_and_uncovered_borders(pad):
    gen = torch.Generator().manual_seed(8 + pad)
    x = torch.randint(-2, 3, (2, 4, 10, 8), generator=gen).float()
    x[:, :, 2:6, 1:5] = 1.5                       # constant patches: every window inside ties
    x[:, :, -1, :] = 9.0                          # at padding 0 the last row and column belong to no window
    x[:, :, :, -1] = 9.0
    x[1, 2, 4, 4] = float("nan")
    x[0, 1, 0, 0] = float("nan")                  # NaN on the first tap of the corner window
    xo = x.double().requires_grad_(True)
    ry, _ = F.max_pool2d(xo, 3, 2, pad, return_indices=True)
    gy = torch.randint(-3, 4, tuple(ry.shape), generator=gen).float()
    (rgx,) = torch.autograd.grad(ry, [xo], gy.double())
    xr = x.permute(0, 2, 3, 1).contiguous().cuda().requires_grad_(True)
    y = ops.rn_maxpool(xr, pad)
    (gx,) = torch.autograd.grad(y, [xr], gy.permute(0, 2, 3, 1).cuda())
    got = y.permute(0, 3, 1, 2).double().cpu()
    assert got.shape == ry.shape and torch.isnan(got).sum() > 0
    assert torch.equal(torch.nan_to_num(got, 99.), torch.nan_to_num(ry.detach(), 99.))
    assert torch.equal(gx.permute(0, 3, 1, 2).double().cpu(), rgx)
    if pad == 0:
        assert float(gx[:, -1].abs().sum()) == 0 and float(gx[:, :, -1].abs().sum()) == 0


def test_reproducible_and_deterministic():
    for cls in (I.ResNet18Pyramid, I.CityscapesResNet18Pyramid):
        m = make(cls, seed=9).train()
        x = torch.randn(2, 3, 40, 48, device="cuda")
        gy = torch.randn(2, 1024 if cls is I.ResNet18Pyramid else 1088, 40, 48, device="cuda")
        st = {k: v.clone() for k, v in m.state_dict().items()}
        a = run(m, x, gy)
        m.load_state_dict(st)
        b = run(m, x, gy)
        torch.use_deterministic_algorithms(True)
        try:
            m.load_state_dict(st)
            c = run(m, x, gy)
        finally:
            torch.use_deterministic_algorithms(False)
        for r in (b, c):
            assert torch.equal(a[0], r[0]) and torch.equal(a[1], r[1])
            assert all(torch.equal(a[2][k], r[2][k]) for k in a[2])
        m.load_state_dict(st)
        d = run(m, x.contiguous(memory_format=torch.channels_last), gy)
        assert torch.equal(a[0], d[0]) and torch.equal(a[1], d[1])


def test_dtypes_and_autocast():
    for cls in (I.ResNet18TruncatedLayer1, I.CityscapesResNet18TruncatedLayer1):
        m = make(cls, seed=10).eval()
        x = torch.randn(2, 3, 32, 40, device="cuda")
        y32 = m(x)
        for dt in (torch.float16, torch.bfloat16, torch.float64):
            xd = x.to(dt).requires_grad_(True)
            y = m(xd)
            assert y.dtype == dt and y.is_contiguous(memory_format=torch.channels_last)
            assert torch.equal(y, m(xd.detach().float()).to(dt))
            (gx,) = torch.autograd.grad(y.float().sum(), [xd])
            assert gx.dtype == dt
        with torch.autocast("cuda", dtype=torch.float16):
            ya = m(x.half())
        assert ya.dtype == torch.float32 and torch.equal(ya, m(x.half().float()))
        assert torch.equal(m(x.double()), y32.double())


def test_checkpoint_recompute_counts_twice():
    """Under reentrant checkpointing the recompute is a second train-mode call: the same outputs and gradients, the
    running stats moved twice and num_batches_tracked 2, as torch's BatchNorm2d gives."""
    m = make(I.ResNet18TruncatedLayer2, seed=11).train()
    x = torch.randn(2, 3, 30, 34, device="cuda", requires_grad=True)
    gy = torch.randn(2, 128, 4, 5, device="cuda")
    st = {k: v.clone() for k, v in m.state_dict().items()}
    y = m(x)
    y.backward(gy)
    g_plain = [x.grad.clone()] + [p.grad.clone() for p in m.parameters()]
    once = _running(m)
    m.load_state_dict(st)
    m.zero_grad(set_to_none=True)
    x.grad = None
    yc = torch.utils.checkpoint.checkpoint(m, x, use_reentrant=True)
    yc.backward(gy)
    g_ckpt = [x.grad.clone()] + [p.grad.clone() for p in m.parameters()]
    assert torch.equal(y, yc) and all(torch.equal(a, b) for a, b in zip(g_plain, g_ckpt))
    twice = _running(m)
    assert all(int(v) == 2 for k, v in twice.items() if "num_batches_tracked" in k)
    m.load_state_dict({**st, **once})
    with torch.no_grad():
        m(x)
    assert all(torch.equal(v, _running(m)[k]) for k, v in twice.items())


def test_value_errors_before_any_launch():
    n0 = _lib.launch_count()
    m = make(I.ResNet18TruncatedLayer4).train()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(torch.randn(1, 3, 32, 32, device="cuda"))
    with pytest.raises(ValueError, match=r"\[B, 3, H, W\]"):
        m(torch.randn(1, 4, 64, 64, device="cuda"))
    with pytest.raises(ValueError, match=r"\[B, 128, H, W\]"):
        make(I.CityscapesResNet18Layer1)(torch.randn(2, 64, 8, 8, device="cuda"))
    with pytest.raises(ValueError, match="smaller than one window"):
        make(I.CityscapesResNet18TruncatedLayer0).eval()(torch.randn(1, 3, 4, 64, device="cuda"))
    assert _lib.launch_count() == n0
    m.eval()
    assert m(torch.randn(1, 3, 32, 32, device="cuda")).shape == (1, 512, 1, 1)


_FOREIGN = re.compile(r"cudnn|cublas|cutlass|xmma|gemm|conv|norm|pool|upsample|interp|adaptive", re.I)


@pytest.mark.parametrize("cls", ["ResNet18Pyramid", "CityscapesResNet18Pyramid"])
def test_a_train_step_launches_only_the_projects_kernels(cls):
    m = make(getattr(I, cls), seed=12).train()
    x = torch.randn(2, 3, 45, 61, device="cuda", requires_grad=True)
    y = m(x)
    gy = torch.randn_like(y)
    st = {k: v.clone() for k, v in m.state_dict().items()}

    def step():
        m.load_state_dict(st)
        return torch.autograd.grad(m(x), [x] + list(m.parameters()), gy)

    _, names = record(step, canon=lambda n: n, seen=set())
    ours = {n for n in names if "dva_resnet::" in n}
    foreign = sorted(n for n in names - ours if _FOREIGN.search(n))
    assert not foreign, foreign
    for k in ("rn_weight_prep_kernel", "rn_conv_gemm_kernel<0>", "rn_conv_gemm_kernel<1>", "rn_conv_wgrad_kernel",
              "rn_wgrad_reduce_kernel", "rn_bn_stats_kernel", "rn_bn_apply_kernel", "rn_bn_bwd_partial_kernel",
              "rn_bn_bwd_reduce_kernel", "rn_bn_bwd_dz_kernel", "rn_maxpool_kernel", "rn_maxpool_bwd_kernel",
              "rn_resize_kernel", "rn_resize_bwd_kernel"):
        assert any(k in n for n in ours), (k, sorted(ours))


class _OracleResNet(torch.nn.Module):
    """The float64 restatement on the parameters of `enc`, on the kernels' branches, fp32 out."""

    def __init__(self, enc):
        super().__init__()
        self.enc = enc

    def forward(self, x, *args, **kwargs):
        masks = kernel_branches(self.enc, x)
        p = {k: v.double().cpu() if v.is_floating_point() else v.cpu().clone()
             for k, v in self.enc.state_dict(keep_vars=True).items()}
        fam, layers, prefixes = _oracle_args(self.enc)
        y = O.forward(x.double().cpu(), p, fam, layers, _bn_training(self.enc), self.enc.scale_factor,
                      masks=masks, prefixes=prefixes)
        return y.float().cuda()


@pytest.mark.parametrize("cls", ["ResNet18TruncatedLayer0", "CityscapesResNet18TruncatedLayer0"])
def test_unimodal_branch_over_a_mapping(cls):
    """UnimodalBranch(conv=<family>TruncatedLayer0(scale_factor=-1)) over the toy mapping, against the same branch on
    the float64 restatement; bitwise equal in deterministic mode with and without reentrant checkpointing."""
    enc = make(getattr(I, cls), seed=13, scale_factor=-1).train()
    st = {k: v.clone() for k, v in enc.state_dict().items()}
    out, grads = _branch_run(enc, enc)
    enc.load_state_dict(st)
    ref, rgrads = _branch_run(_OracleResNet(enc), enc)
    bo, bg = bounds(enc)
    assert out.shape == (1000, 12 + enc.output_nc)
    assert maxrel(out, ref) <= bo, maxrel(out, ref)
    for a, b in zip(grads, rgrads):
        assert l2rel(a, b) <= bg, l2rel(a, b)
    torch.use_deterministic_algorithms(True)
    try:
        enc.load_state_dict(st)
        out_d, grads_d = _branch_run(enc, enc)
        enc.load_state_dict(st)
        out_c, grads_c = _branch_run(enc, enc, checkpointing="c")
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(out_c, out_d) and all(torch.equal(a, b) for a, b in zip(grads_c, grads_d))
