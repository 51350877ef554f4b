"""The ADE20K ResNet-18 encoders (ADE20KResNet18TruncatedLayer*, Layer*, Pyramid on libdva_resnet.so) on the GPU,
against the float64 restatement oracle/image_resnet18_oracle.py on the same parameters.

Parameters come from the seeded integer-hash generator of the oracle.  The oracle takes the ReLU masks and max-pool
indices of the kernels' own forward (kernel_branches), so both compute the same piecewise-linear function: a
pre-activation within rounding of zero, or a window whose maxima tie within rounding, cannot send the two down
different branches.

Bounds: those of tests/test_gpu_image_unet.py.  Outputs: max |got - ref| / max |ref| <= max(L * K_max * u32, 4 e32);
gradients, normwise, <= max(4 * L * K_max * u32, 4 e32), with L the convolution count of the module, K_max =
T^2 * C_in of its widest convolution and e32 the error of the same restatement in fp32 on cuDNN with TF32 off (on the
same branches).  Running stats within a few fp32 ulps of the float64 update."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
import torch.utils.checkpoint

from conftest import GOLDEN
from deepviewagg_b200 import _lib, ops
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_resnet18_oracle as O
from test_gpu_image_encoder import l2rel, maxrel

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24


def bounds(m):
    convs = [c for c in m.modules() if isinstance(c, torch.nn.Conv2d)]
    b = len(convs) * max(c.kernel_size[0] ** 2 * c.in_channels for c in convs) * U32
    return b, 4 * b


def make(cls, seed=0, **kw):
    m = cls(**kw)
    m.load_state_dict(O.hashed_state(m.state_dict(), seed + 10), strict=True)
    return m.cuda()


def kernel_branches(m, x):
    """The ReLU masks and max-pool indices of the kernels' forward of m on x, in the oracle's order (the module's
    state, running stats included, is left as it was)."""
    st = {k: v.clone() for k, v in m.state_dict().items()}
    out = []
    with torch.no_grad():
        h = I._rows(x)
        for layer in m.conv:
            if isinstance(layer[0], I.BasicBlock):
                for blk in layer:
                    # the block's hidden activation: the same kernels on the same operands as inside rn_basic_block
                    out.append(ops.rn_conv_bn_relu(h, blk.conv1, blk.bn1) > 0)
                    h = ops.rn_basic_block(h, blk)
                    out.append(h > 0)
            else:
                for i in (0, 3, 6):
                    h = ops.rn_conv_bn_relu(h, layer[i], layer[i + 1])
                    out.append(h > 0)
                # torch's CUDA max pool takes the first max of a window, as rn_maxpool does
                out.append(F.max_pool2d(h.permute(0, 3, 1, 2), 3, 2, 1, return_indices=True)[1].permute(0, 2, 3, 1))
                h = ops.rn_maxpool(h)
    m.load_state_dict(st)
    return [t.permute(0, 3, 1, 2).contiguous().cpu() for t in out]


def _bn_training(m):
    return next(b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)).training


def _running(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}


def oracle(m, x, gy, dtype=torch.float64, device="cpu", masks=None):
    """(y, gx, {param: grad}, {buffer: value after the step}) of the restatement in `dtype` on `device`."""
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    p = {k: v.detach().to(device, dtype if v.is_floating_point() else v.dtype).clone()
         for k, v in m.state_dict().items()}
    for k in names:
        p[k].requires_grad_(True)
    xo = x.detach().to(device, dtype).requires_grad_(True)
    pyramid = isinstance(m, I.ADE20KResNet18Pyramid)
    y = O.forward(xo, p, m._LAYERS, _bn_training(m), m.scale_factor, pyramid, masks)
    g = torch.autograd.grad(y, [xo] + [p[k] for k in names], gy.to(device, dtype))
    return y.detach(), g[0], dict(zip(names, g[1:])), {k: v for k, v in p.items() if "running" in k}


def cudnn_fp32(m, x, gy, masks):
    """The restatement in fp32 on cuDNN with TF32 off, on the same branches."""
    tf = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return oracle(m, x, gy, torch.float32, "cuda", masks)
    finally:
        torch.backends.cudnn.allow_tf32 = tf


def run(m, x, gy):
    x = x.detach().clone().requires_grad_(True)
    y = m(x)
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    params = dict(m.named_parameters())
    g = torch.autograd.grad(y, [x] + [params[k] for k in names], gy)
    return y, g[0], dict(zip(names, g[1:]))


def check(m, x, gy):
    """One forward + backward of m against the float64 oracle."""
    before = _running(m)
    y, gx, gp = run(m, x, gy)
    after = _running(m)
    # the oracle and cuDNN runs start from the running stats m had before the step
    with torch.no_grad():
        for k, v in before.items():
            m.state_dict()[k].copy_(v)
    masks = kernel_branches(m, x)
    ry, rgx, rgp, rrun = oracle(m, x, gy, masks=masks)
    cy, cgx, cgp, _ = cudnn_fp32(m, x, gy, masks)
    with torch.no_grad():
        for k, v in after.items():
            m.state_dict()[k].copy_(v)
    assert y.shape == ry.shape and y.is_contiguous(memory_format=torch.channels_last)
    bo, bg = bounds(m)
    assert maxrel(y.detach(), ry) <= max(bo, 4 * maxrel(cy, ry)), (maxrel(y.detach(), ry), maxrel(cy, ry))
    assert l2rel(gx, rgx) <= max(bg, 4 * l2rel(cgx, rgx)), (l2rel(gx, rgx), l2rel(cgx, rgx))
    assert set(gp) == set(rgp)
    for k in gp:
        assert l2rel(gp[k], rgp[k]) <= max(bg, 4 * l2rel(cgp[k], rgp[k])), (k, l2rel(gp[k], rgp[k]),
                                                                            l2rel(cgp[k], rgp[k]))
    for k, v in rrun.items():
        got = after[k].double().cpu()
        ulp = 2.0 ** -23 * float(v.abs().max())
        assert float((got - v).abs().max()) <= 4 * ulp, (k, float((got - v).abs().max()), ulp)
    for k, v in after.items():
        if "num_batches_tracked" in k:
            assert int(v) == 0
    return y, gx, gp


@pytest.mark.parametrize("B,H,W", [(2, 61, 45), (1, 64, 96)])
def test_truncated_layer4_train_step(B, H, W):
    m = make(I.ADE20KResNet18TruncatedLayer4).train()
    x = torch.randn(B, 3, H, W, device="cuda")
    Ho = ops.rn_out(ops.rn_out(ops.rn_out(H, 2), 2), 2)
    Wo = ops.rn_out(ops.rn_out(ops.rn_out(W, 2), 2), 2)
    gy = torch.randn(B, 512, Ho, Wo, device="cuda")
    before = _running(m)
    y, _, gp = check(m, x, gy)
    assert y.shape == (B, 512, Ho, Wo) and len(gp) == len(list(m.parameters())) == 69
    assert not torch.equal(before["conv.4.1.bn2.running_var"], _running(m)["conv.4.1.bn2.running_var"])


def test_eval_mode_and_frozen():
    m = make(I.ADE20KResNet18TruncatedLayer2, seed=3).eval()
    x = torch.randn(2, 3, 40, 52, device="cuda")
    gy = torch.randn(2, 128, 5, 7, device="cuda")
    before = _running(m)
    check(m, x, gy)
    assert all(torch.equal(v, _running(m)[k]) for k, v in before.items())
    f = make(I.ADE20KResNet18TruncatedLayer2, seed=3, frozen=True)
    assert not f.training and f.frozen and not any(p.requires_grad for p in f.parameters())
    f.train()
    assert not f.training and not _bn_training(f)
    xg = x.clone().requires_grad_(True)
    y = f(xg)
    (gx,) = torch.autograd.grad(y, [xg], gy)
    assert all(p.grad is None for p in f.parameters())
    assert all(torch.equal(v, _running(f)[k]) for k, v in before.items())
    masks = kernel_branches(f, x)
    ry, rgx, _, _ = oracle(f, x, gy, masks=masks)
    cy, cgx, _, _ = cudnn_fp32(f, x, gy, masks)
    bo, bg = bounds(f)
    assert maxrel(y.detach(), ry) <= max(bo, 4 * maxrel(cy, ry)) and l2rel(gx, rgx) <= max(bg, 4 * l2rel(cgx, rgx))


@pytest.mark.parametrize("training", [False, True])
def test_truncated_layer0_on_the_pretrained_stem(training):
    """The checkpoint's real layer0 parameters and running stats (running_var up to ~3e4)."""
    g = np.load(f"{GOLDEN}/image_resnet18_layer0.npz")
    m = I.ADE20KResNet18TruncatedLayer0()
    m.load_state_dict({k: torch.from_numpy(g[k]) for k in m.state_dict()}, strict=True)
    m = m.cuda().train(training)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 50, 66, generator=gen).cuda()
    gy = torch.randn(2, 128, 13, 17, generator=gen).cuda()
    check(m, x, gy)


def test_layer3_alone():
    m = make(I.ADE20KResNet18Layer3, seed=4).train()
    assert m.input_nc == 128 and m.output_nc == 256 and m.conv_scale_factor == 1
    check(m, torch.randn(2, 128, 13, 11, device="cuda"), torch.randn(2, 256, 13, 11, device="cuda"))


@pytest.mark.parametrize("sf", [2, -1])
def test_scale_factor(sf):
    m = make(I.ADE20KResNet18TruncatedLayer2, seed=6, scale_factor=sf).train()
    s = 2 if sf == 2 else 8
    x = torch.randn(2, 3, 37, 50, device="cuda")
    gy = torch.randn(2, 128, 5 * s, 7 * s, device="cuda")
    y, _, _ = check(m, x, gy)
    assert y.shape == (2, 128, 5 * s, 7 * s)
    assert ("scale_factor=" in repr(m))


@pytest.mark.parametrize("sf", [1, 2])
def test_pyramid(sf):
    m = make(I.ADE20KResNet18Pyramid, seed=7, scale_factor=sf).train()
    x = torch.randn(2, 3, 48, 72, device="cuda")
    size = (int(48 * sf / 8), int(72 * sf / 8))
    gy = torch.randn(2, 1088, *size, device="cuda")
    y, _, _ = check(m, x, gy)
    assert y.shape == (2, 1088, *size) and m.output_nc == 512


def test_maxpool_ties_and_nan_route_to_the_first_max():
    gen = torch.Generator().manual_seed(8)
    x = torch.randint(-2, 3, (2, 4, 9, 7), generator=gen).float()
    x[:, :, 2:6, 1:5] = 1.5                       # constant patches: every window inside ties
    x[1, 2, 4, 4] = float("nan")
    gy = torch.randint(-3, 4, (2, 4, 5, 4), generator=gen).float()
    xo = x.double().requires_grad_(True)
    ry, idx = torch.nn.functional.max_pool2d(xo, 3, 2, 1, return_indices=True)
    (rgx,) = torch.autograd.grad(ry, [xo], gy.double())
    xr = x.permute(0, 2, 3, 1).contiguous().cuda().requires_grad_(True)
    y = ops.rn_maxpool(xr)
    (gx,) = torch.autograd.grad(y, [xr], gy.permute(0, 2, 3, 1).cuda())
    got = y.permute(0, 3, 1, 2).double().cpu()
    assert torch.isnan(got).sum() > 0 and torch.equal(torch.nan_to_num(got, 99.), torch.nan_to_num(ry.detach(), 99.))
    assert torch.equal(gx.permute(0, 3, 1, 2).double().cpu(), rgx)


def test_reproducible_and_deterministic():
    m = make(I.ADE20KResNet18Pyramid, seed=9, scale_factor=2).train()
    x = torch.randn(2, 3, 40, 48, device="cuda")
    gy = torch.randn(2, 1088, 10, 12, device="cuda")
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
    # NCHW and channels-last inputs give the same bits
    m.load_state_dict(st)
    d = run(m, x.contiguous(memory_format=torch.channels_last), gy)
    assert torch.equal(a[0], d[0]) and torch.equal(a[1], d[1])


def test_dtypes_and_autocast():
    m = make(I.ADE20KResNet18TruncatedLayer1, seed=10).eval()
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


def test_checkpointing_recompute_updates_the_running_stats_twice():
    """Under reentrant checkpointing (the reference's checkpointing: c) the recompute is a second train-mode call:
    outputs and gradients are those of the plain call, and the running stats move twice."""
    m = make(I.ADE20KResNet18TruncatedLayer2, seed=11).train()
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
    m.load_state_dict({**st, **once})
    with torch.no_grad():
        m(x)
    assert all(torch.equal(v, _running(m)[k]) for k, v in twice.items())


def test_value_errors_before_any_launch():
    m = make(I.ADE20KResNet18TruncatedLayer4).train()
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(torch.randn(1, 3, 8, 8, device="cuda"))
    with pytest.raises(ValueError, match=r"\[B, 3, H, W\]"):
        m(torch.randn(1, 4, 32, 32, device="cuda"))
    with pytest.raises(ValueError, match=r"\[B, 128, H, W\]"):
        make(I.ADE20KResNet18Layer3)(torch.randn(1, 3, 32, 32, device="cuda"))
    assert _lib.launch_count() == n0
    m.eval()
    assert m(torch.randn(1, 3, 8, 8, device="cuda")).shape == (1, 512, 1, 1)


def resnet_scenario():
    """A Pyramid train step with the input's gradient: every kernel of libdva_resnet.so."""
    m = make(I.ADE20KResNet18Pyramid, seed=12, scale_factor=2).train()
    x = torch.randn(2, 3, 40, 48, device="cuda", requires_grad=True)
    y = m(x)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    return bool(torch.isfinite(x.grad).all())


def test_resnet_scenario():
    assert resnet_scenario()


class _OracleResNet(torch.nn.Module):
    """The float64 restatement on the parameters of `enc`, on the kernels' branches, fp32 out."""

    def __init__(self, enc):
        super().__init__()
        self.enc = enc

    def forward(self, x, *args, **kwargs):
        masks = kernel_branches(self.enc, x)
        p = {k: v.double().cpu() for k, v in self.enc.state_dict(keep_vars=True).items()}
        y = O.forward(x.double().cpu(), p, self.enc._LAYERS, _bn_training(self.enc), self.enc.scale_factor,
                      masks=masks)
        return y.float().cuda()


def _branch_run(conv, enc, checkpointing=""):
    """UnimodalBranch(conv, max atomic pool, group view pool, concatenation) on the two-setting toy mapping of
    tests/golden/unimodal_branch_toy.npz, its images cut to 3 channels; returns the fused 3D features and the
    gradients of a weighted sum w.r.t. the 3D features, the images of both settings and the encoder's parameters."""
    from conftest import load_golden
    from test_containers import _toy_image_data
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool, GroupBimodalCSRPool
    g = load_golden("unimodal_branch_toy")
    mod = _toy_image_data(g, "cuda")
    xs = []
    for im in mod:
        x = im.x[:, :3].detach().clone().contiguous().requires_grad_(True)
        im._x = x
        xs.append(x)
    torch.manual_seed(13)
    view_pool = GroupBimodalCSRPool(in_map=8, in_mod=enc.output_nc, num_groups=4, use_num=True)
    branch = UnimodalBranch(conv, BimodalCSRPool(mode="max"), view_pool, BimodalFusion("concatenation"),
                            checkpointing=checkpointing).cuda()
    branch.train()
    params = list(enc.parameters())
    for p in params:
        p.grad = None
    x_3d = g["x_3d"].cuda().requires_grad_(True)
    out = branch({"x_3d": x_3d, "x_seen": None, "modalities": {"image": mod}}, "image")
    w = torch.from_numpy(O.hash_grid(14, 0, tuple(out["x_3d"].shape), 8, 3)).float().cuda()
    (out["x_3d"] * w).sum().backward()     # reentrant checkpointing supports .backward() only
    return out["x_3d"].detach(), [x_3d.grad] + [x.grad for x in xs] + [p.grad.clone() for p in params]


def test_unimodal_branch_over_a_mapping():
    """UnimodalBranch(conv=ADE20KResNet18TruncatedLayer0(scale_factor=-1)) forward + backward over the toy mapping
    (channels-last output into the gather kernels) against the same branch on the float64 restatement.  With
    checkpointing='c' (reentrant recompute) the branch gives the same bits, and the recompute, a second train-mode
    call, moves the running stats a second time, as in the reference."""
    enc = make(I.ADE20KResNet18TruncatedLayer0, seed=12, scale_factor=-1).train()
    st = {k: v.clone() for k, v in enc.state_dict().items()}
    out, grads = _branch_run(enc, enc)
    once = _running(enc)
    enc.load_state_dict(st)
    ref, rgrads = _branch_run(_OracleResNet(enc), enc)
    bo, bg = bounds(enc)
    assert out.shape == (1000, 12 + 128)
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
    # the plain branch runs the encoder once per setting and moves every running stat; under 'c' the recompute moves
    # them again
    twice = _running(enc)
    for k, v in twice.items():
        if k.endswith(("running_mean", "running_var")) and "_tmp" not in k:
            assert not torch.equal(once[k], st[k]) and not torch.equal(v, once[k]), k
