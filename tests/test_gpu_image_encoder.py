"""The from-scratch image encoder (ResNetDown on libdva_conv2d.so) on the GPU, against the float64 reference.

Bounds.  Every product is 3xTF32 with fp32 accumulation: a dot product of length K = R*S*C_in errs by at most
~K * u32 (u32 = 2^-24) relative to sum |a||b|, and the GroupNorm that follows each convolution renormalises, so the
error of an L-convolution chain stays below L * K_max * u32 of the output's scale.  Outputs are compared as
max |got - ref| / max |ref| <= L * K_max * u32.  Gradients also pass ReLU kinks: an element whose pre-activation is
within rounding of 0 may take the other branch, a difference of the size of the gradient itself at that element,
so they are compared normwise, ||got - ref||_2 / ||ref||_2 <= 4 * L * K_max * u32 (the backward runs two products
per convolution and the GroupNorm backward one more reduction over the group of C/G * H * W elements, summed in
fp64).  For the fixtures (widths 4 .. 32, K_max = 288, L = 21) that is 3.6e-4 / 1.4e-3; for the shipped widths
(K_max = 2304) 2.9e-3 / 1.2e-2; measured errors are far below (u32-scale sums, the K bound is worst-case)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200 import _lib
from deepviewagg_b200.modules.multimodal.modalities.image import ResNetDown
from oracle import image_encoder_oracle as O

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
CHANNELS = lambda f: [[4, f], [f, f], [f, 2 * f], [2 * f, 4 * f], [4 * f, 8 * f]]  # noqa: E731
N = [0, 2, 2, 2, 2]
KERNEL = [3, 2, 2, 2, 2]
STRIDE = [1, 2, 2, 2, 2]
PADDING = [1, 0, 0, 0, 0]
N_CONV = 21   # 5 conv_in + 8 blocks x 2 (the downsamples are 1 x 1, K = C_in)


def stage_kwargs(i, f):
    return dict(down_conv_nn=CHANNELS(f)[i], kernel_size=KERNEL[i], stride=STRIDE[i], padding=PADDING[i], N=N[i],
                block="ResBlock", normalization="GroupNorm", weight_standardization=True)


def encoder(f, seed=0, device="cuda"):
    torch.manual_seed(seed)
    stages = torch.nn.Sequential(*[ResNetDown(**stage_kwargs(i, f)) for i in range(5)])
    gen = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for m in stages.modules():
            if isinstance(m, torch.nn.GroupNorm):
                m.weight.copy_(1 + 0.2 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen))
    return stages.to(device)


def bounds(f):
    kmax = 9 * 8 * f
    return N_CONV * kmax * U32, 4 * N_CONV * kmax * U32


def maxrel(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max() / b.double().abs().max())


def l2rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().norm())


def oracle_grads(stages, x, gy):
    sds = [{k: v.detach().double().cpu().requires_grad_(True) for k, v in st.state_dict().items()} for st in stages]
    xo = x.detach().double().cpu().requires_grad_(True)
    y = O.encoder(xo, [(sd, KERNEL[i], STRIDE[i], PADDING[i]) for i, sd in enumerate(sds)])
    params = [p for sd in sds for p in sd.values()]
    g = torch.autograd.grad(y, [xo] + params, gy.double().cpu())
    return y.detach(), g[0], g[1:]


def run(stages, x, gy):
    x = x.detach().clone().requires_grad_(True)
    y = stages(x)
    params = [p for st in stages for p in st.state_dict(keep_vars=True).values()]
    g = torch.autograd.grad(y, [x] + params, gy)
    return y, g[0], g[1:]


# ---- fixtures: the executed reference (oracle/make_golden_image_encoder.py)
@pytest.mark.parametrize("name", ["b2", "b1"])
def test_fixture_parity(name):
    z = np.load(os.path.join(GOLDEN, f"image_encoder_{name}.npz"), allow_pickle=False)
    stages = encoder(4)
    for i, st in enumerate(stages):
        keys = list(z[f"keys{i}"])
        assert list(st.state_dict().keys()) == keys
        st.load_state_dict({k: torch.from_numpy(z[f"p{i}:{k}"]).float() for k in keys}, strict=True)
    x = torch.from_numpy(z["x"]).float().cuda()
    gy = torch.from_numpy(z["gy"]).float().cuda()
    y, gx, gp = run(stages, x, gy)
    by, bg = bounds(4)
    assert maxrel(y, torch.from_numpy(z["y"])) <= by
    assert l2rel(gx, torch.from_numpy(z["gx"])) <= bg
    names = [(i, k) for i, st in enumerate(stages) for k in st.state_dict()]
    for (i, k), g in zip(names, gp):
        assert l2rel(g, torch.from_numpy(z[f"g{i}:{k}"])) <= bg, (i, k)


@pytest.mark.parametrize("B, H, W", [(2, 96, 128), (1, 67, 91)])
def test_full_width_against_oracle(B, H, W):
    stages = encoder(32, seed=3)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(B, 4, H, W, generator=gen).cuda()
    gy = torch.randn(B, 256, H // 16, W // 16, generator=torch.Generator().manual_seed(6)).cuda()
    y, gx, gp = run(stages, x, gy)
    ry, rgx, rgp = oracle_grads(stages, x, gy)
    by, bg = bounds(32)
    assert y.shape == ry.shape
    assert maxrel(y, ry) <= by
    assert l2rel(gx, rgx) <= bg
    for g, r in zip(gp, rgp):
        assert l2rel(g, r) <= bg


def test_layouts_bits_determinism_and_autocast():
    stages = encoder(8, seed=2)
    x = torch.randn(3, 4, 40, 56, device="cuda")
    gy = torch.randn(3, 64, 2, 3, device="cuda")
    y, gx, gp = run(stages, x, gy)
    assert y.is_contiguous(memory_format=torch.channels_last) and y.shape == (3, 64, 2, 3)
    y2, gx2, gp2 = run(stages, x.contiguous(memory_format=torch.channels_last), gy)
    assert torch.equal(y, y2) and torch.equal(gx, gx2) and all(torch.equal(a, b) for a, b in zip(gp, gp2))
    torch.use_deterministic_algorithms(True)
    try:
        y3, gx3, gp3 = run(stages, x, gy)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(y, y3) and torch.equal(gx, gx3) and all(torch.equal(a, b) for a, b in zip(gp, gp3))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ya = stages(x)
    assert ya.dtype == torch.float32 and torch.equal(ya, y)


def test_cpu_and_small_images_raise():
    stages = encoder(8)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        stages[0](torch.zeros(1, 4, 8, 8))
    with pytest.raises(ValueError, match=">= 2"):
        stages[0](torch.zeros(1, 4, 1, 8, device="cuda"))
    with pytest.raises(ValueError, match=">= 2"):
        stages(torch.zeros(1, 4, 24, 24, device="cuda"))     # stage 4 would be 1 x 1


def test_positional_reset_flag_and_checkpointing():
    from torch.utils.checkpoint import checkpoint
    st = encoder(8)[:2]
    x = torch.randn(2, 4, 20, 18, device="cuda", requires_grad=True)
    y = st[1](st[0](x, True), True)
    g = torch.autograd.grad(y.sum(), x)[0]
    x2 = x.detach().clone().requires_grad_(True)
    h = checkpoint(st[0], x2, torch.BoolTensor([True]), use_reentrant=True)
    y2 = checkpoint(st[1], h, torch.BoolTensor([False]), use_reentrant=True)
    y2.sum().backward()     # reentrant checkpointing supports .backward() only
    assert torch.equal(y, y2) and torch.equal(g, x2.grad)


def encoder_scenario():
    """Forward + backward of a two-stage encoder with the input's gradient: every kernel of libdva_conv2d.so."""
    torch.manual_seed(11)
    st = torch.nn.Sequential(ResNetDown(**{**stage_kwargs(0, 8), "down_conv_nn": [4, 8]}),
                             ResNetDown(**{**stage_kwargs(1, 8), "down_conv_nn": [8, 32]})).cuda()
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(2, 4, 27, 30, generator=gen).cuda()
    gy = torch.randn(2, 32, 13, 15, generator=gen).cuda()
    y, gx, gp = run(st, x, gy)
    sds = [{k: v.detach().double().cpu().requires_grad_(True) for k, v in s.state_dict().items()} for s in st]
    xo = x.double().cpu().requires_grad_(True)
    ry = O.encoder(xo, [(sds[0], 3, 1, 1), (sds[1], 2, 2, 0)])
    params = [p for sd in sds for p in sd.values()]
    rg = torch.autograd.grad(ry, [xo] + params, gy.double().cpu())
    tol = 7 * 9 * 32 * U32
    assert maxrel(y, ry) <= tol
    for a, b in zip((gx,) + tuple(gp), rg):
        assert l2rel(a, b) <= 4 * tol
    return True


def test_encoder_scenario():
    n0 = _lib.launch_count()
    assert encoder_scenario()
    assert _lib.launch_count() > n0


def test_half_double_and_strided_inputs():
    """The kernels read fp32 channels-last rows: any other dtype or layout is cast / copied first, outside autocast
    too.  The output takes the input's dtype; the gradients take the dtypes of the input and of the parameters."""
    from deepviewagg_b200 import ops
    stages = encoder(8, seed=2)[:3]
    x = torch.randn(2, 4, 40, 56, device="cuda")
    gy = torch.randn(2, 16, 10, 14, device="cuda")
    y32, gx32, gp32 = run(stages, x, gy)
    # one stage: every ResNetDown returns the input's dtype, so a chain rounds to it between stages
    first = stages[:1]
    g1 = torch.randn(2, 8, 40, 56, device="cuda")
    for dt in (torch.float16, torch.bfloat16):
        xd = x.to(dt)
        y, gx, _ = run(first, xd, g1.to(dt))
        yr, gxr, _ = run(first, xd.float(), g1.to(dt).float())
        assert y.dtype == dt and gx.dtype == dt and y.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(y, yr.to(dt)) and torch.equal(gx, gxr.to(dt))
    s64 = encoder(8, seed=2)[:3].double()
    y64, gx64, gp64 = run(s64, x.double(), gy.double())
    assert y64.dtype == torch.float64 and gx64.dtype == torch.float64 and all(g.dtype == torch.float64 for g in gp64)
    assert torch.equal(y64, y32.double()) and torch.equal(gx64, gx32.double())
    assert all(torch.equal(a, b.double()) for a, b in zip(gp64, gp32))
    # the operators on strided rows (a view of an NCHW tensor) give the bits of contiguous rows
    blk = stages[2].blocks[0]
    xn = torch.randn(2, 8, 10, 14, device="cuda")
    assert torch.equal(ops.res_block(xn.permute(0, 2, 3, 1), blk),
                       ops.res_block(xn.permute(0, 2, 3, 1).contiguous(), blk))
    conv, norm, _ = stages[1].conv_in
    rows = torch.randn(2, 20, 28, 8, device="cuda", dtype=torch.float64)
    assert torch.equal(ops.conv_gn_relu_ws(rows, conv, norm, 1), ops.conv_gn_relu_ws(rows.float(), conv, norm, 1))
    with pytest.raises(ValueError, match="channels-last rows"):
        ops.conv_gn_relu_ws(rows.permute(0, 3, 1, 2), conv, norm, 1)


class _OracleEncoder(torch.nn.Module):
    """The float64 oracle (F.pad reflect, F.conv2d, F.group_norm) on the parameters of `enc`, fp32 out."""

    def __init__(self, enc, shape):
        super().__init__()
        self.enc, self.shape = enc, shape

    def forward(self, x, *args, **kwargs):
        sd = {k: v.double() for k, v in self.enc.state_dict(keep_vars=True).items()}
        return O.resnet_down(x.double(), sd, *self.shape).float()


def _branch_run(conv, checkpointing=""):
    """UnimodalBranch(conv, max atomic pool, group view pool, concatenation) on the two-setting toy mapping of
    tests/golden/unimodal_branch_toy.npz; returns the fused 3D features and the gradients of a weighted sum w.r.t.
    the 3D features, the input images of both settings and the encoder's parameters."""
    from conftest import load_golden
    from test_containers import _toy_image_data
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool, GroupBimodalCSRPool
    g = load_golden("unimodal_branch_toy")
    mod = _toy_image_data(g, "cuda")
    xs = []
    for im in mod:
        x = im.x.detach().clone().requires_grad_(True)
        im._x = x
        xs.append(x)
    view_pool = GroupBimodalCSRPool(in_map=8, in_mod=16, num_groups=4, use_num=True)
    view_pool.load_state_dict(g["sd"], strict=True)
    branch = UnimodalBranch(conv, BimodalCSRPool(mode="max"), view_pool, BimodalFusion("concatenation"),
                            checkpointing=checkpointing).cuda()
    branch.train()
    params = [p for p in conv.parameters()]
    for p in params:
        p.grad = None
    x_3d = g["x_3d"].cuda().requires_grad_(True)
    out = branch({"x_3d": x_3d, "x_seen": None, "modalities": {"image": mod}}, "image")
    (out["x_3d"] * g["w"].cuda()).sum().backward()     # reentrant checkpointing supports .backward() only
    return out["x_3d"].detach(), [x_3d.grad] + [x.grad for x in xs] + [p.grad.clone() for p in params]


def test_unimodal_branch_over_a_mapping():
    """UnimodalBranch(conv=ResNetDown(...)) forward + backward over the toy mapping against the same branch on the
    float64 oracle encoder with the same parameters (the pools and fusion are the same kernels; the encoder and the
    map layout differ: ours is channels-last, the oracle's NCHW).  The max pool can move a gradient to another
    pixel where two pixels tie within the encoder's rounding, so gradients are compared normwise.  With
    checkpointing='c' (the positional reset flag, reentrant recompute) the branch gives the same bits, under
    torch.use_deterministic_algorithms(True)."""
    torch.manual_seed(31)
    enc = ResNetDown(down_conv_nn=[16, 16], kernel_size=3, stride=1, padding=1, N=1, block="ResBlock",
                     normalization="GroupNorm", weight_standardization=True).cuda()
    out, grads = _branch_run(enc)
    ref, rgrads = _branch_run(_OracleEncoder(enc, (3, 1, 1)))
    tol = 2 * 3 * 9 * 16 * U32
    assert out.shape == (1000, 28)
    assert maxrel(out, ref) <= tol
    for a, b in zip(grads, rgrads):
        assert l2rel(a, b) <= 4 * tol
    # bit-for-bit needs the ordered pool backwards too (the atomic ones add in any order)
    torch.use_deterministic_algorithms(True)
    try:
        out_d, grads_d = _branch_run(enc)
        out_c, grads_c = _branch_run(enc, checkpointing="c")
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(out_c, out_d) and all(torch.equal(a, b) for a, b in zip(grads_c, grads_d))
