"""The image UNet (ResNetDown + ResNetUp + UnaryConv on libdva_conv2d.so and libdva_unet.so) on the GPU, against
the float64 reference.

Bounds: those of tests/test_gpu_image_encoder.py.  Outputs: max |got - ref| / max |ref| <= L * K_max * u32;
gradients, normwise, <= 4 * L * K_max * u32, with L the convolution count of the whole UNet (21 in the encoder, 4
up-stages of 1 + 2 and a stride-1 one of 1 + 2, the downsamples and last_conv being 1x1) and K_max = 9 * C_in of
the widest 3x3: the first transposed convolution of up-stage 0, 9 * (8 f + 4 f) at f = in_feat (432 at f = 4, 3456
at f = 32)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from deepviewagg_b200 import _lib
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_unet_oracle as O
from test_gpu_image_encoder import l2rel, maxrel
from test_image_unet_oracle import DOWN, UP, small_opt, unpack

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
N_CONV = 21 + 15


def bounds(f):
    kmax = 9 * 12 * f
    return N_CONV * kmax * U32, 4 * N_CONV * kmax * U32


def perturbed(net, seed):
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.GroupNorm):
                m.weight.copy_(1 + 0.2 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen))
    return net


def run(net, x, gy, *args):
    x = x.detach().clone().requires_grad_(True)
    y = net(x, *args)
    params = list(net.state_dict(keep_vars=True).values())
    g = torch.autograd.grad(y, [x] + params, gy)
    return y, g[0], g[1:]


def oracle_grads(net, x, gy, topo, last=None):
    sd = {k: v.detach().double().cpu().requires_grad_(True) for k, v in net.state_dict().items()}
    xo = x.detach().double().cpu().requires_grad_(True)
    y = O.unet(xo, sd, DOWN, UP[topo], last=last or {})
    g = torch.autograd.grad(y, [xo] + list(sd.values()), gy.double().cpu())
    return y.detach(), g[0], g[1:]


@pytest.mark.parametrize("name", ["unet5_b2", "unet4_b1"])
def test_fixture_parity(name):
    z = np.load(os.path.join(GOLDEN, f"image_unet_{name}.npz"), allow_pickle=False)
    net = I.UNet(small_opt(name.split("_")[0])).cuda()
    keys, params, grads, _ = unpack(z)
    net.load_state_dict(params, strict=True)
    x = torch.from_numpy(z["x"]).float().cuda()
    gy = torch.from_numpy(z["gy"]).float().cuda()
    y, gx, gp = run(net, x, gy)
    by, bg = bounds(4)
    assert y.shape == z["y"].shape and y.is_contiguous(memory_format=torch.channels_last)
    assert maxrel(y, torch.from_numpy(z["y"])) <= by
    assert l2rel(gx, torch.from_numpy(z["gx"])) <= bg
    for k, g in zip(keys, gp):
        assert l2rel(g, grads[k]) <= bg, k


def full_width(topo="unet5", seed=3):
    torch.manual_seed(seed)
    return perturbed(I.UNet(small_opt(topo, 32)), seed + 1).cuda()


def test_full_width_against_oracle():
    net = full_width()
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 4, 128, 256, generator=gen).cuda()
    gy = torch.randn(2, 13, 128, 256, generator=gen).cuda()
    y, gx, gp = run(net, x, gy)
    ry, rgx, rgp = oracle_grads(net, x, gy, "unet5")
    by, bg = bounds(32)
    assert maxrel(y, ry) <= by
    assert l2rel(gx, rgx) <= bg
    for g, r in zip(gp, rgp):
        assert l2rel(g, r) <= bg


def test_layouts_bits_determinism_autocast_and_dtypes():
    torch.manual_seed(2)
    net = perturbed(I.UNet(small_opt("unet4", 8)), 3).cuda()
    x = torch.randn(2, 4, 48, 64, device="cuda")
    gy = torch.randn(2, 13, 48, 64, device="cuda")
    y, gx, gp = run(net, x, gy)
    y2, gx2, gp2 = run(net, x.contiguous(memory_format=torch.channels_last), gy)
    assert torch.equal(y, y2) and torch.equal(gx, gx2) and all(torch.equal(a, b) for a, b in zip(gp, gp2))
    y3, gx3, gp3 = run(net, x, gy)
    assert torch.equal(y, y3) and torch.equal(gx, gx3) and all(torch.equal(a, b) for a, b in zip(gp, gp3))
    torch.use_deterministic_algorithms(True)
    try:
        y4, gx4, gp4 = run(net, x, gy)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(y, y4) and torch.equal(gx, gx4) and all(torch.equal(a, b) for a, b in zip(gp, gp4))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ya = net(x)
    assert ya.dtype == torch.float32 and torch.equal(ya, y)
    for dt in (torch.float16, torch.bfloat16):
        yd, gxd, _ = run(net, x.to(dt), gy.to(dt))
        yr, gxr, _ = run(net, x.to(dt).float(), gy.to(dt).float())
        assert yd.dtype == dt and gxd.dtype == dt
        assert torch.equal(yd, yr.to(dt)) and torch.equal(gxd, gxr.to(dt))
    n64 = perturbed(I.UNet(small_opt("unet4", 8)), 3).cuda()
    n64.load_state_dict(net.state_dict())
    n64 = n64.double()
    y64, gx64, gp64 = run(n64, x.double(), gy.double())
    assert y64.dtype == torch.float64 and all(g.dtype == torch.float64 for g in gp64)
    assert torch.equal(y64, y.double()) and torch.equal(gx64, gx.double())
    assert all(torch.equal(a, b.double()) for a, b in zip(gp64, gp))


def test_bad_sizes_raise_before_any_launch():
    net = I.UNet(small_opt("unet5")).cuda()
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="UNet up stage 2"):
        net(torch.zeros(1, 4, 50, 32, device="cuda"))
    assert _lib.launch_count() == n0


def test_dropout_masks():
    x = torch.randn(3, 32, 5, 7, device="cuda")
    d = I.Dropout2d(p=0.5, inplace=True).train()
    torch.manual_seed(4)
    ref = F.dropout2d(x, 0.5, True)
    torch.manual_seed(4)
    mask = d.draw_mask(x)
    assert mask.shape == (3, 32, 1, 1) and torch.equal(x * mask, ref)
    torch.manual_seed(4)
    assert torch.equal(d(x.clone()), ref)
    pd = I.PersistentDropout2d(32, p=0.5).train()
    y1 = pd(x, True)
    m1 = pd.mask.clone()
    assert torch.equal(pd(x, False), y1) and torch.equal(pd.mask, m1)
    torch.manual_seed(5)
    pd(x, True)
    torch.manual_seed(5)
    expect = x.new_empty(1, 32, 1, 1).bernoulli_(0.5).div_(0.5)
    assert torch.equal(pd.mask, expect)
    pd.eval()
    assert pd(x, True) is x and pd.mask is None


@pytest.mark.parametrize("persistent", [False, True])
def test_unet_with_drawn_masks_matches_oracle(persistent):
    opt = small_opt("unet4", 8)
    opt["last_conv"] = dict(input_nc=8, output_nc=13, in_drop=0.5, out_drop=0.25, persistent_drop=persistent,
                            weight_standardization=True, activation="ReLU")
    torch.manual_seed(6)
    net = perturbed(I.UNet(opt), 7).cuda().train()
    x = torch.randn(2, 4, 32, 48, device="cuda")
    gy = torch.randn(2, 13, 32, 48, device="cuda")
    torch.manual_seed(8)
    y, gx, gp = run(net, x, gy, True)
    # the masks the dropouts drew, redrawn from the same seed in the same order
    torch.manual_seed(8)
    h = torch.empty(2, 8, 1, 1, device="cuda")
    o = torch.empty(2, 13, 1, 1, device="cuda")
    if persistent:
        m_in = h.new_empty(1, 8, 1, 1).bernoulli_(0.5).div_(0.5)
        m_out = o.new_empty(1, 13, 1, 1).bernoulli_(0.75).div_(0.75)
        assert torch.equal(net.last.input_dropout.mask, m_in)
    else:
        m_in = h.new_empty(2, 8, 1, 1).bernoulli_(0.5).div_(0.5)
        m_out = o.new_empty(2, 13, 1, 1).bernoulli_(0.75).div_(0.75)
    last = dict(standardize=True, activation="ReLU", in_mask=m_in.double().cpu(), out_mask=m_out.double().cpu())
    ry, rgx, rgp = oracle_grads(net, x, gy, "unet4", last=last)
    by, bg = bounds(8)
    assert maxrel(y, ry) <= by
    assert l2rel(gx, rgx) <= bg
    for g, r in zip(gp, rgp):
        assert l2rel(g, r) <= bg
    if persistent:      # reset=False keeps the mask
        y2 = net(x, False)
        assert torch.equal(y2, y.detach())


def branch_opt():
    """A UNet for the 16-channel images of the toy mapping (sides multiples of 4): 16 channels out."""
    down = dict(module_name="ResNetDown", block="ResBlock", normalization="GroupNorm", weight_standardization=True,
                N=[0, 1, 1], stride=[1, 2, 2], kernel_size=[3, 2, 2], padding=[1, 0, 0],
                down_conv_nn=[[16, 16], [16, 32], [32, 32]])
    up = dict(module_name="ResNetUp", block="ResBlock", normalization="GroupNorm", weight_standardization=True, N=1,
              kernel_size=[2, 2, 3], stride=[2, 2, 1], padding=[0, 0, 1],
              up_conv_nn=[[32, 32, 32], [32, 16, 16], [16, 0, 16]])
    return dict(down_conv=down, up_conv=up, last_conv=dict(input_nc=16, output_nc=16))


class _OracleUNet(torch.nn.Module):
    """The float64 oracle on the parameters of `net`, fp32 out."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x, *args, **kwargs):
        sd = {k: v.double() for k, v in self.net.state_dict(keep_vars=True).items()}
        return O.unet(x.double(), sd, [(3, 1, 1), (2, 2, 0), (2, 2, 0)], [(2, 2, 0), (2, 2, 0), (3, 1, 1)],
                      last={}).float()


def test_unimodal_branch_over_a_mapping():
    """UnimodalBranch(conv=UNet(...)) forward + backward over the two-setting toy mapping against the same branch on
    the float64 oracle UNet; with checkpointing='c' the same bits under deterministic mode.  The output is held to
    the UNet's bound (L = 13 convolutions, K_max = 9 * 64).  The max pool sends each point's gradient to its argmax
    pixel, and where two pixels tie within the UNet's rounding the two runs pick different ones: a whole gradient
    entry moves, and the UNet's backward spreads it over the image and the parameters, so those gradients are held
    to 2e-2 normwise (measured ~1e-2; the 3D features' gradient, which does not pass the pool, to the bound).  The
    parameters' gradients are checked against float64 by the tests above; here only for identical bits."""
    from test_gpu_image_encoder import _branch_run
    torch.manual_seed(31)
    net = perturbed(I.UNet(branch_opt()), 32).cuda()
    out, grads = _branch_run(net)
    ref, rgrads = _branch_run(_OracleUNet(net))
    tol = 13 * 9 * 64 * U32
    assert out.shape == (1000, 28)
    assert maxrel(out, ref) <= tol
    assert l2rel(grads[0], rgrads[0]) <= 4 * tol
    for a, b in zip(grads[1:3], rgrads[1:3]):     # the images of the two settings
        assert l2rel(a, b) <= 2e-2
    torch.use_deterministic_algorithms(True)
    try:
        out_d, grads_d = _branch_run(net)
        out_c, grads_c = _branch_run(net, checkpointing="c")
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(out_c, out_d) and all(torch.equal(a, b) for a, b in zip(grads_c, grads_d))


def unet_scenario():
    """Forward + backward of a small UNet (2x2 upsampling stages, transposed 3x3 blocks) with a ReLUWS last_conv,
    with the input's gradient, against the oracle: every kernel of libdva_unet.so.  A gradient may exceed the
    bound where plain fp32 arithmetic (the oracle on cuDNN without TF32) is itself that far from float64 here; it
    then stays within 4x of that fp32 error."""
    opt = small_opt("unet4", 8)
    opt["last_conv"] = dict(input_nc=8, output_nc=13, weight_standardization=True, activation="ReLU")
    torch.manual_seed(11)
    net = perturbed(I.UNet(opt), 12).cuda()
    gen = torch.Generator().manual_seed(13)
    x = torch.randn(2, 4, 32, 48, generator=gen).cuda()
    gy = torch.randn(2, 13, 32, 48, generator=gen).cuda()
    y, gx, gp = run(net, x, gy)
    last = dict(standardize=True, activation="ReLU")
    ry, rgx, rgp = oracle_grads(net, x, gy, "unet4", last=last)
    # the same arithmetic in plain fp32 (cuDNN without TF32): how far rounding alone moves each gradient here
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in net.state_dict().items()}
    xf = x.clone().requires_grad_(True)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yf = O.unet(xf, sd, DOWN, UP["unet4"], last=last)
        gf = torch.autograd.grad(yf, [xf] + list(sd.values()), gy)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    by, bg = bounds(8)
    assert maxrel(y, ry) <= by
    for a, f, b in zip((gx,) + tuple(gp), gf, (rgx,) + tuple(rgp)):
        assert l2rel(a, b) <= max(bg, 4 * l2rel(f, b)), (l2rel(a, b), l2rel(f, b))
    return True


def test_unet_scenario():
    n0 = _lib.launch_count()
    assert unet_scenario()
    assert _lib.launch_count() > n0
