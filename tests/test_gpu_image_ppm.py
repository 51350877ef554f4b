"""ADE20KResNet18PPM (the ResNet-18 trunk and the PPM head, ops.rn_ppm_head) on the GPU, against the float64
restatement oracle/image_ppm_oracle.py on the same parameters and on the kernels' own ReLU masks and max-pool
indices (kernel_branches), with the bounds of tests/test_gpu_image_resnet18.py: L = 28 convolutions, K_max = 9 * 2560
= 23040 (conv_last)."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from deepviewagg_b200 import _lib, ops
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_ppm_oracle as O
from oracle import image_resnet18_oracle as R
from test_gpu_image_encoder import l2rel, maxrel
from test_gpu_image_resnet18 import _bn_training, _running, bounds
from test_gpu_kernel_matrix import record

pytestmark = pytest.mark.gpu

CASES = {  # oracle/make_golden_image_ppm.py:CASES
    "train_b2": (True, (2, 3, 61, 45), None, 21),
    "train_b1": (True, (1, 3, 50, 66), None, 22),
    "eval_outsize": (False, (2, 3, 40, 56), (40, 56), 23),
}


def make(seed=0, **kw):
    m = I.ADE20KResNet18PPM(**kw)
    m.load_state_dict(R.hashed_state(m.state_dict(), seed), strict=True)
    return m.cuda()


def conv5_of(m, x):
    for h in I._run_trunk(m.encoder._trunk(), I._rows(x)):
        pass
    return h


def kernel_branches(m, x):
    """The ReLU masks and max-pool indices of the kernels' forward of m on x in the oracle's order: the trunk's, each
    pyramid branch's (its pooled map from the same gather-pool kernel and index, then the same conv + BN + ReLU
    kernels) and conv_last's.  The module's state is left as it was."""
    st = {k: v.clone() for k, v in m.state_dict().items()}
    out = []
    with torch.no_grad():
        h = I._rows(x)
        for layer in m.encoder._trunk():
            if isinstance(layer, list):
                for conv, bn in layer:
                    h = ops.rn_conv_bn_relu(h, conv, bn)
                    out.append(h > 0)
                out.append(F.max_pool2d(h.permute(0, 3, 1, 2), 3, 2, 1, return_indices=True)[1].permute(0, 2, 3, 1))
                h = ops.rn_maxpool(h)
            else:
                for blk in layer:
                    out.append(ops.rn_conv_bn_relu(h, blk.conv1, blk.bn1) > 0)
                    h = ops.rn_basic_block(h, blk)
                    out.append(h > 0)
        B, hh, ww, C = h.shape
        img, pix, aptr, offsets = ops._ppm_index(B, hh, ww, O.SCALES, h.device)
        pooled = ops.gather_pool(h, img, pix, aptr, "mean", channels_last=True)
        for k, (s, br) in enumerate(zip(O.SCALES, m.decoder.ppm)):
            mode = br[2].training
            br[2].training = ops.ppm_branch_training(br[2], B, s)
            try:
                out.append(ops.rn_conv_bn_relu(pooled[offsets[k]:offsets[k] + B * s * s].view(B, s, s, C), br[1],
                                               br[2]) > 0)
            finally:
                br[2].training = mode
        out.append(ops.rn_ppm_head(h, m.decoder) > 0)
    m.load_state_dict(st)
    return [t.permute(0, 3, 1, 2).contiguous().cpu() for t in out]


def oracle(m, x, gy, out_size=None, dtype=torch.float64, device="cpu", masks=None):
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    p = {k: v.detach().to(device, dtype if v.is_floating_point() else v.dtype).clone()
         for k, v in m.state_dict().items()}
    for k in names:
        p[k].requires_grad_(True)
    xo = x.detach().to(device, dtype).requires_grad_(True)
    y = O.forward(xo, p, _bn_training(m), out_size, masks)
    g = torch.autograd.grad(y, [xo] + [p[k] for k in names], gy.to(device, dtype))
    return y.detach(), g[0], dict(zip(names, g[1:])), {k: v for k, v in p.items() if "running" in k}


def cudnn_fp32(m, x, gy, out_size, masks):
    tf = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return oracle(m, x, gy, out_size, torch.float32, "cuda", masks)
    finally:
        torch.backends.cudnn.allow_tf32 = tf


def run(m, x, gy, out_size=None):
    x = x.detach().clone().requires_grad_(True)
    y = m(x, out_size=out_size)
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    params = dict(m.named_parameters())
    g = torch.autograd.grad(y, [x] + [params[k] for k in names], gy)
    return y, g[0], dict(zip(names, g[1:]))


def _stat_bound(k, before, rrun, bo, momentum=0.001):
    """momentum * (the output bound on z) for running_mean, momentum * 2 * rms(z) * (that bound) for running_var, with
    rms(z) from the batch statistics the float64 update implies."""
    pre, stat = k.rsplit(".", 1)
    if stat not in ("running_mean", "running_var"):
        return 0.0
    mean, var = [(rrun[f"{pre}.{s}"] - (1 - momentum) * before[f"{pre}.{s}"].double().cpu()) / momentum
                 for s in ("running_mean", "running_var")]
    rms = float((var.clamp(min=0) + mean ** 2).sqrt().max())
    return momentum * bo * rms * (1 if stat == "running_mean" else 2 * rms)


def check(m, x, gy, out_size=None):
    """One forward + backward of m against the float64 oracle; returns (y, gx, param grads, running before)."""
    before = _running(m)
    y, gx, gp = run(m, x, gy, out_size)
    after = _running(m)
    with torch.no_grad():
        for k, v in before.items():
            m.state_dict()[k].copy_(v)
    masks = kernel_branches(m, x)
    ry, rgx, rgp, rrun = oracle(m, x, gy, out_size, masks=masks)
    cy, cgx, cgp, crun = cudnn_fp32(m, x, gy, out_size, masks)
    with torch.no_grad():
        for k, v in after.items():
            m.state_dict()[k].copy_(v)
    assert y.shape == ry.shape and y.is_contiguous(memory_format=torch.channels_last)
    bo, bg = bounds(m)
    assert bo == 28 * 23040 * 2.0 ** -24
    assert maxrel(y.detach(), ry) <= max(bo, 4 * maxrel(cy, ry)), (maxrel(y.detach(), ry), maxrel(cy, ry))
    assert l2rel(gx, rgx) <= max(bg, 4 * l2rel(cgx, rgx)), (l2rel(gx, rgx), l2rel(cgx, rgx))
    assert set(gp) == set(rgp)
    for k in gp:
        assert l2rel(gp[k], rgp[k]) <= max(bg, 4 * l2rel(cgp[k], rgp[k])), (k, l2rel(gp[k], rgp[k]),
                                                                            l2rel(cgp[k], rgp[k]))
    for k, v in rrun.items():
        # a few fp32 ulps, 4 x the cuDNN fp32 error, or the momentum times the output bound on the batch statistics
        # (conv_last's K = 23040 products in 3xTF32 leave its batch mean well above a few ulps of the running mean)
        got = after[k].double().cpu()
        ulp = 2.0 ** -23 * float(v.abs().max())
        e32 = float((crun[k].double().cpu() - v).abs().max())
        assert float((got - v).abs().max()) <= max(4 * ulp, 4 * e32, _stat_bound(k, before, rrun, bo)), \
            (k, float((got - v).abs().max()), ulp, e32)
    assert all(int(v) == 0 for k, v in after.items() if "num_batches_tracked" in k)
    return y, gx, gp, before


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixture_cases(name):
    training, shape, out_size, seed = CASES[name]
    m = I.ADE20KResNet18PPM().train(training)
    m.load_state_dict(R.hashed_state(m.state_dict(), seed), strict=True)
    m = m.cuda()
    x = torch.from_numpy(R.hash_grid(seed, 50000, shape, 8, 2)).float().cuda()
    g = np.load(f"{GOLDEN}/image_ppm_{name}.npz")
    yshape = (shape[0], 512, *(out_size or [ops.rn_out(ops.rn_out(ops.rn_out(n, 2), 2), 2) for n in shape[2:]]))
    gy = torch.from_numpy(R.hash_grid(seed, 60000, yshape, 8, 3)).float().cuda()
    y, _, gp, before = check(m, x, gy, out_size)
    assert y.shape == yshape and len(gp) == 84
    # the fixture's float64 output norm, within the same bound
    assert abs(float(y.detach().double().norm()) / float(g["y_norm"]) - 1) <= max(bounds(m)[0], 1e-5)
    after = _running(m)
    for k in before:
        if k.endswith(("running_mean", "running_var")) and "_tmp" not in k:
            moved = not torch.equal(before[k], after[k])
            if name == "train_b1":
                # the Prudent switch: the scale-1 branch at batch size 1 normalises with its running stats
                assert moved == (not k.startswith("decoder.ppm.0.2.")), k
            else:
                assert moved == training, k


def test_frozen_runs_no_wgrad():
    """frozen=True: eval-mode BatchNorms (train() keeps them so), no weight-gradient kernel, no parameter gradient,
    running stats unchanged, and the input gradient against the oracle."""
    m = make(seed=3, frozen=True)
    m.train()
    assert not m.training and not any(mod.training for mod in m.modules())
    x = torch.randn(2, 3, 48, 40, device="cuda")
    gy = torch.randn(2, 512, 6, 5, device="cuda")
    before = _running(m)
    xg = x.clone().requires_grad_(True)
    (y, gx), names = record(lambda: (lambda y: (y.detach(), torch.autograd.grad(y, [xg], gy)[0]))(m(xg)),
                            canon=lambda n: n, seen=set())
    assert not any("rn_conv_wgrad_kernel" in n for n in names)
    assert any("rn_conv_gemm_kernel" in n for n in names)
    assert all(p.grad is None for p in m.parameters())
    assert all(torch.equal(v, _running(m)[k]) for k, v in before.items())
    masks = kernel_branches(m, x)
    ry, rgx, _, _ = oracle(m, x, gy, masks=masks)
    cy, cgx, _, _ = cudnn_fp32(m, x, gy, None, masks)
    bo, bg = bounds(m)
    assert maxrel(y, ry) <= max(bo, 4 * maxrel(cy, ry)) and l2rel(gx, rgx) <= max(bg, 4 * l2rel(cgx, rgx))


def test_out_size_dtypes_and_autocast():
    m = make(seed=4).eval()
    x = torch.randn(2, 3, 37, 50, device="cuda")
    y32 = m(x)
    assert y32.shape == (2, 512, 5, 7) and y32.dtype == torch.float32
    yo = m(x, out_size=(37, 50))
    assert yo.shape == (2, 512, 37, 50) and yo.is_contiguous(memory_format=torch.channels_last)
    ref = F.interpolate(y32.double(), size=(37, 50), mode="bilinear", align_corners=False)
    assert maxrel(yo, ref) <= 16 * 2.0 ** -24
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        xd = x.to(dt).requires_grad_(True)
        y = m(xd, out_size=[20, 30])
        assert y.dtype == dt and y.shape == (2, 512, 20, 30) and y.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(y, m(xd.detach().float(), out_size=[20, 30]).to(dt))
        (gx,) = torch.autograd.grad(y.float().sum(), [xd])
        assert gx.dtype == dt
    with torch.autocast("cuda", dtype=torch.float16):
        ya = m(x.half())
    assert ya.dtype == torch.float32 and torch.equal(ya, m(x.half().float()))
    assert torch.equal(m(x.double()), y32.double())


def test_reproducible_and_deterministic():
    m = make(seed=5).train()
    x = torch.randn(2, 3, 61, 45, device="cuda")
    gy = torch.randn(2, 512, 8, 6, device="cuda")
    st = {k: v.clone() for k, v in m.state_dict().items()}
    a = run(m, x, gy)
    ra = _running(m)
    m.load_state_dict(st)
    b = run(m, x, gy)
    torch.use_deterministic_algorithms(True)
    try:
        m.load_state_dict(st)
        c = run(m, x, gy)
    finally:
        torch.use_deterministic_algorithms(False)
    m.load_state_dict(st)
    d = run(m, x.contiguous(memory_format=torch.channels_last), gy)
    for r in (b, c, d):
        assert torch.equal(a[0], r[0]) and torch.equal(a[1], r[1])
        assert all(torch.equal(a[2][k], r[2][k]) for k in a[2])
    assert all(torch.equal(v, _running(m)[k]) for k, v in ra.items())


def test_value_errors_before_any_launch():
    m = make().train()
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=r"\[B, 3, H, W\]"):
        m(torch.randn(2, 4, 32, 32, device="cuda"))
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(torch.randn(1, 3, 8, 8, device="cuda"))          # layer2 onwards at 1 x 1
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(torch.randn(1, 3, 2, 2, device="cuda"))          # the stem
    for bad in ((0, 4), (4,), (4.0, 4), (True, 4), 8, (4, 4, 4)):
        with pytest.raises(ValueError, match="out_size"):
            m(torch.randn(2, 3, 32, 32, device="cuda"), out_size=bad)
    assert _lib.launch_count() == n0
    # the scale-1 branch at batch size 1 is the Prudent case, not an error
    assert m(torch.randn(1, 3, 16, 24, device="cuda")).shape == (1, 512, 2, 3)
    m.eval()
    assert m(torch.randn(1, 3, 8, 8, device="cuda")).shape == (1, 512, 1, 1)


_FOREIGN = re.compile(r"cudnn|cublas|cutlass|xmma|gemm|conv|norm|pool|upsample|interp|adaptive", re.I)


def test_a_train_step_launches_only_the_projects_kernels():
    """Every convolution, BatchNorm, pool and resize of a PPM train step (with out_size and the input's gradient) is
    one of this project's kernels: no cuDNN, cuBLAS, or torch pooling, normalisation or interpolation kernel."""
    m = make(seed=6).train()
    x = torch.randn(2, 3, 45, 61, device="cuda", requires_grad=True)
    gy = torch.randn(2, 512, 45, 61, device="cuda")
    st = {k: v.clone() for k, v in m.state_dict().items()}

    def step():
        m.load_state_dict(st)
        return torch.autograd.grad(m(x, out_size=(45, 61)), [x] + list(m.parameters()), gy)

    _, names = record(step, canon=lambda n: n, seen=set())
    ours = {n for n in names if "dva::" in n or "dva_resnet::" in n}
    foreign = sorted(n for n in names - ours if _FOREIGN.search(n))
    assert not foreign, foreign
    for k in ("rn_conv_gemm_kernel", "rn_conv_wgrad_kernel", "rn_bn_stats_kernel", "rn_bn_apply_kernel",
              "rn_bn_bwd_dz_kernel", "rn_resize_kernel", "rn_resize_bwd_kernel", "rn_maxpool_kernel",
              "gather_pool_fwd_cl_kernel", "gather_pool_bwd_det_cl_kernel"):
        assert any(k in n for n in ours), (k, sorted(ours))
    # the pool's backward is the deterministic one even outside deterministic mode
    assert not any("gather_pool_bwd_cl_kernel" in n for n in ours)


class _OraclePPM(torch.nn.Module):
    """The float64 restatement on the parameters of `enc`, on the kernels' branches, fp32 out."""

    def __init__(self, enc):
        super().__init__()
        self.enc = enc

    def forward(self, x, *args, **kwargs):
        masks = kernel_branches(self.enc, x)
        p = {k: v.double().cpu() for k, v in self.enc.state_dict(keep_vars=True).items()}
        return O.forward(x.double().cpu(), p, _bn_training(self.enc), masks=masks).float().cuda()


def test_unimodal_branch_over_a_mapping():
    """UnimodalBranch(conv=ADE20KResNet18PPM) forward + backward over the toy mapping (the 1/8-resolution
    channels-last output into the gather kernels through the scaled mappings) against the same branch on the float64
    restatement."""
    from test_gpu_image_resnet18 import _branch_run
    enc = make(seed=7).train()
    st = {k: v.clone() for k, v in enc.state_dict().items()}
    out, grads = _branch_run(enc, enc)
    enc.load_state_dict(st)
    ref, rgrads = _branch_run(_OraclePPM(enc), enc)
    bo, bg = bounds(enc)
    assert out.shape == (1000, 12 + 512)
    assert maxrel(out, ref) <= bo, maxrel(out, ref)
    for a, b in zip(grads, rgrads):
        assert l2rel(a, b) <= bg, l2rel(a, b)
    # in deterministic mode (the branch's own pools then reduce without atomics) two runs give the same bits
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            enc.load_state_dict(st)
            runs.append(_branch_run(enc, enc))
    finally:
        torch.use_deterministic_algorithms(False)
    (out_d, grads_d), (out_e, grads_e) = runs
    assert torch.equal(out, out_d) and torch.equal(out_d, out_e)
    assert all(torch.equal(a, b) for a, b in zip(grads_d, grads_e))
