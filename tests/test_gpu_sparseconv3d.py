"""Class-weighted NLL, Lovász-softmax and the sparse-conv fusion models on the H100.

  * ops.csr_nll_loss(weight=w) against float64 F.nll_loss(weight=w) at the bounds of the NLL row of
    tests/test_rest_matrix_table.py, with count / the row's share replaced by W / w[y] (stated in
    tests/test_loss_matrix_table.py): zero weights, all rows
    ignored, fp32 / bf16 / fp16 logits; two calls give the same bits; weight=None gives the bits of weight = 1;
  * ops.lovasz_softmax against the float64 oracle (oracle/lovasz_oracle.py): loss and gradient on tie-free
    inputs (errors distinct multiples of 2^-22, exact in fp32), loss and per-block gradient sums on tied
    inputs, log_probs=True against exp-then-call, the edge cases, 2 M points x 19 classes; two calls give the
    same bits;
  * APIModel, LateFeatureFusion and LateLogitFusion against the reference's fixtures
    (oracle/make_golden_sparseconv3d.py): outputs and losses <= 1e-6 relative, head gradients <= 1e-5, strict
    state-dict loads, and LateFeatureFusion restores input.data.x.
"""
import os

import numpy as np
import pytest
import torch

from oracle import lovasz_oracle as LO
from oracle import sparseconv3d_fakes as fk
from oracle.make_golden_sparseconv3d import MODEL_CASES
from test_kernel_matrix_table import DTYPES, K_ERR, TINY, U32, U_S, violations

pytestmark = pytest.mark.gpu
KE = K_ERR * U32
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30)) if b.numel() else 0.0


# ------------------------------------------------------------------------------------------------
# class-weighted NLL
# ------------------------------------------------------------------------------------------------
def wnll_inputs(N, K, dt, seed, zero_classes=()):
    gen = torch.Generator().manual_seed(seed)
    x = 3 * torch.randn(N, K, generator=gen)
    x[::11] += 40
    lab = torch.randint(0, K, (N,), generator=gen)
    lab[torch.rand(N, generator=gen) < 0.2] = -1
    w = torch.rand(K, generator=gen) * 2 + 0.1
    for c in zero_classes:
        w[c] = 0.0
    return x.to(DTYPES[dt]), lab, w


def wnll_reference(x, lab, w, ignore_index=-1):
    """float64 log_softmax + nll_loss(weight=w) (mean) and its gradient; mag_v and w[y_v] per row, W."""
    xd = x.detach().double().cpu().requires_grad_(True)
    loss = torch.nn.functional.nll_loss(torch.log_softmax(xd, -1), lab, weight=w.double(), ignore_index=ignore_index)
    g, = torch.autograd.grad(loss, xd)
    xd = xd.detach()
    counted = lab != ignore_index
    wy = torch.where(counted, w.double()[lab.clamp(min=0)], torch.zeros(lab.shape, dtype=torch.float64))
    mag = xd.abs().max(-1).values + torch.logsumexp(xd, -1).abs()
    return dict(loss=float(loss.detach()), grad=g, mag=mag, p=torch.softmax(xd, -1), wy=wy, W=float(wy.sum()))


def wnll_bounds(ref, K, dt):
    """The NLL row's bounds with the mean over counted rows weighted by w[y] and count replaced by W / w[y]."""
    W = ref["W"]
    wmag = float((ref["wy"].abs() * ref["mag"]).sum()) / W if W > 0 else 0.0
    b_loss = KE * (K + 2) * wmag + U32 * abs(ref["loss"])
    gs = (ref["wy"].abs() / W if W > 0 else torch.zeros_like(ref["wy"])).view(-1, 1)
    b_grad = U_S[dt] * ref["grad"].abs() + KE * ((K + 2) * ref["mag"].view(-1, 1) * ref["p"] + 1) * gs + TINY[dt]
    return b_loss, b_grad


def check_wnll(x, lab, w, dt):
    from deepviewagg_b200 import ops
    K = x.shape[1]
    xg = x.cuda().requires_grad_(True)
    loss = ops.csr_nll_loss(xg, lab.cuda(), weight=w.cuda())
    g, = torch.autograd.grad(loss, xg)
    ref = wnll_reference(x, lab, w)
    b_loss, b_grad = wnll_bounds(ref, K, dt)
    loss_v = float(loss.detach())
    assert abs(loss_v - ref["loss"]) <= b_loss, (loss_v, ref["loss"], b_loss)
    n, msg = violations(g, ref["grad"], b_grad)
    assert n == 0, f"weighted nll gradient: {msg}"
    # two calls, same bits
    loss2 = ops.csr_nll_loss(xg, lab.cuda(), weight=w.cuda())
    g2, = torch.autograd.grad(loss2, xg)
    assert torch.equal(loss, loss2) and torch.equal(g, g2)


def wnll_scenario(dt):
    for K in (2, 13, 64):
        check_wnll(*wnll_inputs(3000, K, dt, seed=K, zero_classes=(1,)), dt)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_weighted_nll_against_float64(dt):
    wnll_scenario(dt)


def test_weighted_nll_edges():
    from deepviewagg_b200 import ops
    x, lab, w = wnll_inputs(500, 13, "f32", seed=5)
    xg = x.cuda().requires_grad_(True)
    # every row ignored: NaN, zero gradient
    none = torch.full_like(lab, -1).cuda()
    loss = ops.csr_nll_loss(xg, none, weight=w.cuda())
    assert torch.isnan(loss) and (torch.autograd.grad(loss, xg)[0] == 0).all()
    # the counted rows' weights sum to 0: NaN, as torch
    zero = w.clone()
    zero[lab[lab >= 0].unique()] = 0.0
    loss = ops.csr_nll_loss(xg, lab.cuda(), weight=zero.cuda())
    ref = torch.nn.functional.nll_loss(torch.log_softmax(x.double(), -1), lab, weight=zero.double(),
                                     ignore_index=-1)
    assert torch.isnan(loss) and torch.isnan(ref)
    # weight = 1 gives the bits of weight=None (which runs the unweighted kernels)
    for dt in DTYPES:
        xs = x.to(DTYPES[dt]).cuda().requires_grad_(True)
        a = ops.csr_nll_loss(xs, lab.cuda())
        ga, = torch.autograd.grad(a, xs)
        b = ops.csr_nll_loss(xs, lab.cuda(), weight=torch.ones(13, device="cuda"))
        gb, = torch.autograd.grad(b, xs)
        assert torch.equal(a, b) and torch.equal(ga, gb), dt
    with pytest.raises(ValueError, match="weight"):
        ops.csr_nll_loss(xg, lab.cuda(), weight=torch.ones(12, device="cuda"))


# ------------------------------------------------------------------------------------------------
# Lovász-softmax
# ------------------------------------------------------------------------------------------------
def lovasz_tiefree(P, K, seed, p_ignore=0.15):
    """Labels and probabilities whose errors |fg - p| are, per class, distinct multiples of 2^-22 (exact in
    fp32, so the kernel and the float64 oracle sort the same values)."""
    gen = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, K, (P,), generator=gen)
    lab[torch.rand(P, generator=gen) < p_ignore] = -1
    e = torch.stack([torch.randperm(2 ** 22 - 1, generator=gen)[:P] + 1 for _ in range(K)], 1).double() * 2.0 ** -22
    fg = (lab.view(-1, 1) == torch.arange(K)).double()
    p = torch.where(fg > 0, 1 - e, e)
    return p.float(), lab


def lovasz_tied(P, K, seed, p_ignore=0.15):
    gen = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, K, (P,), generator=gen)
    lab[torch.rand(P, generator=gen) < p_ignore] = -1
    p = torch.randint(0, 9, (P, K), generator=gen).float() / 8          # exact in fp32, bf16 and fp16
    return p, lab


def run_lovasz(p, lab, classes="present", log_probs=False, dtype=torch.float32):
    from deepviewagg_b200 import ops
    x = (p.log() if log_probs else p).to(dtype).cuda().requires_grad_(True)
    loss = ops.lovasz_softmax(x, lab.cuda(), classes=classes, log_probs=log_probs)
    g, = torch.autograd.grad(loss, x)
    return loss, g


def check_lovasz_tiefree(p, lab, classes="present"):
    loss, g = run_lovasz(p, lab, classes)
    ref, rgrad, _ = LO.lovasz_softmax(p.numpy(), lab.numpy(), classes)
    assert abs(float(loss) - ref) <= 2 * U32 * abs(ref) + 1e-12, (float(loss), ref)
    rg = torch.from_numpy(rgrad)
    # the oracle's 1 - I / U loses ~1e-16 absolute on a Jaccard difference; the kernel's (j + 1) / U does not
    n, msg = violations(g, rg, 4 * U32 * rg.abs() + 1e-15)
    assert n == 0, f"lovasz gradient: {msg}"
    loss2, g2 = run_lovasz(p, lab, classes)
    assert torch.equal(loss, loss2) and torch.equal(g, g2)


def check_lovasz_tied(p, lab, dtype, classes="present"):
    """Loss, and per tied block the sum of grad * d|fg - p|/dp (independent of the order of the ties)."""
    loss, g = run_lovasz(p, lab, classes, dtype=dtype)
    ref, rgrad, _ = LO.lovasz_softmax(p.numpy(), lab.numpy(), classes)
    assert abs(float(loss) - ref) <= 2 * U32 * abs(ref) + 1e-12, (float(loss), ref)
    gd = g.double().cpu().numpy()
    pn, ln = p.numpy().astype(np.float64), lab.numpy()
    dt = next(k for k, v in DTYPES.items() if v == dtype)
    for c in range(p.shape[1]):
        for blk in LO.sorted_blocks(pn, ln, c):
            s = -np.sign((ln[blk] == c) - pn[blk, c])
            got, want = float((gd[blk, c] * s).sum()), float((rgrad[blk, c] * s).sum())
            # each element rounded to the storage type (subnormal in fp16 below 2^-14)
            bound = U_S[dt] * float(np.abs(rgrad[blk, c]).sum()) + len(blk) * TINY[dt] + 4 * U32 * abs(want) + 1e-12
            assert abs(got - want) <= bound, (c, len(blk), got, want)


def lovasz_scenario(dt):
    from deepviewagg_b200 import ops
    dtype = DTYPES[dt]
    for K in (2, 13, 64):
        check_lovasz_tied(*lovasz_tied(4000, K, seed=K), dtype)
        check_lovasz_tied(*lovasz_tied(4000, K, seed=K + 1), dtype, classes="all")
        # log-probabilities against exp-then-call: the kernel takes exp in fp32 and chains the gradient through it
        p, lab = lovasz_tied(3000, K, seed=K + 2)
        logp = p.clamp(min=1 / 16).log().to(dtype)
        x = logp.cuda().requires_grad_(True)
        la = ops.lovasz_softmax(x, lab.cuda(), log_probs=True)
        ga, = torch.autograd.grad(la, x)
        pe = logp.cuda().float().exp().requires_grad_(True)
        lb = ops.lovasz_softmax(pe, lab.cuda())
        gb, = torch.autograd.grad(lb, pe)
        assert abs(float(la) - float(lb)) <= 4 * U32 * abs(float(lb)), (dt, K, float(la), float(lb))
        want = (gb * pe.detach()).cpu()
        n, msg = violations(ga, want, U_S[dt] * want.abs() + 8 * U32 * want.abs() + TINY[dt])
        assert n == 0, f"log_probs gradient: {msg}"
    if dt == "f32":
        for K, classes in ((2, "present"), (13, "present"), (13, "all"), (13, [0, 3, 3, 12]), (64, "present")):
            check_lovasz_tiefree(*lovasz_tiefree(5000, K, seed=K), classes)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_lovasz_against_float64(dt):
    lovasz_scenario(dt)


def test_lovasz_edges():
    from deepviewagg_b200 import ops
    p, lab = lovasz_tiefree(50, 5, seed=3)
    # no valid point: loss 0, gradient 0
    loss, g = run_lovasz(p, torch.full_like(lab, -1))
    assert float(loss) == 0.0 and not g.any()
    # a single valid point (the reference's squeeze() breaks here)
    one = torch.full_like(lab, -1)
    one[7] = 2
    check_lovasz_tiefree(p, one)
    check_lovasz_tiefree(p[7:8], torch.tensor([2]))
    # no kept class: 0, as the reference's mean([])
    loss, g = run_lovasz(p, lab, classes=[])
    assert float(loss) == 0.0 and not g.any()
    # a class absent from the labels: skipped by 'present', kept by 'all' and by a list
    absent = lab.clone()
    absent[absent == 4] = 0
    for classes in ("present", "all", [4, 1]):
        check_lovasz_tiefree(p, absent, classes)
    with pytest.raises(NotImplementedError):
        ops.lovasz_softmax(p.cuda(), lab.cuda(), per_image=True)
    with pytest.raises(NotImplementedError):
        ops.lovasz_softmax(p[:, :1].cuda(), lab.clamp(max=0).cuda())
    with pytest.raises(ValueError):
        ops.lovasz_softmax(p.cuda(), lab.cuda(), classes=[5])


def test_lovasz_2m_points_19_classes():
    p, lab = lovasz_tiefree(2_000_000, 19, seed=19, p_ignore=0.1)
    check_lovasz_tiefree(p, lab)


# ------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------
def _fixtures():
    return np.load(os.path.join(GOLDEN, "sparseconv3d_models.npz"))


def build_model(z, case, cls_name, opts):
    from deepviewagg_b200.models.multimodal import sparseconv3d as S
    K, c3 = int(z["num_classes"]), int(z["c_3d"])
    x, y = torch.from_numpy(z["x"]), torch.from_numpy(z["y"])
    opts = dict(opts)
    weight = torch.from_numpy(z["weight_classes"]) if opts.pop("weighted", False) else None
    sd = {k[len(case) + 4:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{case}/sd/")}
    if cls_name == "APIModel":
        model = S.APIModel(fk.DenseBackbone3D(x.shape[1], c3), K, weight_classes=weight, **opts)
        data = fk.Data(x=x.cuda(), y=y.cuda(), batch=torch.zeros(x.shape[0], dtype=torch.long, device="cuda"))
    else:
        data = fk.MMData(fk.Data(x=x.cuda(), y=y.cuda(), batch=torch.zeros(x.shape[0], dtype=torch.long,
                                                                            device="cuda")))
        if cls_name == "LateLogitFusion":
            model = S.LateLogitFusion(fk.DenseBackbone3D(x.shape[1], c3), fk.DenseNo3D(x.shape[1], K), K)
        else:
            n3 = c3 + 4 if opts["mode"] == "concatenation" else c3
            model = S.LateFeatureFusion(fk.DenseBackbone3D(x.shape[1], c3), fk.DenseNo3D(c3, n3),
                                        fk.DenseLateConv(c3 + n3), K, **opts)
    model.load_state_dict(sd, strict=True)
    return model.cuda(), data


@pytest.mark.parametrize("case", [c[0] for c in MODEL_CASES])
def test_models_match_reference(case):
    z = _fixtures()
    _, cls_name, opts = next(c for c in MODEL_CASES if c[0] == case)
    model, data = build_model(z, case, cls_name, opts)
    x_in = data.x if cls_name == "APIModel" else data.data.x
    model.set_input(data)
    model.forward()
    assert _rel(model.output, z[f"{case}/output"]) <= 1e-6, case
    assert model.loss_names == [str(n) for n in z[f"{case}/loss_names"]]
    for name in model.loss_names:
        assert _rel(getattr(model, name).reshape(()), z[f"{case}/{name}"]) <= 1e-6, (case, name)
    if cls_name != "APIModel":
        assert data.data.x is x_in                              # the input's 3D features are restored
    model.backward()
    grads = {k[len(case) + 6:]: v for k, v in z.items() if k.startswith(f"{case}/grad/")}
    assert grads and set(grads) == {k for k, p in model.named_parameters() if k.startswith("head")}
    for k, p in model.named_parameters():
        if k in grads:
            assert _rel(p.grad, grads[k]) <= 1e-5, (case, k, _rel(p.grad, grads[k]))
