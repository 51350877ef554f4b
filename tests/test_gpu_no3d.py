"""No3D models, the CSR log-softmax NLL and the query / search k-NN on the H100.

  * the four No3D classes against the reference's fixtures (oracle/make_golden_no3d.py), train and
    eval: outputs and loss <= 1e-6 relative, masked labels and propagated rows exact, pixel-head
    maps <= 1e-5; the reference-shaped state dicts load with strict=True;
  * ops.csr_nll_loss forward and gradient against torch's log_softmax + nll_loss chain in float64;
  * mapping.knn_query against the brute-force oracle (ties, k = 1 / 20 / 128, far queries) and
    against knn_grid when the query set is the search set.
"""
import numpy as np
import pytest
import torch

from oracle import no3d_oracle as O
from test_no3d_oracle import CLASSES, SAMPLES, classes_of, fixture_inputs, load_no3d

pytestmark = pytest.mark.gpu


class _Data:
    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)


def _rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30)) if b.numel() else 0.0


def _build(g, cls_name):
    from deepviewagg_b200.core.multimodal.image import ImageData, ImageMapping, SameSettingImageData
    from deepviewagg_b200.models.multimodal import no3d as N
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import MultimodalBlockDown, UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool
    settings, maps, sd, x3d = fixture_inputs(g, cls_name)
    n = g["pos"].shape[0]
    ims = []
    for st, x in zip(settings, maps):
        W, H, n_img = [int(v) for v in st["size"]]
        im = SameSettingImageData(pos=torch.zeros(n_img, 3), opk=torch.zeros(n_img, 3), ref_size=(W, H),
                                  proj_upscale=1, downscale=1)
        im.mappings = ImageMapping.from_dense(torch.from_numpy(st["pid"]), torch.from_numpy(st["iid"]),
                                              torch.from_numpy(st["pix"]), torch.from_numpy(st["feat"]),
                                              num_points=n)
        im.x = torch.from_numpy(x).clone()
        ims.append(im)
    mod = ImageData(ims).to("cuda")
    c = maps[0].shape[1] if maps else x3d.shape[1]
    branch = UnimodalBranch(None, BimodalCSRPool(mode="max"), BimodalCSRPool(mode="mean"), BimodalFusion("residual"),
                            keep_last_view=True, out_channels=c)
    mlp = "backbone.mlp.0.0.weight" in sd
    enc = N.No3DEncoder([MultimodalBlockDown(None, None, image=branch)], output_nc=5 if mlp else None,
                        default_output_nc=c)
    model = getattr(N, cls_name)(enc, num_classes=5)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    model = model.cuda()
    data = _Data(x=torch.from_numpy(x3d).cuda() if x3d is not None else None, pos=torch.from_numpy(g["pos"]).cuda(),
                 y=torch.from_numpy(g["labels"]).cuda(), batch=None, modalities={"image": mod})
    return model, data


@pytest.mark.parametrize("kind", SAMPLES)
def test_no3d_models_match_reference(kind):
    g = load_no3d(kind)
    errs = {}
    for cls_name in classes_of(g):
        for mode in ("train", "eval"):
            model, data = _build(g, cls_name)
            model.train(mode == "train")
            with torch.no_grad():
                model.set_input(data)
                out = model.forward()
            what = f"{kind} {cls_name} {mode}"
            ref = g[f"{cls_name}/{mode}/output"]
            errs[what] = _rel(out, ref)
            assert errs[what] <= 1e-6, (what, errs[what])
            assert torch.equal(model.labels.cpu(), torch.from_numpy(g[f"{cls_name}/{mode}/labels"])), what
            ref_loss = float(g[f"{cls_name}/{mode}/loss"])
            loss = float(model.loss_seg)
            if np.isnan(ref_loss):
                assert np.isnan(loss), what
            else:
                assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss), (what, loss, ref_loss)
            seen = torch.from_numpy(g["seen"])
            if mode == "eval" and seen.any() and not seen.all():
                # every unseen row is, bit for bit, the row of its nearest seen point (ties: lowest seen index)
                seen_idx, unseen = torch.nonzero(seen).squeeze(1), torch.nonzero(~seen).squeeze(1)
                nn_idx, _ = O.knn_query_bruteforce(g["pos"][unseen.numpy()], g["pos"][seen_idx.numpy()], 1)
                o = out.cpu()
                assert torch.equal(o[unseen], o[seen_idx[torch.from_numpy(nn_idx[:, 0])]]), what
            for i, im in enumerate(data.modalities["image"]):
                if f"{cls_name}/pred{i}" in g:
                    assert _rel(im.pred, g[f"{cls_name}/pred{i}"]) <= 1e-5, what
                    assert im.feat is im.x
                else:
                    assert im.pred is im.x
    print(kind, {k: f"{v:.1e}" for k, v in errs.items()})


def test_no3d_channels_last_pixel_head():
    """A channels-last feature map is read in place by the pixel head: same values as NCHW."""
    g = load_no3d("main")
    model, data = _build(g, "No3DFeatureFusion")
    model.eval()
    with torch.no_grad():
        model.set_input(data)
        model.forward()
        ref = [im.pred.clone() for im in data.modalities["image"]]
        model2, data2 = _build(g, "No3DFeatureFusion")
        model2.eval()
        for im in data2.modalities["image"]:
            im._x = im.x.contiguous(memory_format=torch.channels_last)
        model2.set_input(data2)
        model2.forward()
    for a, im in zip(ref, data2.modalities["image"]):
        assert torch.equal(a, im.pred)


def test_no3d_training_step_backward():
    """One training step of the view-loss class: the gradient reaches the head through csr_nll_loss."""
    g = load_no3d("main")
    model, data = _build(g, "No3DImageFeatureFusion")
    model.train()
    model.set_input(data)
    model.forward()
    model.backward()
    assert model.head[0].weight.grad is not None and torch.isfinite(model.head[0].weight.grad).all()


# ------------------------------------------------------------------------------------------------
# csr_nll_loss
# ------------------------------------------------------------------------------------------------
def _torch_chain(logits, labels, csr):
    x = logits.detach().double().cpu().requires_grad_(True)
    lab = labels.cpu()
    target = lab if csr is None else torch.repeat_interleave(lab, (csr[1:] - csr[:-1]).cpu())
    loss = torch.nn.functional.nll_loss(torch.log_softmax(x, -1), target, ignore_index=-1)
    g, = torch.autograd.grad(loss, x) if x.shape[0] else (torch.zeros_like(x),)
    return loss.detach(), g


def _nll_case(n, k, dtype, with_csr, p_ignore=0.2, seed=0):
    gen = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, 5, (n,), generator=gen)
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]) if with_csr else None
    v = int(csr[-1]) if with_csr else n
    logits = (3 * torch.randn(v, k, generator=gen)).to(dtype)
    labels = torch.randint(0, k, (n,), generator=gen)
    labels[torch.rand(n, generator=gen) < p_ignore] = -1
    return logits.cuda(), labels.cuda(), (csr.cuda() if with_csr else None)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_csr", [True, False])
@pytest.mark.parametrize("k", [13, 20, 64])
def test_csr_nll_loss_matches_torch_chain(dtype, with_csr, k):
    from deepviewagg_b200 import ops
    logits, labels, csr = _nll_case(3000, k, dtype, with_csr)
    x = logits.clone().requires_grad_(True)
    loss = ops.csr_nll_loss(x, labels, csr)
    g, = torch.autograd.grad(loss, x)
    ref_loss, ref_g = _torch_chain(logits, labels, csr)
    assert loss.dtype == torch.float32 and g.dtype == dtype
    assert abs(float(loss.detach()) - float(ref_loss)) <= 1e-6 * abs(float(ref_loss))
    # fp32 math; bf16 / fp16 gradients carry their storage rounding (fp16: down to its subnormal spacing 2^-24)
    tol = 1e-5 if dtype == torch.float32 else (8e-3 if dtype == torch.bfloat16 else 1e-3)
    floor = 2.0 ** -24 if dtype == torch.float16 else 0.0
    err = (g.double().cpu() - ref_g).abs()
    assert (err <= tol * ref_g.abs() + 1e-6 * ref_g.abs().max() + floor).all(), float(err.max())


def test_csr_nll_loss_ignored_rows_are_zero_and_all_ignored_is_nan():
    from deepviewagg_b200 import ops
    logits, labels, csr = _nll_case(500, 13, torch.float32, True)
    labels[::2] = -1
    x = logits.clone().requires_grad_(True)
    g, = torch.autograd.grad(ops.csr_nll_loss(x, labels, csr), x)
    ign = torch.repeat_interleave(labels, csr[1:] - csr[:-1]) == -1
    assert ign.any() and (g[ign] == 0).all() and (g[~ign] != 0).any()
    labels[:] = -1
    x = logits.clone().requires_grad_(True)
    loss = ops.csr_nll_loss(x, labels, csr)
    assert torch.isnan(loss)
    assert torch.isnan(_torch_chain(logits, labels, csr)[0])        # the mean over no element
    g, = torch.autograd.grad(loss, x)
    assert (g == 0).all()


def test_csr_nll_loss_empty_points():
    from deepviewagg_b200 import ops
    x = torch.empty(0, 13, device="cuda", requires_grad=True)
    lab = torch.empty(0, dtype=torch.long, device="cuda")
    loss = ops.csr_nll_loss(x, lab, torch.zeros(1, dtype=torch.long, device="cuda"))
    assert torch.isnan(loss)
    g, = torch.autograd.grad(loss, x)
    assert g.shape == (0, 13)
    assert torch.isnan(ops.csr_nll_loss(x, lab, None))
    # points without views: nothing counts
    lab = torch.tensor([1, 2], device="cuda")
    assert torch.isnan(ops.csr_nll_loss(x, lab, torch.zeros(3, dtype=torch.long, device="cuda")))


def test_csr_nll_loss_deterministic():
    from deepviewagg_b200 import ops
    logits, labels, csr = _nll_case(200000, 13, torch.float32, True, seed=5)
    res = []
    for _ in range(2):
        x = logits.clone().requires_grad_(True)
        loss = ops.csr_nll_loss(x, labels, csr)
        g, = torch.autograd.grad(loss, x)
        res.append((loss, g))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_csr_nll_loss_rejects_bad_input():
    from deepviewagg_b200 import ops
    logits, labels, csr = _nll_case(100, 13, torch.float32, True)
    bad = labels.clone()
    bad[int(torch.nonzero(csr[1:] > csr[:-1])[0])] = 13
    with pytest.raises(ValueError, match="label"):
        ops.csr_nll_loss(logits, bad, csr)
    bad[bad == 13] = -7
    with pytest.raises(ValueError, match="label"):
        ops.csr_nll_loss(logits, bad, csr)
    with pytest.raises(ValueError, match="classes"):
        ops.csr_nll_loss(torch.zeros(4, 65, device="cuda"), torch.zeros(4, dtype=torch.long, device="cuda"))
    short = csr.clone()
    short[-1] -= 1
    with pytest.raises(ValueError, match="csr_idx"):
        ops.csr_nll_loss(logits, labels, short)
    # the device is still healthy
    assert torch.isfinite(ops.csr_nll_loss(logits, labels, csr))


# ------------------------------------------------------------------------------------------------
# knn_query
# ------------------------------------------------------------------------------------------------
def _check_knn(query, search, k, **kw):
    from deepviewagg_b200.core.multimodal.mapping import knn_query
    nbr, d2 = knn_query(query.cuda(), search.cuda(), k, return_dist2=True, **kw)
    ref_n, ref_d = O.knn_query_bruteforce(query.numpy(), search.numpy(), k)
    assert np.array_equal(nbr.cpu().numpy(), ref_n)
    assert np.array_equal(d2.cpu().numpy(), ref_d)


@pytest.mark.parametrize("k", [1, 20, 128])
def test_knn_query_matches_bruteforce(k):
    gen = torch.Generator().manual_seed(k)
    search = torch.rand(6000, 3, generator=gen) * torch.tensor([6.0, 5.0, 3.0])
    query = torch.rand(2000, 3, generator=gen) * torch.tensor([8.0, 7.0, 4.0]) - 1.0     # some outside the grid
    _check_knn(query, search, k)


@pytest.mark.parametrize("k", [1, 20, 128])
def test_knn_query_ties(k):
    gen = torch.Generator().manual_seed(10 + k)
    a = torch.arange(8, dtype=torch.float32)
    lat = torch.stack(torch.meshgrid(a, a, a[:3], indexing="ij"), -1).reshape(-1, 3)
    search = torch.cat([lat, lat[::2], lat[::5]])[torch.randperm(lat.shape[0] + 96 + 39, generator=gen)]
    query = torch.cat([lat + 0.5, lat[:50] + torch.tensor([0.5, 0.0, 0.0]), lat[:20]])
    _check_knn(query, search, k)


@pytest.mark.parametrize("k", [1, 20, 128])
def test_knn_query_far_cluster(k):
    """Queries far from a dense search set walk the coarse level (no exhaustive scan is needed)."""
    gen = torch.Generator().manual_seed(20 + k)
    n = 60000
    # a room: floor and two walls, densely sampled; the queries are a cluster 30 m away
    u = torch.rand(n, 2, generator=gen) * 10
    which = torch.randint(0, 3, (n,), generator=gen)
    search = torch.zeros(n, 3)
    search[which == 0] = torch.stack([u[which == 0, 0], u[which == 0, 1], torch.zeros(int((which == 0).sum()))], 1)
    search[which == 1] = torch.stack([u[which == 1, 0], torch.zeros(int((which == 1).sum())), u[which == 1, 1] * 0.3], 1)
    search[which == 2] = torch.stack([torch.zeros(int((which == 2).sum())), u[which == 2, 0], u[which == 2, 1] * 0.3], 1)
    query = torch.randn(400, 3, generator=gen) + torch.tensor([40.0, 5.0, 1.0])
    query = torch.cat([query, torch.rand(400, 3, generator=gen) * 3 + torch.tensor([5.0, 5.0, 0.5])])
    _check_knn(query, search, k)


@pytest.mark.parametrize("k", [1, 16, 128])
def test_knn_query_self_equals_knn_grid(k):
    from deepviewagg_b200.core.multimodal.mapping import knn_grid, knn_query
    gen = torch.Generator().manual_seed(30 + k)
    pos = (torch.rand(20000, 3, generator=gen) * torch.tensor([10.0, 8.0, 3.0])).cuda()
    a, da = knn_grid(pos, k, return_dist2=True)
    b, db = knn_query(pos, pos, k, return_dist2=True)
    assert torch.equal(a, b) and torch.equal(da, db)


def test_knn_query_empty_and_small():
    from deepviewagg_b200 import _lib
    from deepviewagg_b200.core.multimodal.mapping import knn_query
    s = torch.rand(10, 3, device="cuda")
    n0 = _lib.launch_count()
    out = knn_query(torch.empty(0, 3, device="cuda"), s, 4)
    assert out.shape == (0, 4) and _lib.launch_count() == n0
    with pytest.raises(ValueError):
        knn_query(torch.rand(3, 3, device="cuda"), s, 11)
    with pytest.raises(ValueError):
        knn_query(torch.rand(3, 3, device="cuda"), torch.empty(0, 3, device="cuda"), 1)
