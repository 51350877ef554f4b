"""ADE20KResNet18PPM without a GPU: the float64 restatement oracle/image_ppm_oracle.py against the fixtures made by
executing the reference's wrapper (oracle/make_golden_image_ppm.py), the module's state-dict keys against the
reference's, load_mit_semseg_decoder against the decoder checkpoint's layout, the torch bins of the pool index, and
the frozen / train() semantics."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from deepviewagg_b200 import ops
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_ppm_oracle as O
from oracle import image_resnet18_oracle as R

CASES = {  # oracle/make_golden_image_ppm.py:CASES
    "train_b2": (True, (2, 3, 61, 45), None, 21),
    "train_b1": (True, (1, 3, 50, 66), None, 22),
    "eval_outsize": (False, (2, 3, 40, 56), (40, 56), 23),
}
Y_CHANNEL_STEP = {"eval_outsize": 32}


def _keys():
    return np.load(f"{GOLDEN}/image_ppm_keys.npz")


def case_inputs(name):
    """(module, float64 state, x, seed) of a seeded case, regenerated from the integer-hash generator."""
    training, shape, _, seed = CASES[name]
    m = I.ADE20KResNet18PPM().train(training)
    state = R.hashed_state(m.state_dict(), seed)
    x = torch.from_numpy(R.hash_grid(seed, 50000, shape, 8, 2))
    return m, state, x, seed


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_seeded_reference_cases(name):
    g = np.load(f"{GOLDEN}/image_ppm_{name}.npz")
    m, state, x, seed = case_inputs(name)
    out_size = CASES[name][2]
    assert float(x.sum()) == float(g["checksum:x"])
    for k, v in state.items():
        if k.endswith((".weight", ".bias", ".running_mean", ".running_var")):
            assert float(v.double().sum()) == float(g[f"checksum:{k}"]), k
            assert torch.equal(v.float().double(), v), k            # the grid is exact in float32
    p = {k: v.clone() for k, v in state.items()}
    names = [k for k, _ in m.named_parameters()]
    for k in names:
        p[k].requires_grad_(True)
    x.requires_grad_(True)
    y = O.forward(x, p, m.training, out_size)
    gy = torch.from_numpy(R.hash_grid(seed, 60000, tuple(y.shape), 8, 3))
    grads = torch.autograd.grad(y, [x] + [p[k] for k in names], gy)
    u = 2.0 ** -24
    ys = y.detach()[:, ::Y_CHANNEL_STEP.get(name, 1)].float().numpy()
    assert np.abs(ys - g["y"]).max() <= u * np.abs(g["y"]).max()
    assert np.abs(grads[0].float().numpy() - g["gx"]).max() <= u * np.abs(g["gx"]).max()
    assert abs(float(y.detach().norm()) / float(g["y_norm"]) - 1) <= 1e-12
    assert abs(float(grads[0].norm()) / float(g["gx_norm"]) - 1) <= 1e-12
    for tag, (k, gp) in enumerate(zip(names, grads[1:])):
        assert abs(float(gp.norm()) / float(g[f"gnorm:{k}"]) - 1) <= 1e-12, k
        proj = float((gp * R.projection(seed, tag, tuple(gp.shape))).sum())
        assert abs(proj - float(g[f"gproj:{k}"])) <= 1e-12 * float(g[f"gnorm:{k}"]) * gp.numel() ** 0.5, k
    for k in state:
        if k.endswith((".running_mean", ".running_var")):
            assert np.allclose(p[k].detach().numpy(), g[f"after:{k}"], rtol=1e-14, atol=0), k


def test_the_prudent_branch_keeps_its_running_stats_at_batch_size_1():
    g = np.load(f"{GOLDEN}/image_ppm_train_b1.npz")
    _, state, _, _ = case_inputs("train_b1")
    for k in state:
        if k.endswith((".running_mean", ".running_var")):
            same = np.array_equal(g[f"after:{k}"], state[k].numpy())
            assert same == k.startswith("decoder.ppm.0.2."), k


def test_state_dict_keys_are_the_reference_wrappers():
    assert list(I.ADE20KResNet18PPM().state_dict()) == list(_keys()["keys:ADE20KResNet18PPM"])


def _decoder_state_dict():
    k = _keys()
    shapes = [tuple(int(v) for v in s.strip("()").split(",") if v.strip()) for s in k["ckpt_shapes"]]
    return {name: (torch.zeros(shape, dtype=torch.int64) if name.endswith("num_batches_tracked")
                   else torch.full(shape, 0.5)) for name, shape in zip(k["ckpt_keys"], shapes)}


def test_load_mit_semseg_decoder_takes_exactly_the_checkpoint_layout():
    sd = _decoder_state_dict()
    assert len(sd) == 58
    enc = {k[len("encoder."):]: v for k, v in I.ADE20KResNet18PPM().state_dict().items() if k.startswith("encoder.")}
    m = I.ADE20KResNet18PPM(weights=(enc, sd), pretrained=True)
    assert all(float(p.detach().min()) == 0.5 for p in m.decoder.parameters())
    assert torch.equal(m.encoder.conv1.weight, enc["conv1.weight"])
    dec = I.load_mit_semseg_decoder(I.PPMFeatMap(fc_dim=512), sd)
    assert float(dec.conv_last[0].weight.detach().min()) == 0.5
    missing = dict(sd)
    missing.pop("conv_last_deepsup.bias")
    with pytest.raises(KeyError, match="missing"):
        I.load_mit_semseg_decoder(I.ADE20KResNet18PPM(), missing)
    with pytest.raises(KeyError, match="unexpected"):
        I.load_mit_semseg_decoder(I.ADE20KResNet18PPM(), {**sd, "conv_last.5.weight": torch.zeros(1)})


def test_module_tree_frozen_and_train():
    m = I.ADE20KResNet18PPM(pretrained=False, foo=1)
    assert (m.input_nc, m.output_nc) == (3, 512)
    assert [b[0].output_size for b in m.decoder.ppm] == [1, 2, 3, 6]
    assert all(isinstance(b[2], I.PrudentSynchronizedBatchNorm2d) for b in m.decoder.ppm)
    assert type(m.decoder.conv_last[1]) is I.SynchronizedBatchNorm2d and m.decoder.conv_last[1].momentum == 0.001
    assert m.decoder.conv_last[0].weight.shape == (512, 2560, 3, 3)
    assert len(list(m.parameters())) == 69 + 15
    assert m.training and all(p.requires_grad for p in m.parameters())
    f = I.ADE20KResNet18PPM(frozen=True)
    assert f.frozen and not f.training and not any(p.requires_grad for p in f.parameters())
    # the reference's quirk: frozen=True sets only the wrapper's training flag until train() is called
    assert f.decoder.training
    f.train()
    assert not f.training and not any(mod.training for mod in f.modules())
    f.frozen = False
    f.train()
    assert f.training and all(p.requires_grad for p in f.parameters())
    for mod in (m.decoder.ppm[0][0], m.decoder.ppm[0][2]):
        with pytest.raises(NotImplementedError):
            mod(torch.zeros(1, 512, 4, 4))


@pytest.mark.parametrize("h,w", [(1, 1), (2, 5), (5, 7), (6, 6), (8, 6), (13, 4)])
def test_pool_index_is_torchs_bins(h, w):
    """The gather-pool index (built here on the CPU): the mean of each atom's pixels is F.adaptive_avg_pool2d, scale
    by scale, image by image, bin by bin (bins overlap and repeat where s does not divide the side)."""
    B = 2
    x = torch.randn(B, h, w, 3, dtype=torch.float64)
    img, pix, aptr, offsets = ops._ppm_index(B, h, w, O.SCALES, "cpu")
    assert offsets == [0, B, 5 * B, 14 * B] and img.numel() == 50 * B and int(aptr[-1]) == pix.shape[0]
    vals = x[img.repeat_interleave(aptr.diff()), pix[:, 1].long(), pix[:, 0].long()]
    got = torch.zeros(img.numel(), 3, dtype=torch.float64).index_add_(
        0, torch.arange(img.numel()).repeat_interleave(aptr.diff()), vals) / aptr.diff()[:, None]
    for k, s in enumerate(O.SCALES):
        ref = F.adaptive_avg_pool2d(x.permute(0, 3, 1, 2), s).permute(0, 2, 3, 1).reshape(-1, 3)
        assert torch.allclose(got[offsets[k]:offsets[k] + B * s * s], ref, rtol=1e-13, atol=1e-15), (h, w, s)


def test_prudent_rule():
    bn = I.PrudentSynchronizedBatchNorm2d(8)
    assert not ops.ppm_branch_training(bn, 1, 1)
    assert ops.ppm_branch_training(bn, 2, 1) and ops.ppm_branch_training(bn, 1, 2)
    assert not ops.ppm_branch_training(bn.eval(), 2, 2)
