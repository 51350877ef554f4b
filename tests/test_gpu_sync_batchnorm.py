"""nn.SyncBatchNorm on the ResNet-18 and PPM encoders (ops._rn_conv_bn / ops._rn_bn_bwd split around one all-reduce
per BatchNorm and direction), with ranks spawned by torch.multiprocessing: gloo with two ranks on one device, and
NCCL with two ranks on two devices when there are two.

  * In a 1-rank group, the split path forced at the op level gives the fused path's bits: outputs, every gradient,
    running stats and counters.
  * Two ranks with 2 + 2, 1 + 3 and 0 + 4 images: the outputs concatenated, the input gradients and the parameter
    gradients summed over ranks match one unconverted process on all four images, and the float64 restatements on
    the union batch, within the bounds of tests/test_gpu_image_resnet18*.py; running stats and counters are equal on
    both ranks.  Eval mode and frozen encoders run no collective; two runs are bitwise equal; a global count of one
    value per channel raises ValueError on both ranks; a converted pool MLP equals nn.Linear + nn.SyncBatchNorm +
    LeakyReLU; a converted step runs no torch BatchNorm or cuDNN kernel."""
import os
import re
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

from deepviewagg_b200 import ops
from deepviewagg_b200.core.common_modules import FastBatchNorm1d, MLPLayer
from deepviewagg_b200.modules.multimodal.modalities import image as I
from test_gpu_image_encoder import l2rel, maxrel

pytestmark = pytest.mark.gpu

NAMES = ("ADE20KResNet18TruncatedLayer4", "ADE20KResNet18Pyramid", "ResNet18TruncatedLayer4", "CityscapesResNet18",
         "ADE20KResNet18PPM")
IMAGES = (4, 3, 64, 64)
_FOREIGN = re.compile(r"cudnn|batch_norm|batchnorm|bn_fw|bn_bw", re.I)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _helpers(name):
    """(make, kernel_branches, oracle) of the GPU test module of the encoder family."""
    if name == "ADE20KResNet18PPM":
        import test_gpu_image_ppm as T
        return (lambda seed: T.make(seed)), T.kernel_branches, T.oracle
    if name.startswith("ADE20K"):
        import test_gpu_image_resnet18 as T
    else:
        import test_gpu_image_resnet18_families as T
    return (lambda seed: T.make(getattr(I, name), seed)), T.kernel_branches, T.oracle


def build(name, seed=3):
    return _helpers(name)[0](seed).train()


def inputs(name, seed=11):
    """The union batch x [4, 3, 64, 64] and an output gradient for it (CPU generator: the same on every rank)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(IMAGES, generator=g)
    with torch.no_grad():
        shape = build(name).eval()(x[:1].cuda()).shape[1:]
    return x.cuda(), torch.randn(IMAGES[0], *shape, generator=g).cuda()


def step(m, x, gy):
    """(y, gx, {parameter: grad}) of one forward + backward."""
    x = x.detach().clone().requires_grad_(True)
    y = m(x)
    names = [k for k, p in m.named_parameters() if p.requires_grad]
    params = dict(m.named_parameters())
    g = torch.autograd.grad(y, [x] + [params[k] for k in names], gy)
    return y.detach(), g[0], dict(zip(names, g[1:]))


def buffers(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}


class _Collectives:
    """Counts torch.distributed.all_reduce calls while installed."""

    def __init__(self):
        self.calls, self._orig = 0, dist.all_reduce

    def __enter__(self):
        def counted(*a, **kw):
            self.calls += 1
            return self._orig(*a, **kw)
        dist.all_reduce = counted
        return self

    def __exit__(self, *exc):
        dist.all_reduce = self._orig


def _cpu(t):
    """A tensor (or a dict of them) as numpy arrays: tensors in a Queue are shared through fds that die with the
    sender."""
    if isinstance(t, dict):
        return {k: _cpu(v) for k, v in t.items()}
    return t.detach().cpu().numpy()


def _tensors(obj):
    """The numpy arrays _cpu made, back as CPU tensors, through tuples and dicts."""
    if isinstance(obj, dict):
        return {k: _tensors(v) for k, v in obj.items()}
    if isinstance(obj, (tuple, list)):
        return type(obj)(_tensors(v) for v in obj)
    return torch.from_numpy(obj) if hasattr(obj, "dtype") and hasattr(obj, "shape") else obj


def _init(rank, world, port, backend):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dist.init_process_group(backend, rank=rank, world_size=world)


def _spawn(target, world, *args):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, port, q, *args)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(_tensors(q.get(timeout=900)) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


# ---- one rank: the split path forced at the op level against the fused path
def _one_rank_worker(rank, world, port, q, backend):
    _init(rank, world, port, backend)
    out = {}
    for name in NAMES:
        x, gy = inputs(name)
        m = nn.SyncBatchNorm.convert_sync_batchnorm(build(name))
        state = {k: v.clone() for k, v in m.state_dict().items()}
        n_bn = sum(isinstance(b, nn.SyncBatchNorm) for b in m.modules())
        with _Collectives() as fused_calls:
            fused = step(m, x, gy), buffers(m)
        m.load_state_dict(state)
        with ops.sync_batchnorm_split_at_one_rank(), _Collectives() as split_calls:
            split = step(m, x, gy), buffers(m)
        out[name] = (_cpu(fused[0][0]), _cpu(fused[0][1]), _cpu(fused[0][2]), _cpu(fused[1]), _cpu(split[0][0]),
                     _cpu(split[0][1]), _cpu(split[0][2]), _cpu(split[1]), fused_calls.calls, split_calls.calls, n_bn)
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_split_path_in_a_one_rank_group_is_bitwise_the_fused_path():
    backend = "nccl" if dist.is_nccl_available() else "gloo"
    (out,) = _spawn(_one_rank_worker, 1, backend)
    for name, (y, gx, gp, run, ys, gxs, gps, runs, n_fused, n_split, n_bn) in out.items():
        assert n_fused == 0 and n_split == 2 * n_bn, (name, n_fused, n_split, n_bn)
        assert torch.equal(y, ys) and torch.equal(gx, gxs), name
        assert set(gp) == set(gps) and all(torch.equal(gp[k], gps[k]) for k in gp), name
        assert set(run) == set(runs) and all(torch.equal(run[k], runs[k]) for k in run), name


# ---- two ranks
def _two_rank_worker(rank, world, port, q, backend, split):
    _init(rank, world, port, backend)
    lo = sum(split[:rank])
    hi = lo + split[rank]
    out = {}
    for name in NAMES:
        x, gy = inputs(name)
        m = nn.SyncBatchNorm.convert_sync_batchnorm(build(name))
        state = {k: v.clone() for k, v in m.state_dict().items()}
        with _Collectives() as calls:
            y, gx, gp = step(m, x[lo:hi], gy[lo:hi])
        run = buffers(m)
        m.load_state_dict(state)
        y2, gx2, gp2 = step(m, x[lo:hi], gy[lo:hi])
        again = (torch.equal(y, y2) and torch.equal(gx, gx2) and all(torch.equal(gp[k], gp2[k]) for k in gp)
                 and all(torch.equal(v, buffers(m)[k]) for k, v in run.items()))
        n_bn = sum(isinstance(b, nn.SyncBatchNorm) for b in m.modules())
        out[name] = (_cpu(y), _cpu(gx), _cpu(gp), _cpu(run), again, calls.calls, n_bn)
    # eval mode and a frozen encoder: no collective
    m = nn.SyncBatchNorm.convert_sync_batchnorm(build(NAMES[0])).eval()
    f = nn.SyncBatchNorm.convert_sync_batchnorm(I.ADE20KResNet18TruncatedLayer4(frozen=True).cuda()).train()
    x, _ = inputs(NAMES[0])
    with _Collectives() as calls, torch.no_grad():
        m(x[:2])
        f(x[:2])
    out["no_collective_in_eval"] = calls.calls
    # one value per channel over both ranks: ValueError on each
    conv = I.FusedConv2d(3, 8, kernel_size=3, padding=1, bias=False).cuda()
    bn = nn.SyncBatchNorm(8).cuda().train()
    try:
        ops.rn_conv_bn_relu(torch.randn(1 - rank, 1, 1, 3, device="cuda"), conv, bn)
        out["value_error"] = None
    except ValueError as e:
        out["value_error"] = str(e)
    # a converted pool MLP against nn.Linear + nn.SyncBatchNorm + LeakyReLU
    torch.manual_seed(5)
    mlp = MLPLayer(nn.Linear(24, 40, bias=False), FastBatchNorm1d(40), nn.LeakyReLU(0.2)).cuda()
    ref = nn.Sequential(nn.Linear(24, 40, bias=False), nn.BatchNorm1d(40), nn.LeakyReLU(0.2)).cuda()
    ref.load_state_dict({k.replace("1.batch_norm.", "1."): v for k, v in mlp.state_dict().items()})
    mlp, ref = (nn.SyncBatchNorm.convert_sync_batchnorm(t) for t in (mlp, ref))
    rows = torch.randn(37 + 20 * rank, 24, device="cuda")
    torch.backends.cuda.matmul.allow_tf32 = False
    out["mlp"] = (maxrel(mlp(rows).detach(), ref(rows).detach()),
                  maxrel(mlp[1].batch_norm.running_var, ref[1].running_var))
    # no torch BatchNorm or cuDNN kernel in a converted step
    from torch.profiler import ProfilerActivity, profile
    m = nn.SyncBatchNorm.convert_sync_batchnorm(build(NAMES[-1]))
    x, gy = inputs(NAMES[-1])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(m, x[lo:hi], gy[lo:hi])
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    out["foreign"] = sorted(n for n in names if _FOREIGN.search(n) and "dva_resnet::" not in n)
    out["ours"] = any("rn_bn_stats_kernel" in n for n in names) or hi == lo
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _reference(name):
    """One unconverted process on the union batch: (y, gx, grads, buffers), the model and its inputs."""
    m = build(name)
    x, gy = inputs(name)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    y, gx, gp = step(m, x, gy)
    run = buffers(m)
    m.load_state_dict(state)
    return _tensors((_cpu(y), _cpu(gx), _cpu(gp), _cpu(run))), m, x, gy


def _bounds(m):
    import test_gpu_image_resnet18 as T
    return T.bounds(m)


BACKENDS = [pytest.param("gloo", id="gloo-one-device"),
            pytest.param("nccl", id="nccl-two-devices", marks=pytest.mark.skipif(
                torch.cuda.device_count() < 2 or not dist.is_nccl_available(), reason="needs two GPUs and NCCL"))]


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("split", [(2, 2), (1, 3), (0, 4)], ids=lambda s: f"{s[0]}+{s[1]}")
def test_two_ranks_match_one_process_on_the_union_batch(backend, split):
    ranks = _spawn(_two_rank_worker, 2, backend, split)
    for name in NAMES:
        (y0, gx0, gp0, run0, again0, calls0, n_bn), (y1, gx1, gp1, run1, again1, calls1, _) = (r[name] for r in ranks)
        (ry, rgx, rgp, rrun), m, x, gy = _reference(name)
        bo, bg = _bounds(m)
        y, gx = torch.cat([y0, y1]), torch.cat([gx0, gx1])
        assert y.shape == ry.shape and maxrel(y, ry) <= bo, (name, maxrel(y, ry))
        assert l2rel(gx, rgx) <= bg, (name, l2rel(gx, rgx))
        # the gradient all-reduce sums the per-rank parameter gradients
        assert set(gp0) == set(gp1) == set(rgp)
        for k in rgp:
            assert l2rel(gp0[k] + gp1[k], rgp[k]) <= bg, (name, k, l2rel(gp0[k] + gp1[k], rgp[k]))
        # running stats identical on both ranks and those of the union batch; every counter moved once
        for k in run0:
            assert torch.equal(run0[k], run1[k]), (name, k)
            if "num_batches_tracked" in k:
                assert int(run0[k]) == int(build(name).state_dict()[k]) + 1, (name, k)
            else:
                assert maxrel(run0[k], rrun[k]) <= bo, (name, k, maxrel(run0[k], rrun[k]))
        assert again0 and again1, name
        assert calls0 == calls1 == 2 * n_bn, (name, calls0, calls1, n_bn)
        # the float64 restatement on the union batch, on the unconverted kernels' masks
        _, branches, oracle = _helpers(name)
        oy, ogx, ogp, _ = oracle(m, x, gy, masks=branches(m, x))
        assert maxrel(y, oy.float()) <= bo, (name, maxrel(y, oy.float()))
        assert l2rel(gx, ogx.float()) <= bg, (name, l2rel(gx, ogx.float()))
        for k in ogp:
            assert l2rel(gp0[k] + gp1[k], ogp[k].float()) <= bg, (name, k)
    r0, r1 = ranks
    assert r0["no_collective_in_eval"] == r1["no_collective_in_eval"] == 0
    assert r0["value_error"] and r0["value_error"] == r1["value_error"]
    assert "Expected more than 1 value per channel" in r0["value_error"]
    for r in ranks:
        assert r["mlp"][0] <= 1e-5 and r["mlp"][1] <= 1e-6, r["mlp"]
        assert not r["foreign"], r["foreign"]
        assert r["ours"]
