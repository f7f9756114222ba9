"""-m gpu: the LPIPS distance on the device (gaussianavatars_b200.lpips, gab200_lpips) and in the evaluation graph
(GraphedEval(lpips=)), with seeded weights (tests/lpips_oracle.py) and avatar renders scored against the display image
of the same avatar with perturbed parameters.

  * per conv layer: the kernel's own previous activations (its exact pools) through a float64 conv; every output
    within |d| <= (2^-10 + K 2^-23) sum|w x| + 2^-23 |b| (K = Cin k k) -- TF32 rounding to nearest of both operands
    (relative 2^-11 each, so 2^-10 + 2^-22 on a product, within the first term with room), FP32 accumulation of K
    products (at most K - 1 roundings of 2^-24 relative to the running sum of magnitudes, doubled for the tensor
    cores' internal ordering) and the FP32 bias add (2^-24 |b|, doubled);
  * pools bit for bit against max_pool2d of the kernel's own conv output; the head, given the kernel's target
    features, within 1e-6 relative of float64;
  * end to end, both networks, both sources, each network's smallest image, 97x131, 550x802 and 1920x1080: per view
    the error against the float64 oracle at most twice the largest error, over the same views, of the float32 torch
    restatement run with torch's default (TF32 cuDNN) convolution;
  * two calls give the same bits; GraphedEval rows equal eager lpips() bit for bit at K = 1 and 4 and through a
    schedule; an overflowed replay leaves its row NaN; the metric columns are the same with lpips= on and off."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import lpips_oracle as ol
from tests.test_gpu_camera_fov import _rig
from tests.test_gpu_metrics import Pipe, _eager_record, _models, _truth_u8

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIZES = {"alex": [(31, 31), (97, 131), (550, 802), (1920, 1080)],
         "vgg": [(16, 16), (97, 131), (550, 802), (1920, 1080)]}   # (W, H)
_NETS = {}


def _net(name):
    from gaussianavatars_b200.lpips import LpipsNet
    if name not in _NETS:
        feats, lin = ol.seeded_weights(name, ol.SEED[name])
        _NETS[name] = (LpipsNet(name, feats, lin, DEV), feats, lin)
    return _NETS[name]


@pytest.fixture(scope="module")
def avatar():
    return _models()


def _view(avatar, W, H, i, source):
    """(render source, gt_u8) of rig camera i at W x H: the avatar's float render or display bytes, and the display
    image of the perturbed avatar."""
    pc, truth, _ = avatar
    cam = _rig(W, H, n=4)[i % 4]
    bg = torch.ones(3)
    gt = _truth_u8(truth, cam, i % 8, bg)
    _, src = _eager_record(pc, cam, i % 8, bg, gt, source)
    return src.contiguous(), gt


def _u(b):
    """Bytes as value/255 correctly rounded to float32, as the kernel reads them: formed in double and rounded once, so
    the reference does not depend on how torch rounds a float32 division by a scalar."""
    return (b.double() / 255).float()


def _x(src):
    """The kernel's reading of a render source as a float32 (3,H,W) image in [0, 1]."""
    return _u(src.permute(2, 0, 1)) if src.dtype == torch.uint8 else src.clamp(0, 1)


# ---- per layer ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name, W, H", [("alex", 131, 97), ("vgg", 131, 97), ("alex", 802, 550)])
def test_every_conv_within_the_tf32_bound_pools_exact_head_float64(avatar, name, W, H):
    from gaussianavatars_b200.lpips import lpips, lpips_features
    net, feats, lin = _net(name)
    src, gt = _view(avatar, W, H, 1, "float")
    f = lpips_features(src, gt, net)
    d = float(lpips(src, gt, net))
    # the input stage is lpipsPyTorch's z-score of both images, in float32, exactly
    both = torch.stack([_x(src), _u(gt)])
    assert torch.equal(f["input"], ol.z_score(both)), "z-score"
    prev = f["input"]
    worst = 0.0
    for mod, s, p, pool, target in ol.conv_specs(name):
        w, b = feats[f"features.{mod}.weight"].to(DEV).double(), feats[f"features.{mod}.bias"].to(DEV).double()
        x = prev.double()
        ref = F.relu(F.conv2d(x, w, b, stride=s, padding=p))
        mag = F.conv2d(x.abs(), w.abs(), stride=s, padding=p)
        K = w.shape[1] * w.shape[2] * w.shape[3]
        bound = (2.0 ** -10 + K * 2.0 ** -23) * mag + 2.0 ** -23 * b.abs()[None, :, None, None]
        got = f[mod + 1].double()
        err = (got - ref).abs()
        ratio = float((err / bound.clamp_min(1e-300)).max())
        worst = max(worst, ratio)
        assert bool((err <= bound).all()), f"{name} conv {mod}: |d| over the bound (max ratio {ratio:.3f})"
        prev = f[mod + 1]
        if pool:
            k = ol.NETS[name]["pool"]
            assert torch.equal(f[mod + 2], F.max_pool2d(prev, k, 2)), f"{name} pool {mod + 2}"
            prev = f[mod + 2]
    targets = [f[mod + 1].double() for mod, _, _, _, t in ol.conv_specs(name) if t]
    head = float(ol.head([t[0:1] for t in targets], [t[1:2] for t in targets], lin)[0])
    rel = abs(d - head) / abs(head)
    print(f"[lpips] {name} {W}x{H}: worst |d| / bound over the convs {worst:.3f}; head rel {rel:.2e}")
    assert rel <= 1e-6, f"{name}: head {d!r} vs float64 {head!r} (rel {rel:.2e})"


# ---- end to end -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("source", ["float", "u8"])
@pytest.mark.parametrize("name", ["alex", "vgg"])
def test_end_to_end_error_is_within_twice_the_float32_reference(avatar, name, source):
    from gaussianavatars_b200.lpips import lpips
    net, feats, lin = _net(name)
    f32 = {k: v.to(DEV) for k, v in feats.items()}, {k: v.to(DEV) for k, v in lin.items()}
    f64 = {k: v.to(DEV).double() for k, v in feats.items()}, {k: v.to(DEV).double() for k, v in lin.items()}
    rows = []
    for (W, H) in SIZES[name]:
        for i in range(2 if W * H < 10 ** 5 else 1):
            src, gt = _view(avatar, W, H, 2 * i + 1, source)
            got = float(lpips(src, gt, net))
            x, y = _x(src)[None], _u(gt)[None]
            ref = float(ol.lpips(x.double(), y.double(), name, *f64)[0])
            torch32 = float(ol.lpips(x, y, name, *f32)[0])
            rows.append((W, H, got, ref, abs(got - ref), abs(torch32 - ref)))
    cap = 2 * max(r[5] for r in rows)
    for W, H, got, ref, e, e32 in rows:
        print(f"[lpips] {name} {source} {W}x{H}: {got:.8f} float64 {ref:.8f} |d| kernel {e:.2e} "
              f"torch float32 (TF32 cuDNN) {e32:.2e}")
    for W, H, got, ref, e, e32 in rows:
        assert math.isfinite(got) and ref > 0
        assert e <= cap, f"{name} {source} {W}x{H}: |d| {e:.2e} > 2 x {cap / 2:.2e}"


# ---- consistency ----------------------------------------------------------------------------------------------------
def test_two_calls_give_identical_bits(avatar):
    from gaussianavatars_b200.lpips import lpips
    for name in ("alex", "vgg"):
        net = _net(name)[0]
        for source in ("float", "u8"):
            src, gt = _view(avatar, 802, 550, 2, source)
            first = lpips(src, gt, net).clone()
            for _ in range(2):
                assert torch.equal(lpips(src, gt, net), first), (name, source)


def test_identical_pair_scores_exactly_zero():
    from gaussianavatars_b200.lpips import lpips
    g = torch.Generator().manual_seed(4)
    gt = torch.randint(0, 256, (3, 64, 80), generator=g, dtype=torch.uint8).to(DEV)
    for name in ("alex", "vgg"):
        net = _net(name)[0]
        assert float(lpips(_u(gt), gt, net)) == 0.0
        assert float(lpips(gt.permute(1, 2, 0).contiguous(), gt, net)) == 0.0


def test_default_device_from_the_hub_cache_serves_lpips_and_graphed_eval(avatar, tmp_path):
    """LpipsNet.from_hub_cache("alex") as the documents show it: no device argument, so "cuda" -- resolved to the
    indexed current device that the images and the model report."""
    from gaussianavatars_b200.graph import GraphedEval
    from gaussianavatars_b200.lpips import LpipsNet, lpips
    explicit, feats, lin = _net("alex")
    ck = tmp_path / "checkpoints"
    ck.mkdir()
    torch.save({**feats, "classifier.1.weight": torch.zeros(4, 4)}, ck / "alexnet-owt-7be5be79.pth")
    torch.save({f"lin{i}.model.1.weight": lin[f"{i}.1.weight"] for i in range(5)}, ck / "alex.pth")
    net = LpipsNet.from_hub_cache("alex", hub_dir=str(tmp_path))
    assert net.device == torch.device("cuda", torch.cuda.current_device()) == explicit.device
    assert torch.equal(net.weights, explicit.weights)
    src, gt = _view(avatar, 400, 304, 1, "float")
    assert torch.equal(lpips(src, gt, net), lpips(src, gt, explicit))
    pc, _, _ = avatar
    cam = _rig(400, 304, n=4)[1]
    ev = GraphedEval(pc, 400, 304, torch.ones(3), views=1, warm_cameras=[cam], warm_timesteps=[1], lpips=net)
    ev.set_inputs(camera=cam, timestep=1, gt_u8=gt, view=0)
    ev.run(check=True)
    assert torch.equal(ev.scores()["lpips_per_view"][0], lpips(src, gt, net).cpu())


@pytest.mark.parametrize("source", ["float", "u8"])
def test_graphed_eval_rows_equal_eager_lpips_and_leave_the_metrics_alone(avatar, source):
    from gaussianavatars_b200.graph import GraphedEval
    from gaussianavatars_b200.lpips import lpips
    pc, truth, _ = avatar
    net = _net("alex")[0]
    W, H = 400, 304
    cams = _rig(W, H, n=6)
    ts = [3 * i % 8 for i in range(6)]
    bg = torch.ones(3)
    gts = [_truth_u8(truth, c, t, bg) for c, t in zip(cams, ts)]
    on = GraphedEval(pc, W, H, bg, views=6, source=source, warm_cameras=cams, warm_timesteps=range(8), lpips=net)
    off = GraphedEval(pc, W, H, bg, views=6, source=source, warm_cameras=cams, warm_timesteps=range(8))
    for ev in (on, off):
        for i in range(6):
            ev.set_inputs(camera=cams[i], timestep=ts[i], gt_u8=gts[i], view=i)
            ev.run(check=True)
    a, b = on.scores(), off.scores()
    assert torch.equal(a["per_view"], b["per_view"]), "lpips= changed a metric column"
    assert "lpips" not in b and a["lpips_per_view"].shape == (6,)
    for i in range(6):
        _, src = _eager_record(pc, cams[i], ts[i], bg, gts[i], source)
        ref = lpips(src, gts[i], net).cpu()
        assert torch.equal(a["lpips_per_view"][i], ref), f"view {i}: {float(a['lpips_per_view'][i])} vs {float(ref)}"
    total = 0.0
    for v in a["lpips_per_view"].tolist():
        total += v
    assert a["lpips"] == total / 6
    print(f"[lpips eval {source}] per view {a['lpips_per_view'].tolist()} mean {a['lpips']:.6f}")


def test_graphed_eval_k_views_rows_equal_single_view_rows_and_overflow_writes_none():
    from gaussianavatars_b200.graph import GraphedEval
    from tests.test_gpu_multiview import H_IMG, W_IMG, _flame_setup
    pc = _flame_setup()
    net = _net("vgg")[0]
    cams = [c.to(DEV) for c in _rig(W_IMG, H_IMG, n=8)]
    bg = torch.ones(3)
    gts = torch.randint(0, 256, (8, 3, H_IMG, W_IMG), generator=torch.Generator().manual_seed(5),
                        dtype=torch.uint8).to(DEV)
    steps = (1, 6)
    one = GraphedEval(pc, W_IMG, H_IMG, bg, views=8, warm_cameras=cams, warm_timesteps=steps, lpips=net)
    many = GraphedEval(pc, W_IMG, H_IMG, bg, views=8, views_per_replay=4, warm_cameras=[cams[:4], cams[4:]],
                       warm_timesteps=steps, lpips=net)
    for grp in range(2):
        for k in range(4):
            i = 4 * grp + k
            one.set_inputs(camera=cams[i], timestep=steps[grp], gt_u8=gts[i], view=i)
            one.run(check=True)
        many.set_inputs(cameras=cams[4 * grp:4 * grp + 4], timestep=steps[grp], gt_u8=gts[4 * grp:4 * grp + 4],
                        view=4 * grp)
        many.run(check=True)
    a, b = one.scores(), many.scores()
    assert torch.equal(a["lpips_per_view"], b["lpips_per_view"]), "K-view LPIPS rows differ from single-view rows"
    assert torch.equal(a["per_view"], b["per_view"]) and many.captures == 1

    small = GraphedEval(pc, W_IMG, H_IMG, bg, views=8, views_per_replay=4, capacity=2048, warm_cameras=[cams[:4]],
                        warm_timesteps=steps, lpips=net)
    small.set_inputs(cameras=cams[4:], timestep=1, gt_u8=gts[4:], view=4)
    small.run()
    assert small.overflowed()
    torch.cuda.synchronize()
    assert torch.isnan(small.lpips_table).all(), "an overflowed replay wrote an LPIPS row"
    with pytest.raises(RuntimeError, match="hold no score"):
        small.scores()


@pytest.mark.parametrize("K", [1, 4])
def test_scheduled_eval_lpips_rows_equal_the_host_fed_rows(K):
    from gaussianavatars_b200.graph import GraphedEval
    from tests import test_gpu_multiview_train as MV
    from tests.test_gpu_schedule import H_S, W_S, _records, _schedule
    R = 3
    groups, ts, ids, store = _records(R, K, seed=40 + K)
    s = _schedule(groups, ts, ids, K, None)
    pc, _ = MV._flame_trainable()
    net = _net("alex")[0]
    warm = groups[:2] if K > 1 else [c[0] for c in groups[:2]]
    common = dict(views=R * K, views_per_replay=K, warm_cameras=warm, lpips=net)
    ea = GraphedEval(pc, W_S, H_S, torch.ones(3), schedule=s, frames=store, **common)
    eb = GraphedEval(pc, W_S, H_S, torch.ones(3), **common)
    assert ea.run_all() == R
    for r in range(R):
        gt, _ = store.decode(ids[r])
        pose = dict(cameras=groups[r]) if K > 1 else dict(camera=groups[r][0])
        eb.set_inputs(timestep=ts[r], gt_u8=gt if K > 1 else gt[0], view=r * K, **pose)
        eb.run(check=True)
    a, b = ea.scores(), eb.scores()
    assert torch.equal(a["lpips_per_view"], b["lpips_per_view"]) and torch.equal(a["per_view"], b["per_view"])
