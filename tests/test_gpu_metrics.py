"""-m gpu: the evaluation metrics (training.image_metrics, gab200_image_metrics) and the evaluation graph (GraphedEval).

image_metrics is held to the reference's own float64 values (tests/golden/metrics_vectors.npz, from utils/loss_utils.py
and utils/image_utils.py) and, at full size, to the float64 restatement (tests/metrics_oracle.py): 1e-6 absolute on l1
and ssim (at full size: or the reference's own float32 error, if larger), 1e-4 dB on both PSNRs, in both of the
reference's forms -- train.py's (the clamped float render) and
metrics.py's (the display bytes).  A replay of GraphedEval is compared bit for bit with eager render() /
render_display() followed by image_metrics.  The ground truth of the avatar tests is the display image of the same
synthetic avatar with perturbed parameters (seeded), so the scores are those of a plausible half-trained model."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import metrics_oracle as om
from tests.test_gpu_camera_fov import _rig

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "metrics_vectors.npz"))
W_IMG, H_IMG = 400, 304


class Pipe:
    debug = False
    compute_cov3D_python = False
    convert_SHs_python = False


@pytest.fixture(autouse=True)
def culled_binning():
    """The library's default binning policy, whatever an earlier test left set (the capacities depend on it)."""
    import gaussianavatars_b200.rasterizer as R
    prev = R._EXACT_BINNING
    R.set_exact_binning(False)
    yield
    R.set_exact_binning(prev)


def _metrics(render, gt):
    from gaussianavatars_b200 import image_metrics
    out = image_metrics(render, gt)
    torch.cuda.synchronize()
    return out.cpu().double().numpy()


def _check(got, ref, what):
    """l1 / ssim within 1e-6, the PSNRs within 1e-4 dB (+inf exactly); returns the four absolute errors."""
    err = []
    for i, (name, tol) in enumerate((("l1", 1e-6), ("psnr", 1e-4), ("psnr_all", 1e-4), ("ssim", 1e-6))):
        if math.isinf(ref[i]):
            assert got[i] == ref[i], f"{what}: {name} {got[i]} != {ref[i]}"
            err.append(0.0)
        else:
            e = abs(got[i] - ref[i])
            assert e <= tol, f"{what}: {name} {got[i]!r} vs float64 {ref[i]!r} (|d| {e:.2e} > {tol})"
            err.append(e)
    return err


# ---- image_metrics against the reference --------------------------------------------------------------------------
def test_image_metrics_matches_the_reference_fixture_in_both_forms():
    errs = []
    for case in ("a", "b", "c", "same"):
        gt = torch.from_numpy(GOLD[f"{case}_gt_u8"]).to(DEV)
        got = _metrics(torch.from_numpy(GOLD[f"{case}_render"]).to(DEV), gt)
        errs.append(_check(got, GOLD[f"{case}_train_f64"], f"{case} float (train.py)"))
        got = _metrics(torch.from_numpy(GOLD[f"{case}_display_u8"]).to(DEV), gt)
        errs.append(_check(got, GOLD[f"{case}_metrics_f64"], f"{case} u8 (metrics.py)"))
    e = np.array(errs)
    print("[metrics] fixture |d| vs float64 reference: max l1 %.1e psnr %.1e dB psnr_all %.1e dB ssim %.1e; "
          "median %s" % (*e.max(axis=0), np.median(e, axis=0)))


def _render_like(H, W, seed):
    """A smooth render-like image that strays outside [0, 1], and a uint8 ground truth near it."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, H // 24 + 2, W // 24 + 2, generator=g)
    img = F.interpolate(low, size=(H, W), mode="bicubic", align_corners=False)[0] * 1.2 - 0.1
    gt = (img.clamp(0, 1) + 0.06 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    return img.contiguous(), (gt * 255).round().to(torch.uint8).contiguous()


def _quant(img):
    return img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8).contiguous()


def _ssim_float32(x, y):
    """The reference's own float32 arithmetic: grouped conv2d with the float32 2-D window (utils/loss_utils.py)."""
    from oracle import loss as ol
    return float(ol.photometric_torch(x.to(DEV), y.to(DEV), 0.2)[1])


@pytest.mark.parametrize("W, H", [(1920, 1080), (550, 802)])
def test_image_metrics_matches_the_float64_restatement_at_full_size(W, H):
    """1e-6 on l1 / ssim and 1e-4 dB on the PSNRs -- except that on a 2-megapixel image the float32 evaluation itself
    moves the mean SSIM by more than 1e-6 (sigma^2 = E[x^2] - mu^2 cancels): there the kernel must stay within the
    error of the reference's own float32 conv2d evaluation of the same inputs."""
    img, gt = _render_like(H, W, seed=W)
    disp = _quant(img.clone())
    gt_d = gt.to(DEV)
    for src, what in ((img, "float"), (disp, "u8")):
        got = _metrics(src.to(DEV), gt_d)
        ref = om.metrics(src.numpy(), gt.numpy())
        x = torch.from_numpy(om.inputs(src.numpy(), gt.numpy())[0]).float()
        floor = abs(_ssim_float32(x, gt.float() / 255) - ref[3])
        err = [abs(got[i] - ref[i]) for i in range(4)]
        print(f"[metrics] {W}x{H} {what}: {got} |d| vs float64 {err}; reference float32 ssim |d| {floor:.2e}")
        assert err[0] <= 1e-6 and err[1] <= 1e-4 and err[2] <= 1e-4, f"{W}x{H} {what}"
        assert err[3] <= max(1e-6, floor), f"{W}x{H} {what}: ssim |d| {err[3]:.2e}, float32 reference {floor:.2e}"


def test_records_are_bit_identical_run_to_run():
    from gaussianavatars_b200 import image_metrics
    img, gt = _render_like(1080, 1920, seed=3)
    img, gt, disp = img.to(DEV), gt.to(DEV), _quant(img).to(DEV)
    for src in (img, disp):
        first = image_metrics(src, gt).clone()
        for _ in range(3):
            assert torch.equal(image_metrics(src, gt), first)


def test_u8_source_is_metrics_py_reading_the_png():
    """The display image as a source equals the float source fed with display_u8.cpu().float() / 255 -- what
    metrics.py computes from the PNG render.py wrote (to_tensor: value / 255, correctly rounded)."""
    from gaussianavatars_b200 import image_metrics
    for (H, W), seed in (((802, 550), 1), ((37, 61), 2), ((1, 5), 3)):
        img, gt = _render_like(max(H, 24), max(W, 24), seed)
        img, gt = img[:, :H, :W].contiguous(), gt[:, :H, :W].contiguous().to(DEV)
        disp = _quant(img)
        as_png = (disp.permute(2, 0, 1).float() / 255).contiguous()
        assert torch.equal(image_metrics(disp.to(DEV), gt), image_metrics(as_png.to(DEV), gt)), (H, W)


# ---- GraphedEval ----------------------------------------------------------------------------------------------------
def _models(T=16):
    from tests.test_gpu_flame import _flame_model, _full_size, _lbs
    a, fp = _full_size(T=T, seed=2)
    pc = _flame_model(a, fp, _lbs(a))
    truth = _flame_model(a, fp, _lbs(a))
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():   # the "ground-truth" avatar: the same head, perturbed colours and positions
        truth._features_dc += 1.0 * torch.randn(truth._features_dc.shape, generator=g).to(DEV)
        truth._xyz += 0.01 * torch.randn(truth._xyz.shape, generator=g).to(DEV)
        truth._opacity += 1.0 * torch.randn(truth._opacity.shape, generator=g).to(DEV)
    return pc, truth, (a, fp)


def _truth_u8(truth, cam, t, bg):
    from gaussianavatars_b200.renderer import render_display
    truth.select_mesh_by_timestep(t)
    return render_display(cam.to(DEV), truth, Pipe, bg.to(DEV))["display_u8"].permute(2, 0, 1).contiguous()


def _eager_record(pc, cam, t, bg, gt, source):
    from gaussianavatars_b200 import image_metrics
    from gaussianavatars_b200.renderer import render, render_display
    pc.select_mesh_by_timestep(t)
    if source == "float":
        src = render(cam.to(DEV), pc, Pipe, bg.to(DEV))["render"].detach()
    else:
        src = render_display(cam.to(DEV), pc, Pipe, bg.to(DEV))["display_u8"]
    rec = image_metrics(src, gt).cpu()
    return rec, src


@pytest.mark.parametrize("source", ["float", "u8"])
def test_graphed_eval_rows_equal_eager_render_and_metrics(source):
    from gaussianavatars_b200.graph import GraphedEval
    pc, truth, _ = _models()
    cams = _rig(W_IMG, H_IMG)
    ts = [(5 * i) % 16 for i in range(16)]   # 16 distinct timesteps
    bg = torch.ones(3)
    gts = [_truth_u8(truth, c, t, bg) for c, t in zip(cams, ts)]
    if source == "u8":   # pinned host ground truth: uploaded on the copy stream the replay waits for
        gts = [g.cpu().pin_memory() for g in gts]
    ev = GraphedEval(pc, W_IMG, H_IMG, bg, views=16, source=source, host_slots=2 if source == "u8" else 0,
                     warm_cameras=cams, warm_timesteps=range(16))
    frames = []
    for i in (list(range(16))):
        ev.set_inputs(camera=cams[i], timestep=ts[i], gt_u8=gts[i], view=i)
        ev.run()
        if source == "u8":
            frames.append(ev.host_frame().clone())
    s = ev.scores()
    assert ev.captures == 1 and not ev.overflowed()
    for i in range(16):
        rec, src = _eager_record(pc, cams[i], ts[i], bg, gts[i].to(DEV), source)
        assert torch.equal(s["per_view"][i], rec), f"view {i}: {s['per_view'][i].tolist()} vs eager {rec.tolist()}"
        if source == "u8":
            assert torch.equal(frames[i], src.cpu()), f"view {i}: the host frame is not render.py's bytes"
    pv = s["per_view"].double()
    print(f"[eval {source}] ssim {pv[:, 3].min():.4f}..{pv[:, 3].max():.4f} psnr {pv[:, 1].min():.2f}.."
          f"{pv[:, 1].max():.2f} dB  means l1 {s['l1']:.5f} psnr {s['psnr']:.3f} psnr_all {s['psnr_all']:.3f} "
          f"ssim {s['ssim']:.4f}")
    assert 0.3 < float(pv[:, 3].min()) and float(pv[:, 3].max()) < 0.999, "unrealistic SSIM: the test sees nothing"
    assert bool(torch.isfinite(pv).all())
    assert s["l1"] == sum(float(v) for v in s["per_view"][:, 0].tolist()) / 16


def test_graphed_eval_overflow_leaves_no_score():
    from gaussianavatars_b200.graph import GraphedEval
    pc, truth, _ = _models(T=8)
    cams = _rig(W_IMG, H_IMG, n=4)
    bg = torch.ones(3)
    gts = [_truth_u8(truth, c, i, bg) for i, c in enumerate(cams)]
    ev = GraphedEval(pc, W_IMG, H_IMG, bg, views=4, source="float", capacity=2000)
    for i, c in enumerate(cams):
        ev.set_inputs(camera=c, timestep=i, gt_u8=gts[i], view=i)
        ev.run(check=False)
    assert ev.overflowed()
    torch.cuda.synchronize()
    assert torch.isnan(ev.table).all(), "a truncated render produced a score"
    with pytest.raises(RuntimeError, match=r"rows \[0, 1, 2, 3\].*regrow"):
        ev.scores()
    for i, c in enumerate(cams):
        ev.set_inputs(camera=c, timestep=i, gt_u8=gts[i], view=i)
        ev.run(check=True)
    s = ev.scores()
    assert ev.captures >= 2 and not ev.overflowed()
    for i, c in enumerate(cams):
        rec, _ = _eager_record(pc, c, i, bg, gts[i], "float")
        assert torch.equal(s["per_view"][i], rec), f"view {i} after regrow"


def _train(with_eval):
    """8 full training iterations (capturable Adam over the splat and FLAME groups, densification statistics, the
    photometric loss and the regularisers) over a 4-camera rig; with_eval: a GraphedEval pass over 4 validation views
    after iteration 4, as train.py's testing iterations run one."""
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.graph import GraphedEval, GraphedFrame, camera_block
    from tests.test_gpu_flame import LRS
    pc, truth, _ = _models(T=8)
    bg = torch.ones(3)
    cams = _rig(W_IMG, H_IMG, n=8)
    train_cams, val_cams = cams[0::2], cams[1::2]
    steps = [0, 1, 2, 3, 1, 0, 2, 3]
    gts = {(i, t): _truth_u8(truth, cams[i], t, bg) for i in range(8) for t in range(8)}
    fgroups = g.flame_param_groups(pc.flame_param)
    groups = [{"params": [p], "lr": LRS[n], "name": n} for n, p in zip(LRS, pc.parameters())]
    opt = g.Adam(groups + fgroups, lr=0.0, eps=1e-15, capturable=True)
    P = pc._xyz.shape[0]
    for n in ("xyz_gradient_accum", "denom"):
        setattr(pc, n, torch.zeros((P, 1), device=DEV))
    pc.max_radii2D = torch.zeros((P,), device=DEV)
    blocks = [camera_block(c, fov=True).to(DEV) for c in train_cams]
    fr = GraphedFrame(pc, W_IMG, H_IMG, cams[0].FoVx, cams[0].FoVy, bg, loss="photometric", regularizers={},
                      optimizer=opt, densify_stats=True, per_camera_fov=True, warm_cameras=blocks)
    losses, scores, eager = [], None, None
    for i, t in enumerate(steps):
        if with_eval and i == 4:
            ev = GraphedEval(pc, W_IMG, H_IMG, bg, views=4, warm_cameras=val_cams, warm_timesteps=range(4, 8))
            for j, c in enumerate(val_cams):
                ev.set_inputs(camera=c, timestep=4 + j, gt_u8=gts[(2 * j + 1, 4 + j)], view=j)
                ev.run(check=True)
            scores = ev.scores()
            eager = [_eager_record(pc, c, 4 + j, bg, gts[(2 * j + 1, 4 + j)], "float")[0]
                     for j, c in enumerate(val_cams)]
        k = i % 4
        fr.set_inputs(camera=blocks[k], timestep=t, gt_u8=gts[(2 * k, t)])
        fr.run(check=True)
        losses.append(float(fr.loss))
    assert fr.captures == 1
    return losses, scores, eager


def test_an_evaluation_between_training_replays_changes_no_training_step():
    plain, _, _ = _train(False)
    losses, scores, eager = _train(True)
    for i, (a, b) in enumerate(zip(losses, plain)):
        rel = abs(a - b) / abs(b)
        print(f"[train+eval] step {i} loss {a:.7f} without the evaluation {b:.7f} rel {rel:.1e}")
        assert rel <= 1e-4, f"step {i}: the evaluation changed the training"
    for j in range(4):
        assert torch.equal(scores["per_view"][j], eager[j]), f"validation view {j}"
    print(f"[train+eval] scores at iteration 4: l1 {scores['l1']:.5f} psnr {scores['psnr']:.3f} "
          f"ssim {scores['ssim']:.4f}")
