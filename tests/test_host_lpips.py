"""CPU: the LPIPS surface without a GPU -- the gab200_lpips entry points (exports, ctypes signatures against the
header, the struct mirror, argument checks that reject before any device work, the scratch and weight sizes), the
refusals of LpipsNet, lpips() and from_hub_cache, and GraphedEval(lpips=): its checks, the NaN table, scores()."""
import ctypes as C
import math
import os
import re
from types import SimpleNamespace

import pytest
import torch

from tests import lpips_oracle as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMMY = 0x1000   # never dereferenced: every call below is rejected during argument validation


def _hdr():
    return open(os.path.join(ROOT, "include", "gab200_rasterizer.h")).read()


def _params(sig):
    return [p.strip() for p in re.search(sig, _hdr(), re.S).group(1).split(",")]


def test_lpips_entry_points_are_exported_with_the_header_signatures():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    for s in ("gab200_lpips", "gab200_lpips_pack", "gab200_lpips_weights_bytes", "gab200_lpips_scratch_bytes",
              "gab200_lpips_features_bytes"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(L, s)
    assert L.gab200_lpips.restype is C.c_int32 and L.gab200_lpips.argtypes == [C.POINTER(N.LpipsArgs), C.c_void_p]
    assert _params(r"int32_t gab200_lpips\(([^)]*)\);") == ["const gab200_lpips_args* args", "void* stream"]
    assert L.gab200_lpips_weights_bytes.restype is C.c_size_t
    assert L.gab200_lpips_weights_bytes.argtypes == [C.c_int32]
    assert _params(r"size_t gab200_lpips_weights_bytes\(([^)]*)\);") == ["int32_t net"]
    assert L.gab200_lpips_scratch_bytes.restype is C.c_size_t
    assert L.gab200_lpips_scratch_bytes.argtypes == [C.c_int32] * 3
    assert _params(r"size_t gab200_lpips_scratch_bytes\(([^)]*)\);") == ["int32_t net", "int32_t height",
                                                                         "int32_t width"]
    assert L.gab200_lpips_features_bytes.restype is C.c_size_t
    assert L.gab200_lpips_features_bytes.argtypes == [C.c_int32] * 3
    assert _params(r"size_t gab200_lpips_features_bytes\(([^)]*)\);") == ["int32_t net", "int32_t height",
                                                                          "int32_t width"]
    assert L.gab200_lpips_pack.restype is C.c_int32
    assert L.gab200_lpips_pack.argtypes == [C.c_int32] + [C.POINTER(C.c_void_p)] * 3 + [C.c_void_p] * 2
    assert _params(r"int32_t gab200_lpips_pack\(([^)]*)\);") == [
        "int32_t net", "const float* const* conv_weight", "const float* const* conv_bias",
        "const float* const* lin_weight", "void* packed", "void* stream"]
    assert re.search(r"GAB200_LPIPS_ALEX = (\d+)", _hdr()).group(1) == str(N.LPIPS_ALEX) == "0"
    assert re.search(r"GAB200_LPIPS_VGG16 = (\d+)", _hdr()).group(1) == str(N.LPIPS_VGG16) == "1"
    assert L.gab200_abi_version() == N.ABI_VERSION == 3


def test_lpips_args_mirror_the_header_struct():
    from gaussianavatars_b200 import _native as N

    body = re.search(r"typedef struct gab200_lpips_args \{(.*?)\} gab200_lpips_args;", _hdr(), re.S).group(1)
    names = []
    for line in body.splitlines():
        decl = line.split("/*")[0].strip().rstrip(";")
        if decl:
            names += [n.strip().split()[-1].lstrip("*") for n in decl.split(None, 1)[1].split(",")]
    assert names == [f for f, _ in N.LpipsArgs._fields_]
    assert C.sizeof(N.LpipsArgs) == 96


def _plan_bytes(net, H, W):
    """The scratch formula restated: the per-CTA head partials in double (64 target pixels per CTA), rounded up to
    16 bytes, then two float32 buffers of the largest stage output of both images."""
    from gaussianavatars_b200.lpips import _stages
    stages = _stages(net, H, W)
    targets = [m for m, _, _, _, target in ol.conv_specs(net) if target]
    heads = sum(-(-h * w // 64) for key, c, h, w in stages if key in {m + 1 for m in targets})
    return -(-heads * 8 // 16) * 16 + 2 * 4 * max(2 * c * h * w for _, c, h, w in stages)


@pytest.mark.parametrize("net, side", [("alex", 31), ("vgg", 16)])
def test_scratch_formula_and_smallest_image(net, side):
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200.lpips import NETS

    L, nid = N.lib(), NETS[net]["id"]
    assert NETS[net]["min_side"] == side
    for H, W in ((side, side), (97, 131), (550, 802), (1080, 1920)):
        assert L.gab200_lpips_scratch_bytes(nid, H, W) == _plan_bytes(net, H, W), (H, W)
    assert L.gab200_lpips_scratch_bytes(nid, side - 1, side) == 0
    assert L.gab200_lpips_scratch_bytes(nid, side, side - 1) == 0
    assert L.gab200_lpips_scratch_bytes(nid, 0, 100) == 0 and L.gab200_lpips_scratch_bytes(7, 64, 64) == 0


@pytest.mark.parametrize("net, side", [("alex", 31), ("vgg", 16)])
def test_features_size_is_every_stage_of_both_images(net, side):
    """gab200_lpips_features_bytes sizes the `features` buffer: every stage output of both images in float32, in the
    order lpips_features slices it."""
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200.lpips import NETS, _stages

    L, nid = N.lib(), NETS[net]["id"]
    for H, W in ((side, side), (97, 131), (1080, 1920)):
        assert L.gab200_lpips_features_bytes(nid, H, W) == 4 * sum(2 * c * h * w for _, c, h, w in _stages(net, H, W))
    assert L.gab200_lpips_features_bytes(nid, side - 1, side) == 0
    assert L.gab200_lpips_features_bytes(nid, side, side - 1) == 0 and L.gab200_lpips_features_bytes(9, 64, 64) == 0
    if net == "vgg":   # two buffers of 64 channels of both 1080p images
        assert L.gab200_lpips_scratch_bytes(nid, 1080, 1920) >= 2 * 2 * 1080 * 1920 * 64 * 4


def test_packed_weights_size():
    from gaussianavatars_b200 import _native as N
    from gaussianavatars_b200.lpips import NETS

    for net in ("alex", "vgg"):
        floats = 0
        for _, cin, cout, k, _, target in NETS[net]["convs"]:
            floats += -(-k * k * (4 if cin == 3 else cin) // 32) * 32 * cout + cout + (cout if target else 0)
        assert N.lib().gab200_lpips_weights_bytes(NETS[net]["id"]) == 4 * floats
    assert N.lib().gab200_lpips_weights_bytes(2) == 0


def _args(**kw):
    from gaussianavatars_b200 import _native as N

    a = N.LpipsArgs()
    a.abi_version, a.net, a.height, a.width, a.render_kind = N.ABI_VERSION, N.LPIPS_VGG16, 40, 48, 0
    a.render = a.gt = a.weights = a.table = a.scratch = DUMMY
    a.table_rows = 4
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("bad", [
    dict(render=None), dict(gt=None), dict(weights=None), dict(table=None), dict(scratch=None),
    dict(scratch=DUMMY + 8), dict(weights=DUMMY + 4), dict(features=DUMMY + 4), dict(height=15), dict(width=15),
    dict(height=0), dict(net=2), dict(net=-1), dict(net=0, height=30), dict(table_rows=0), dict(render_kind=2),
    dict(abi_version=2),
], ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_lpips_rejects_invalid_arguments(bad):
    from gaussianavatars_b200 import _native as N

    assert N.lib().gab200_lpips(C.byref(_args(**bad)), None) == -1
    assert N.lib().gab200_lpips(None, None) == -1


def test_pack_rejects_invalid_arguments():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    arr = lambda n, v=DUMMY: (C.c_void_p * n)(*([v] * n))  # noqa: E731
    assert L.gab200_lpips_pack(2, arr(5), arr(5), arr(5), DUMMY, None) == -1               # unknown net
    assert L.gab200_lpips_pack(0, arr(5), arr(5), arr(5), DUMMY + 4, None) == -1           # misaligned
    assert L.gab200_lpips_pack(0, arr(5), arr(5), arr(5), None, None) == -1
    assert L.gab200_lpips_pack(0, None, arr(5), arr(5), DUMMY, None) == -1
    assert L.gab200_lpips_pack(1, arr(13), arr(13, None), arr(5), DUMMY, None) == -1       # a NULL bias
    assert L.gab200_lpips_pack(0, arr(5), arr(5), arr(5, None), DUMMY, None) == -1         # a NULL lin


# ---- LpipsNet -------------------------------------------------------------------------------------------------------
def _with(d, key, value=None, drop=False):
    d = dict(d)
    if drop:
        del d[key]
    else:
        d[key] = value
    return d


@pytest.mark.parametrize("net", ["alex", "vgg"])
def test_lpips_net_checks_every_key_shape_dtype_and_value(net):
    from gaussianavatars_b200.lpips import LpipsNet

    feats, lin = ol.seeded_weights(net, 0)
    w0 = "features.0.weight"
    for f, l, err in (
        (_with(feats, w0, drop=True), lin, KeyError),
        (_with(feats, "features.99.weight", torch.zeros(1)), lin, KeyError),
        (_with(feats, w0, feats[w0].double()), lin, TypeError),
        (_with(feats, w0, feats[w0][:, :, :-1]), lin, ValueError),
        (_with(feats, "features.0.bias", feats["features.0.bias"][:-1]), lin, ValueError),
        (_with(feats, w0, feats[w0].clone().index_fill_(0, torch.tensor([3]), math.nan)), lin, ValueError),
        (_with(feats, w0, feats[w0].clone().index_fill_(0, torch.tensor([0]), math.inf)), lin, ValueError),
        (feats, _with(lin, "0.1.weight", drop=True), KeyError),
        (feats, _with(lin, "5.1.weight", lin["0.1.weight"]), KeyError),
        (feats, {**{f"lin{i}.model.1.weight": lin[f"{i}.1.weight"] for i in range(4)}, "4.1.weight": lin["4.1.weight"]},
         KeyError),   # the two naming forms mixed
        (feats, _with(lin, "2.1.weight", lin["2.1.weight"][:, :-1]), ValueError),
        (feats, _with(lin, "1.1.weight", lin["1.1.weight"].half()), TypeError),
        (feats, _with(lin, "4.1.weight", lin["4.1.weight"] * math.nan), ValueError),
    ):
        with pytest.raises(err):
            LpipsNet(net, f, l, "cpu")
    with pytest.raises(ValueError, match="alex"):
        LpipsNet("squeeze", feats, lin, "cpu")
    # well-formed in both lin forms, with the classifier keys of a whole torchvision state dict: no CPU path
    file_form = {f"lin{i}.model.1.weight": lin[f"{i}.1.weight"] for i in range(5)}
    for l in (lin, file_form):
        with pytest.raises(RuntimeError, match="CPU"):
            LpipsNet(net, {**feats, "classifier.1.weight": torch.zeros(2, 2)}, l, "cpu")


def test_from_hub_cache_on_an_empty_hub_raises_without_downloading(tmp_path, monkeypatch):
    from gaussianavatars_b200.lpips import LpipsNet

    def no_network(*a, **k):
        raise AssertionError("from_hub_cache tried to download")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_network)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_network)
    for net, first, url in (("alex", "alexnet-owt-7be5be79.pth", "download.pytorch.org/models/alexnet-owt-7be5be79"),
                            ("vgg", "vgg16-397923af.pth", "download.pytorch.org/models/vgg16-397923af")):
        with pytest.raises(FileNotFoundError, match=re.escape(os.path.join(str(tmp_path), "checkpoints", first))) as e:
            LpipsNet.from_hub_cache(net, hub_dir=str(tmp_path))
        assert url in str(e.value)
        os.makedirs(tmp_path / "checkpoints", exist_ok=True)
        torch.save({}, tmp_path / "checkpoints" / first)   # the features file alone: the lin file is named next
        with pytest.raises(FileNotFoundError, match=f"{net}.pth") as e:
            LpipsNet.from_hub_cache(net, hub_dir=str(tmp_path))
        assert f"PerceptualSimilarity/master/lpips/weights/v0.1/{net}.pth" in str(e.value)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "default"))
    with pytest.raises(FileNotFoundError, match=re.escape(str(tmp_path / "default" / "checkpoints"))):
        LpipsNet.from_hub_cache("alex")


def _fake_net(net="vgg", device="cpu"):
    from gaussianavatars_b200.lpips import NETS, LpipsNet

    n = object.__new__(LpipsNet)
    n.net, n.id, n.device, n.min_side = net, NETS[net]["id"], torch.device(device), NETS[net]["min_side"]
    n.weights = torch.zeros(16, dtype=torch.uint8)
    return n


def test_lpips_checks_its_inputs():
    from gaussianavatars_b200.lpips import lpips

    net = _fake_net("alex")
    gt = torch.zeros((3, 40, 33), dtype=torch.uint8)
    with pytest.raises(ValueError, match="31x31"):
        lpips(torch.zeros((3, 30, 33)), torch.zeros((3, 30, 33), dtype=torch.uint8), net)
    with pytest.raises(ValueError, match="31x31"):
        lpips(torch.zeros((40, 30, 3), dtype=torch.uint8), gt, net)
    with pytest.raises(ValueError, match="16x16"):
        lpips(torch.zeros((3, 15, 20)), torch.zeros((3, 15, 20), dtype=torch.uint8), _fake_net("vgg"))
    for render in (torch.zeros((3, 40, 33), dtype=torch.float64), torch.zeros((4, 40, 33)),
                   torch.zeros((40, 33, 3)), torch.zeros((1, 3, 40, 33))):
        with pytest.raises(TypeError):
            lpips(render, gt, net)
    with pytest.raises(TypeError, match="uint8"):
        lpips(torch.zeros((3, 40, 33)), gt.float(), net)
    with pytest.raises(ValueError, match="shape"):
        lpips(torch.zeros((3, 40, 33)), torch.zeros((3, 40, 32), dtype=torch.uint8), net)
    with pytest.raises(TypeError, match="LpipsNet"):
        lpips(torch.zeros((3, 40, 33)), gt, "alex")
    with pytest.raises(RuntimeError, match="CPU"):   # well-formed, but there is no CPU path
        lpips(torch.zeros((3, 40, 33)), gt, net)


# ---- GraphedEval(lpips=) --------------------------------------------------------------------------------------------
def _pc():
    return SimpleNamespace(_xyz=torch.zeros(4, 3), verts_rest=torch.zeros(5, 3))


def test_graphed_eval_lpips_argument_checks():
    from gaussianavatars_b200.graph import GraphedEval

    with pytest.raises(TypeError, match="LpipsNet"):
        GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, lpips="alex")
    with pytest.raises(ValueError, match="31x31"):
        GraphedEval(_pc(), 64, 30, torch.zeros(3), views=4, lpips=_fake_net("alex"))
    with pytest.raises(ValueError, match="16x16"):
        GraphedEval(_pc(), 15, 48, torch.zeros(3), views=4, lpips=_fake_net("vgg"))
    with pytest.raises(ValueError, match="cuda"):
        GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, lpips=_fake_net("vgg", "cuda"))
    ev = GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4, lpips=_fake_net("vgg"))
    assert ev.lpips_table.shape == (4,) and torch.isnan(ev.lpips_table).all()
    assert GraphedEval(_pc(), 64, 48, torch.zeros(3), views=4).lpips_table is None


def test_scores_raise_on_a_missing_lpips_row_and_form_the_training_report_mean():
    from gaussianavatars_b200.graph import GraphedEval

    ev = GraphedEval(_pc(), 64, 48, torch.zeros(3), views=3, lpips=_fake_net("alex"))
    ev.table[:] = torch.tensor([[0.1, 20.5, 20.25, 0.7], [0.2, 21.5, 21.0, 0.8], [0.3, 22.0, 22.5, 0.9]])
    with pytest.raises(RuntimeError, match=r"rows \[0, 1, 2\]"):
        ev.scores()
    ev.lpips_table[:2] = torch.tensor([0.125, 0.3])
    with pytest.raises(RuntimeError, match=r"rows \[2\]"):
        ev.scores()
    s = ev.scores(n=2)
    assert s["lpips_per_view"].dtype == torch.float32 and s["lpips_per_view"].shape == (2,)
    v = s["lpips_per_view"].tolist()
    assert s["lpips"] == (0.0 + v[0] + v[1]) / 2    # the float32 values summed in double
    assert torch.equal(s["per_view"], ev.table[:2])
    ev.reset()
    assert torch.isnan(ev.lpips_table).all() and torch.isnan(ev.table).all()
