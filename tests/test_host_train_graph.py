"""CPU: the C ABI of the capturable Adam and of the densification statistics (exports, struct layout of the ctypes
mirror) and the host-side argument checks of the whole-iteration graph -- no compute calls (no GPU)."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
HEADER = os.path.join(ROOT, "include", "gab200_rasterizer.h")


def test_new_entry_points_are_exported_and_abi_version_is_unchanged():
    from gaussianavatars_b200 import _native as N

    lib = N.lib()
    for s in ("gab200_adam_step_device", "gab200_densify_stats"):
        assert s in N.EXPORTED_SYMBOLS and hasattr(lib, s)
    assert lib.gab200_abi_version() == N.ABI_VERSION == 3


def test_adam_device_segment_mirror_matches_the_c_layout(tmp_path):
    from gaussianavatars_b200 import _native as N

    ct, cname = N.AdamDeviceSegment, "gab200_adam_device_segment"
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(){",
             f'printf("{cname} %zu\\n", sizeof({cname}));']
    lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in ct._fields_]
    lines.append("return 0;}")
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run(["/usr/bin/gcc", str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
               if l.strip())
    assert int(got[cname]) == C.sizeof(ct)
    for f, _ in ct._fields_:
        assert int(got[f"{cname}.{f}"]) == getattr(ct, f).offset, f


def test_invalid_arguments_are_rejected_before_any_launch():
    from gaussianavatars_b200 import _native as N

    L = N.lib()
    seg = N.AdamDeviceSegment(None, None, None, None, 4, None, 1e-3)   # no step counter
    assert L.gab200_adam_step_device(1, C.byref(seg), 0.9, 0.999, 1e-15, None, None) == -1
    seg = N.AdamDeviceSegment(1, 1, 1, 1, 4, 1, 1e-3)
    seg.has_schedule, seg.lr_init, seg.lr_final, seg.max_steps = 1, 1e-3, 1e-5, 0   # max_steps must be > 0
    assert L.gab200_adam_step_device(1, C.byref(seg), 0.9, 0.999, 1e-15, None, None) == -1
    assert L.gab200_adam_step_device(1, C.byref(seg), 1.0, 0.999, 1e-15, None, None) == -1
    assert L.gab200_densify_stats(-1, None, None, None, None, None, None, None) == -1
    assert L.gab200_densify_stats(8, None, None, None, None, None, None, None) == -1


def test_capturable_adam_keeps_the_torch_optimizer_surface():
    import gaussianavatars_b200 as g

    p = torch.nn.Parameter(torch.zeros(4, 3))
    sched = g.expon_lr_schedule(lr_init=5e-3, lr_final=5e-5, lr_delay_mult=0.01, max_steps=600_000)
    assert sched == dict(lr_init=5e-3, lr_final=5e-5, lr_delay_steps=0, lr_delay_mult=0.01, max_steps=600_000)
    with pytest.raises(ValueError):
        g.expon_lr_schedule(lr_init=5e-3, lr_final=5e-5, max_steps=0)
    opt = g.Adam([{"params": [p], "lr": 0.0, "name": "xyz", "lr_schedule": sched}], lr=0.0, eps=1e-15, capturable=True)
    assert opt.param_groups[0]["capturable"] is True and opt.state_dict()["param_groups"][0]["lr_schedule"] == sched
    opt.init_state()
    st = opt.state[p]
    assert st["step"].dtype == torch.float32 and st["step"].dim() == 0 and st["step"].device == p.device
    assert float(st["step"]) == 0.0 and not st["exp_avg"].any()
    p.grad = torch.ones_like(p)
    with pytest.raises(RuntimeError, match="no CPU or eager fallback"):
        opt.step()
    # the schedule is evaluated on the device: the host-stepped Adam refuses it instead of ignoring it
    plain = g.Adam([{"params": [p], "lr": 0.0, "lr_schedule": sched}], lr=0.0, eps=1e-15)
    assert plain.param_groups[0]["capturable"] is False
    with pytest.raises(ValueError, match="capturable"):
        plain.step()


def test_graphed_frame_rejects_what_it_cannot_capture():
    import gaussianavatars_b200 as g
    from gaussianavatars_b200.graph import GraphedFrame, pair_with_deferred_reduce

    p = torch.nn.Parameter(torch.zeros(4, 3))
    pc = SimpleNamespace(_xyz=p)
    for opt in (torch.optim.Adam([p]), g.Adam([p])):          # not ours / not capturable
        with pytest.raises(ValueError, match="capturable"):
            GraphedFrame(pc, 8, 8, 1.0, 1.0, torch.zeros(3), optimizer=opt)
    frames = [SimpleNamespace(optimizer=g.Adam([p], capturable=True)), SimpleNamespace(optimizer=None)]
    with pytest.raises(ValueError, match="optimizer"):
        pair_with_deferred_reduce(frames, [None, None])
