"""CPU suite: the deterministic backward pass on the host build of the device headers (tools/cpu_emu).

- Under torch.use_deterministic_algorithms(True), redner.render sets rb_options.deterministic, and nothing else does.
- In that mode the emulator's scatter and camera accumulation go through the exact accumulators of rb_exact.cuh with the library's
  layout (rb_exact_layout.hpp): golden cases, a screen-gradient image included, pass their golden tolerances and match the default
  emulator render within 5e-5.  (Not closer: the default emulator adds the contributions of a whole render one by one into a float,
  and where every sample reaches the same element -- C1's triangle, a constant specular reflectance -- that running sum drifts from
  the exact one by up to ~1e-5; the reference's float gradient buffers drift the same way.)
The device side (bitwise repeatability, band invariance) is tests/test_deterministic_gpu.py.

Run as a script (`python tests/test_deterministic_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

GOLDEN = ["c1_single_triangle_sobol", "glossy_room_sobol_mb2", "env_ball_sobol_mb2", "gbuffer_bwd_glossy_room"]


def deterministic_render(fn, *args):
    import torch
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        return fn(*args)
    finally:
        torch.use_deterministic_algorithms(prev)


def check_golden(rb, dev):
    import parity_utils as pu
    import torch
    for name in GOLDEN:
        cfg = pu.CASES[name]
        img, grads = pu.render_case(rb, dev, cfg, cfg["seed"])
        img_d, grads_d = deterministic_render(pu.render_case, rb, dev, cfg, cfg["seed"])
        assert torch.equal(img, img_d), name
        assert grads.keys() == grads_d.keys() and grads, name
        for k in grads:
            assert pu.rel_l2(grads_d[k].numpy(), grads[k].numpy()) < 5e-5, (name, k, pu.rel_l2(grads_d[k].numpy(), grads[k].numpy()))
        pu.assert_matches_golden(name, img_d.numpy(), grads_d)
    cfg = pu.SCREEN_CASES["screen_gradient_c1"]
    a = pu.render_screen_gradient(rb, dev, cfg).numpy()
    b = deterministic_render(pu.render_screen_gradient, rb, dev, cfg).numpy()
    assert pu.rel_l2(b, a) < 5e-5, pu.rel_l2(b, a)


def check_flag(rb, dev):
    """The options rb_render receives: deterministic = 1 exactly when PyTorch's switch is on, for the forward and the backward call."""
    import parity_utils as pu
    from redner_b200 import _lib
    lib = _lib._lib
    real = lib.rb_render
    seen = []

    def spy(handle, opt, *rest):
        seen.append(opt._obj.deterministic)
        return real(handle, opt, *rest)
    lib.rb_render = spy
    try:
        cfg = dict(pu.CASES["c1_single_triangle_sobol"], res=16)
        pu.render_case(rb, dev, cfg, 1)
        assert seen == [0, 0], seen
        seen.clear()
        deterministic_render(pu.render_case, rb, dev, cfg, 1)
        assert seen == [1, 1], seen
    finally:
        lib.rb_render = real


def _run(checks):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_deterministic_algorithms_switch_the_library_mode():
    _run(["flag"])


def test_exact_accumulation_in_a_render_matches_the_default_render():
    _run(["golden"])


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    checks = {"golden": check_golden, "flag": check_flag}
    for name in names:
        checks[name](rb, torch.device("cpu"))
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
