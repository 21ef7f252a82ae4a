"""GPU suite: the deterministic backward pass (rb_options.deterministic, switched on by torch.use_deterministic_algorithms).

- The exact accumulators through the device scatter (rb_exact_sum_test): ~10^6 contributions of adversarial exponents into a few hot
  and many cold slots equal the exact rational sums rounded to float and double, bit for bit, in two orders; a slot past 2^32
  contributions stays exact.
- Renders: two runs give bitwise-equal gradients (camera and screen-gradient image included), and so do one band and many small
  bands (RB_BAND_BYTES); every gradient is within 1e-5 of the default mode's, and the golden cases pass with their tolerances.
- Callers: rb_render_batch with one shared descriptor equals the sequence of rb_render calls bit for bit; two SceneRenderer Adam
  loops agree bit for bit; the unmodified pyredner on the drop-in gives bitwise-identical numbers in two processes."""
import ctypes as C
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

import parity_utils as pu
import scenes
from redner_b200 import api

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

# (name, case config, kind): gradient cases are rendered with parity_utils.render_case, screen cases with render_screen_gradient
REPEAT_CASES = {
    "glossy_room_both_edges": (dict(pu.CASES["glossy_room_sobol_mb2"], edges=3), "grad"),
    "c2_shadow_blocker_both_edges": (dict(pu.CASES["c2_shadow_blocker_sobol"], edges=3), "grad"),
    "c3_teapot_sobol_mb2": (pu.CASES["c3_teapot_sobol_mb2"], "grad"),
    "env_ball_sobol_mb2": (pu.CASES["env_ball_sobol_mb2"], "grad"),
    "fisheye_room_primary_edges": (pu.CASES["fisheye_room_primary_edges"], "grad"),
    "distort_room_primary_edges": (pu.CASES["distort_room_primary_edges"], "grad"),
    "gbuffer_bwd_glossy_room": (pu.CASES["gbuffer_bwd_glossy_room"], "grad"),
    "screen_gradient_c1": (pu.SCREEN_CASES["screen_gradient_c1"], "screen"),
}


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev)


def render(rb, dev, name):
    """{name: gradient} of one REPEAT_CASES entry (the screen-gradient image under "screen")."""
    cfg, kind = REPEAT_CASES[name]
    if kind == "screen":
        return {"screen": pu.render_screen_gradient(rb, dev, cfg)}
    return pu.render_case(rb, dev, cfg, cfg["seed"])[1]


def assert_bitwise_equal(a, b, what):
    assert a.keys() == b.keys() and a, what
    for k in a:
        x, y = a[k].numpy(), b[k].numpy()
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (what, k, int((x != y).sum()))


# ---------------------------------------------------------------------------------------------------- the exact accumulators
def exact_reference(values, slots, num_slots, repeat=1):
    """Correctly rounded float32 / float64 sums per slot (finite values), from exact integer sums in units of 2^-149."""
    from test_exact_sum_cpu import round_f32
    tot = [0] * num_slots
    for v, s in zip(values.tolist(), slots.tolist()):
        tot[s] += int(Fraction(v) * 2 ** 149)
    f32 = np.array([round_f32(Fraction(t * repeat, 2 ** 149)) for t in tot], dtype=np.float32)
    f64 = np.array([float(Fraction(t * repeat, 2 ** 149)) for t in tot], dtype=np.float64)
    return f32, f64


def exact_sum(rb, dev, values, slots, num_slots, repeat=1):
    from redner_b200 import _lib
    lib = _lib.load()
    v = torch.tensor(values, dtype=torch.float32, device=dev)
    s = torch.tensor(slots, dtype=torch.int32, device=dev)
    o32 = torch.empty(num_slots, dtype=torch.float32, device=dev)
    o64 = torch.empty(num_slots, dtype=torch.float64, device=dev)
    rc = lib.rb_exact_sum_test(C.c_void_p(v.data_ptr()), C.c_void_p(s.data_ptr()), len(values), num_slots, repeat, C.c_void_p(o32.data_ptr()),
                               C.c_void_p(o64.data_ptr()), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert rc == 0, _lib.last_error(lib)
    return o32.cpu().numpy(), o64.cpu().numpy()


def adversarial_values(rng, n):
    """float32 values over the whole exponent range: subnormals, huge values that cancel, and ordinary magnitudes."""
    kind = rng.integers(0, 4, n)
    out = np.empty(n, dtype=np.float32)
    bits = (rng.integers(1, 255, n, dtype=np.uint32) << 23) | rng.integers(0, 1 << 23, n, dtype=np.uint32)
    out[kind == 0] = bits[kind == 0].view(np.float32)                                            # any exponent
    out[kind == 1] = rng.integers(1, 1 << 23, int((kind == 1).sum()), dtype=np.uint32).view(np.float32)  # subnormal
    out[kind == 2] = (rng.uniform(-1, 1, int((kind == 2).sum())) * 2.0 ** rng.integers(100, 127, int((kind == 2).sum()))).astype(np.float32)
    out[kind == 3] = rng.normal(0, 1, int((kind == 3).sum())).astype(np.float32)
    out *= np.where(rng.random(n) < 0.5, -1, 1).astype(np.float32)
    return out


def test_exact_sums_through_the_device_scatter(rb, dev):
    rng = np.random.default_rng(3)
    n, num_slots = 1 << 20, 4096
    values = adversarial_values(rng, n)
    # 4 hot slots take half of the contributions (neighbouring lanes hit them together), the rest is spread over the cold ones
    slots = np.where(rng.random(n) < 0.5, rng.integers(0, 4, n), rng.integers(4, num_slots, n)).astype(np.int32)
    big = np.float32(3.0e38)
    values[:6] = [big, -big, big, -big, np.float32(1e-45), np.float32(-2.0)]  # cancellation of huge values around small ones
    slots[:6] = 0
    ref32, ref64 = exact_reference(values, slots, num_slots)
    a32, a64 = exact_sum(rb, dev, values, slots, num_slots)
    perm = rng.permutation(n)
    b32, b64 = exact_sum(rb, dev, values[perm], slots[perm], num_slots)
    assert a32.tobytes() == b32.tobytes() and a64.tobytes() == b64.tobytes()
    assert a32.tobytes() == ref32.tobytes(), int((a32.view(np.uint32) != ref32.view(np.uint32)).sum())
    assert a64.tobytes() == ref64.tobytes(), int((a64.view(np.uint64) != ref64.view(np.uint64)).sum())


def limb_chunk(v):
    """(limb, low chunk) of a positive float32 as rb_exact.cuh's exact_term splits it: significand m shifted by (biased exponent - 1) & 31
    into limb (biased exponent - 1) >> 5."""
    u = int(np.float32(v).view(np.uint32))
    e, m = (u >> 23) & 0xFF, (u & 0x7FFFFF) | (0x800000 if (u >> 23) & 0xFF else 0)
    p = e - 1 if e else 0
    return p >> 5, (m << (p & 31)) & 0xFFFFFFFF


def test_exact_sum_past_two_to_the_32_contributions(rb, dev):
    """One slot takes 3 * repeat > 2^32 contributions of three floats whose significands are (almost) all ones and sit 8 bits up in one
    limb: every contribution adds nearly 2^32 to that limb, so without the carry normalisation between chunks of RB_EXACT_MAX_ADDS
    contributions the limb would pass 2^63 (the total passes 2^64) and the sum would come out wrong."""
    values = np.array([np.float32((0xFFFFFF - k) * 2.0 ** -13) for k in range(3)], dtype=np.float32)  # m = 0xFFFFFF - k, p = 136
    slots = np.zeros(3, dtype=np.int32)
    repeat = (1 << 32) // 3 + 12345
    chunks = [limb_chunk(v) for v in values]
    assert len({limb for limb, _ in chunks}) == 1 and all(c >= 0xFFFFFD00 for _, c in chunks)
    assert repeat * sum(c for _, c in chunks) > 1 << 64  # the unnormalised limb would overflow
    ref32, ref64 = exact_reference(values, slots, 2, repeat)
    a32, a64 = exact_sum(rb, dev, values, slots, 2, repeat)
    assert a32.tobytes() == ref32.tobytes() and a64.tobytes() == ref64.tobytes(), (a32, ref32, a64, ref64)


# ---------------------------------------------------------------------------------------------------- renders
@pytest.mark.parametrize("name", list(REPEAT_CASES))
def test_two_runs_are_bitwise_equal(rb, dev, name, deterministic):
    assert_bitwise_equal(render(rb, dev, name), render(rb, dev, name), name)


@pytest.mark.parametrize("name", list(REPEAT_CASES))
def test_band_size_does_not_change_a_bit(rb, dev, name, deterministic, monkeypatch):
    one = render(rb, dev, name)
    monkeypatch.setenv("RB_BAND_BYTES", str(1 << 20))
    assert_bitwise_equal(one, render(rb, dev, name), name)


@pytest.mark.parametrize("name", list(REPEAT_CASES))
def test_deterministic_mode_gives_the_default_answer(rb, dev, name):
    default = render(rb, dev, name)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        det = render(rb, dev, name)
    finally:
        torch.use_deterministic_algorithms(False)
    assert default.keys() == det.keys()
    for k in default:
        assert pu.rel_l2(det[k].numpy(), default[k].numpy()) < 1e-5, (name, k, pu.rel_l2(det[k].numpy(), default[k].numpy()))


@pytest.mark.parametrize("name", list(pu.CASES))
def test_golden_case_in_deterministic_mode(rb, dev, name, deterministic):
    cfg = pu.CASES[name]
    img, grads = pu.render_case(rb, dev, cfg, cfg["seed"])
    pu.assert_matches_golden(name, img.numpy(), grads)


# ---------------------------------------------------------------------------------------------------- callers
def _batch_views(dev):
    """Three views of the glossy room (shared shapes / materials / lights), as in the batch test of the emulator."""
    views = [scenes.glossy_room(dev, resolution=(32, 32)) for _ in range(3)]
    cams = [([0.3, 1.4, -4.5], [0.0, 0.6, 0.0]), ([1.2, 1.1, -4.0], [0.1, 0.5, 0.1]), ([-0.8, 1.8, -4.2], [0.0, 0.7, 0.2])]
    for v, (p, l) in zip(views, cams):
        v.camera = api.Camera(position=torch.tensor(p), look_at=torch.tensor(l), up=torch.tensor([0.0, 1.0, 0.0]), fov=torch.tensor([40.0]),
                              clip_near=1e-2, resolution=(32, 32))
        v.shapes, v.materials, v.area_lights = views[0].shapes, views[0].materials, views[0].area_lights
    return views


def test_render_batch_equals_the_sequence_of_renders(rb, dev, deterministic):
    """rb_render_batch with one descriptor for every view == rb_scene_set_camera + rb_render per view into one descriptor, bit for bit."""
    from redner_b200 import _lib as L
    views = _batch_views(dev)
    kw = dict(sampler_type=rb.SamplerType.sobol, device=dev, backend=rb, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    ctxs, scene = [], None
    for k, v in enumerate(views):
        c = api.RenderFunction._unpack((20 + k, 40 + k), api.RenderFunction.serialize_scene(v, 4, 2, **kw), scene=scene)
        scene = c.scene
        ctxs.append(c)
    d_imgs = [torch.rand(32, 32, 3, device=dev) for _ in views]

    def descriptor(c):
        """A gradient descriptor of the scene with zeroed buffers (the layout RenderFunction.backward makes) and the buffers."""
        keep = []

        def zeros(*shape):
            keep.append(torch.zeros(*shape, device=dev))
            return keep[-1]
        return api.RenderFunction.gradient_buffers(c, zeros).d_scene, keep

    def options(c):
        o = L.rb_options(seed=c.seed[1], num_samples=c.num_samples[1], max_bounces=c.options.max_bounces, sampler_type=int(c.options.sampler_type),
                         sample_pixel_center=int(c.options.sample_pixel_center), deterministic=1)
        o.num_channels, o.channels = 1, C.cast(_RADIANCE, C.POINTER(C.c_int))
        return o
    _RADIANCE = (C.c_int * 1)(int(rb.channels.radiance))
    lib = L.load()
    (a, bufs_a), (b, bufs_b) = descriptor(ctxs[0]), descriptor(ctxs[0])
    cams = (L.rb_camera * 3)(*[c.camera._c for c in ctxs])
    opts = (L.rb_options * 3)(*[options(c) for c in ctxs])
    d_img_ptrs = (C.c_void_p * 3)(*[t.data_ptr() for t in d_imgs])
    descs = (C.POINTER(L.rb_dscene_desc) * 3)(*[C.pointer(a._c)] * 3)
    torch.cuda.synchronize()
    assert lib.rb_render_batch(scene._handle, 3, cams, opts, None, d_img_ptrs, descs, None) == 0, L.last_error(lib)
    for k, c in enumerate(ctxs):
        assert lib.rb_scene_set_camera(scene._handle, C.byref(c.camera._c)) == 0
        assert lib.rb_render(scene._handle, C.byref(opts[k]), None, C.c_void_p(d_imgs[k].data_ptr()), C.byref(b._c), None, None) == 0, L.last_error(lib)
    torch.cuda.synchronize()
    assert len(bufs_a) == len(bufs_b) > 0 and sum(bool((t != 0).any()) for t in bufs_a) >= 5
    for x, y in zip(bufs_a, bufs_b):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()


def test_scene_renderer_adam_loops_are_bitwise_equal(rb, dev, deterministic):
    from test_scene_update_cpu import adam_loop
    made = []

    def pick(sc):  # the sphere's vertices, a light's intensity and the camera position
        return [sc.shapes[3].vertices, sc.area_lights[0].intensity, sc.camera.position]

    def make():  # (grad=False: adam_loop marks the picked tensors; the textures' mip pyramids are built without a graph)
        made.append(scenes.glossy_room(dev, resolution=(32, 32), grad=False))
        return made[-1]
    kw = dict(sampler_type=rb.SamplerType.sobol, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    runs = [adam_loop(dev, make, pick, 5, 4, 2, True, **kw) for _ in range(2)]
    (ia, ga), (ib, gb) = runs
    for x, y in zip(ia, ib):
        assert torch.equal(x, y)
    for x, y in zip(ga, gb):
        for p, q in zip(x, y):
            assert p.numpy().tobytes() == q.numpy().tobytes()
    for p, q in zip(pick(made[0]), pick(made[1])):
        assert p.detach().cpu().numpy().tobytes() == q.detach().cpu().numpy().tobytes()


def test_unmodified_pyredner_under_deterministic_algorithms(tmp_path):
    if not os.path.isdir(os.path.join(REF_DIR, "pyredner")):
        pytest.skip("oracle/_ref/pyredner not built (oracle/build_ref.sh copies it from a checkout of the reference)")
    runner = ("import runpy, sys, torch; torch.use_deterministic_algorithms(True, warn_only=True); sys.argv = sys.argv[1:]; "
              "runpy.run_path(sys.argv[0], run_name='__main__')")
    outs = []
    for k in range(2):
        path = str(tmp_path / ("run%d.npz" % k))
        r = subprocess.run([sys.executable, "-W", "ignore", "-c", runner, os.path.join(ROOT, "tests", "dropin_script.py"), "cuda", path, REF_DIR, "cuda"],
                           capture_output=True, text=True, timeout=900, env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"))
        assert r.returncode == 0 and "DONE" in r.stdout, r.stderr[-3000:]
        outs.append(dict(np.load(path)))
    assert set(outs[0]) == set(outs[1])
    for k in outs[0]:
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), k
