"""Checks of the exact records (rb_exact_record_count / rb_render_exact / rb_exact_round), shared by tests/test_exact_records_cpu.py
(host build of the device headers) and tests/test_exact_records_gpu.py (the CUDA library).

partition_sums: a deterministic render split into the stripes of rb_scene_set_partition, each stripe's records summed as int64 and
rounded once, must equal the unpartitioned deterministic rb_render bit for bit in every buffer.  Every stripe's gradient descriptor is
carved out of one tensor in an order of its own, so the buffers of two stripes lie in different address orders: a record numbering that
followed addresses would add unrelated floats together.

crafted_records: hand-made records on a tiny scene: non-finite counts, carries and a zero sum."""
from fractions import Fraction

import numpy as np
import torch

import parity_utils as pu
import scenes
from redner_b200 import _lib as L, api

WORDS = L.RB_EXACT_RECORD_WORDS
LIMBS = 10
CAM_RECORDS = 58  # RB_CAM_ACC: one record per camera gradient scalar comes first


def _deterministic(fn, *args):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        return fn(*args)
    finally:
        torch.use_deterministic_algorithms(prev)


def prepare(rb, dev, cfg, kind):
    """(unpacked call, d_image, with_screen) of one case: a gradient case's d(loss)/d(image) as parity_utils.render_case forms it, or the
    all-ones image of a screen-gradient case."""
    res = pu._res(cfg)
    st = rb.SamplerType.sobol if cfg["sampler"] == "sobol" else rb.SamplerType.independent
    sc = scenes.SCENES[cfg["scene"]](dev, resolution=res, grad=kind != "screen")
    chans = [getattr(rb.channels, ch) for ch in cfg["channels"]] if "channels" in cfg else None
    args = api.RenderFunction.serialize_scene(sc, cfg["spp"], cfg["mb"], channels=chans, sampler_type=st, device=dev, backend=rb,
                                              use_primary_edge_sampling=bool(cfg["edges"] & 1), use_secondary_edge_sampling=bool(cfg["edges"] & 2))
    if kind == "screen":  # as api.visualize_screen_gradient
        c = api.RenderFunction._unpack((cfg["seed"], cfg["seed"]), args)
        c.num_samples = (c.num_samples[0], c.num_samples[0])
    else:
        c = api.RenderFunction._unpack((cfg["seed"], cfg["seed"] + 1000003), args)
    c.keep = args
    nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
    h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
    if kind == "screen":
        return c, torch.ones(h, w, nch, device=dev), True
    img = torch.zeros(h, w, nch, device=dev)
    rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
    wt = torch.linspace(0.5, 1.5, nch, device=dev) if chans is not None else 1.0
    return c, (2 * img * wt * wt).contiguous(), False


def buffers(c, g, screen):
    """Every gradient buffer of gradient_buffers(c) (the camera's included) and the screen-gradient image, in a fixed order."""
    return list(g.grads.values()) + ([screen] if screen is not None else [])


def carve(c, with_screen, reverse):
    """(gradient buffers, screen image) whose tensors are slices of ONE zeroed tensor, taken from its start or, with `reverse`, from its end:
    the two orders put the same buffers in opposite address orders."""
    dev = c.device
    h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
    probe = api.RenderFunction.gradient_buffers(c)
    total = sum(t.numel() for t in buffers(c, probe, None)) + (2 * h * w if with_screen else 0)
    pool = torch.zeros(total, device=dev)
    off = [0]

    def zeros(*shape):
        n = int(np.prod(shape)) if shape else 1
        lo = total - off[0] - n if reverse else off[0]
        off[0] += n
        return pool[lo:lo + n].view(*shape)
    g = api.RenderFunction.gradient_buffers(c, zeros)
    screen = zeros(h, w, 2) if with_screen else None
    return g, screen


def fresh(c, with_screen):
    h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
    return api.RenderFunction.gradient_buffers(c), (torch.zeros(h, w, 2, device=c.device) if with_screen else None)


def _fp(rb, t):
    return api._ptr(rb, t)


def reference(rb, c, d_img, with_screen):
    """Buffers of the unpartitioned deterministic rb_render."""
    c.scene.set_partition(0, 1, 4)
    g, screen = fresh(c, with_screen)
    opts = api.RenderFunction.backward_options(c)
    _deterministic(rb.render, c.scene, opts, rb.float_ptr(0), _fp(rb, d_img), g.d_scene, _fp(rb, screen), rb.float_ptr(0))
    return [t.cpu().numpy().copy() for t in buffers(c, g, screen)]


def partitioned(rb, c, d_img, with_screen, num_parts, rows_per_stripe):
    """Buffers after rounding the int64 sum of the records of every stripe of a num_parts partition."""
    opts = api.RenderFunction.backward_options(c)
    total = None
    for k in range(num_parts):
        c.scene.set_partition(k, num_parts, rows_per_stripe)
        g, screen = carve(c, with_screen, reverse=k % 2 == 1)
        rec = rb.render_exact(c.scene, opts, _fp(rb, d_img), g.d_scene, _fp(rb, screen))
        assert all(not bool(t.any()) for t in buffers(c, g, screen)), "rb_render_exact wrote a gradient buffer"
        rec = rec.cpu().numpy()
        total = rec if total is None else total + rec
    c.scene.set_partition(0, 1, 4)
    g, screen = fresh(c, with_screen)
    rb.round_exact(c.scene, opts, g.d_scene, _fp(rb, screen), torch.from_numpy(total).to(c.device))
    return [t.cpu().numpy().copy() for t in buffers(c, g, screen)]


def assert_bitwise(ref, got, what):
    assert len(ref) == len(got) and sum(int(np.count_nonzero(r)) for r in ref) > 0, what
    for i, (a, b) in enumerate(zip(ref, got)):
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), (what, i, a.shape, int((a.view(np.uint32) != b.view(np.uint32)).sum()))


def partition_sums(rb, dev, cfg, kind, parts, rows=(1, 4)):
    c, d_img, with_screen = prepare(rb, dev, cfg, kind)
    ref = reference(rb, c, d_img, with_screen)
    for n in parts:
        for rps in rows:
            assert_bitwise(ref, partitioned(rb, c, d_img, with_screen, n, rps), (n, rps))


# ---------------------------------------------------------------------------------------------------- crafted records
def normalise(limbs):
    """exact_normalise of rb_exact.cuh on Python integers: limbs 0..8 into [0, 2^32), the rest into limb 9."""
    a = list(limbs)
    for k in range(LIMBS - 1):
        low = a[k] & 0xFFFFFFFF
        a[k + 1] += (a[k] - low) >> 32
        a[k] = low
    return a


def record_of(value):
    """The normalised record of one finite float32 contribution (or a float32 non-finite value: its count)."""
    r = [0] * WORDS
    v = np.float32(value)
    if np.isnan(v):
        r[LIMBS + 2] = 1
    elif np.isinf(v):
        r[LIMBS + (0 if v > 0 else 1)] = 1
    else:
        q = int(Fraction(float(v)) * 2 ** 149)  # exact: every float32 is an integer multiple of 2^-149
        limbs = [0] * LIMBS
        limbs[LIMBS - 1] = q >> (32 * (LIMBS - 1))  # (floor: the carries of normalise do the rest)
        rest = q - (limbs[LIMBS - 1] << (32 * (LIMBS - 1)))
        for k in range(LIMBS - 1):
            limbs[k] = (rest >> (32 * k)) & 0xFFFFFFFF
        r[:LIMBS] = normalise(limbs)
    return r


def crafted_records(rb, dev):
    """One element (the first float of the triangle's vertex gradient) rounded from hand-made sums of records."""
    cfg = dict(pu.CASES["c1_single_triangle_sobol"], res=4)
    c, d_img, _ = prepare(rb, dev, cfg, "grad")
    opts = api.RenderFunction.backward_options(c)
    g, _ = fresh(c, False)
    count, fingerprint = rb.exact_record_count(c.scene, opts, g.d_scene)
    assert count == CAM_RECORDS + sum(t.numel() for t in buffers(c, g, None)[sum(t is not None for t in g.camera):])
    target = CAM_RECORDS  # record of shape 0's vertices[0]

    def rounded(sides, init=0.0):
        total = np.zeros((count, WORDS), dtype=np.int64)
        for side in sides:
            total[target] += np.array(side, dtype=np.int64)
        g, _ = fresh(c, False)
        g.shapes[0][0].view(-1)[0] = init
        rb.round_exact(c.scene, opts, g.d_scene, None, torch.from_numpy(total).to(dev))
        return np.float32(g.shapes[0][0].view(-1)[0].item())

    inf = np.float32(np.inf)
    r = rounded([record_of(inf), record_of(inf)])
    assert np.isposinf(r), r  # (OR-ed flag bits would have summed to the -inf bit)
    assert np.isnan(rounded([record_of(inf), record_of(-inf)]))
    assert np.isnan(rounded([record_of(np.float32(np.nan)), record_of(np.float32(1.5))]))
    # carries: three normalised records whose limb 4 is 2^32 - 1 (limb 4 weighs 2^(128 - 149))
    side = [0] * WORDS
    side[4] = (1 << 32) - 1
    r = rounded([side, side, side])
    expect = np.float32(float(3 * ((1 << 32) - 1)) * 2.0 ** -21)  # (exact in a double, so one rounding)
    assert r.tobytes() == expect.tobytes(), (r, expect)
    # +x and -x: raw limbs that are not zero, a value that is; the element is not touched (-0.0 stays -0.0, a rounded zero would be +0.0)
    a, b = record_of(np.float32(1.0)), record_of(np.float32(-1.0))
    assert any(x + y for x, y in zip(a, b))
    r = rounded([a, b], init=-0.0)
    assert r.tobytes() == np.float32(-0.0).tobytes(), r
    # an ordinary value survives
    assert rounded([record_of(np.float32(0.1)), record_of(np.float32(0.2))]) == np.float32(Fraction(np.float32(0.1).item()) + Fraction(np.float32(0.2).item()))
    return count, fingerprint


def refusals(rb, dev):
    """Wrong count and NULL records are refused by the C ABI and by the Python layer, with messages."""
    import ctypes as C
    cfg = dict(pu.CASES["c1_single_triangle_sobol"], res=4)
    c, d_img, _ = prepare(rb, dev, cfg, "grad")
    opts = api.RenderFunction.backward_options(c)
    g, _ = fresh(c, False)
    count, _ = rb.exact_record_count(c.scene, opts, g.d_scene)
    lib = c.scene._lib
    o, _chs = rb._options(opts, True)
    rec = torch.zeros((count + 1, WORDS), dtype=torch.int64, device=dev)
    p = C.c_void_p(rec.data_ptr())
    for fn, args in (("rb_render_exact", (C.c_void_p(d_img.data_ptr()), C.byref(g.d_scene._c), None)), ("rb_exact_round", (C.byref(g.d_scene._c), None))):
        assert getattr(lib, fn)(c.scene._handle, C.byref(o), *args, p, count + 1, None) == 1
        assert "count is %d but the descriptor has %d records" % (count + 1, count) in L.last_error(lib), L.last_error(lib)
        assert getattr(lib, fn)(c.scene._handle, C.byref(o), *args, None, count, None) == 1
        assert "records" in L.last_error(lib) and "null" in L.last_error(lib), L.last_error(lib)
    for call in (lambda: rb.render_exact(c.scene, opts, _fp(rb, d_img), g.d_scene, None, rec),
                 lambda: rb.round_exact(c.scene, opts, g.d_scene, None, rec),
                 lambda: rb.round_exact(c.scene, opts, g.d_scene, None, None)):
        try:
            call()
        except RuntimeError as e:
            assert "records" in str(e), e
        else:
            raise AssertionError("not refused")
    # overlapping gradient buffers have no record position: shape 0's uv gradient pointed at its vertex gradient
    g.d_scene._shapes[0].uvs = g.d_scene._shapes[0].vertices
    for call in (lambda: rb.exact_record_count(c.scene, opts, g.d_scene), lambda: rb.render_exact(c.scene, opts, _fp(rb, d_img), g.d_scene)):
        try:
            call()
        except RuntimeError as e:
            assert "overlap" in str(e), e
        else:
            raise AssertionError("overlapping buffers not refused")
