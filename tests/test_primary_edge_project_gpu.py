"""GPU suite: the primary-edge pass's per-edge projection (k_prim_edge_project).

Without a lens the default kernel sets sum each edge's screen-space adjoints over its samples and project the sum once per edge; the
deterministic set still projects every sample and sums the results exactly.  The projection is linear in the adjoints, so both must give
the same vertex and camera gradients up to float rounding.  Each case renders the backward pass of one d(loss)/d(image) in both modes,
with primary-edge sampling alone, and compares every gradient buffer (camera included) by relative L2:
- a look-at pinhole on the C2 geometry (the diffuse-only set) and on the single triangle;
- a cam_to_world pinhole on the glossy room (the feature-free set);
- fisheye, panorama, orthographic and a distortion model (the general set);
- an edge that crosses clip_near;
- a thin lens, which keeps the per-sample projection in every set;
- the C2 geometry in two stripes of rb_scene_set_partition (what dist.render_tiles renders on each of two ranks), summed, against the
  unpartitioned image."""
import numpy as np
import pytest
import torch

import exact_records_check as xc
import scenes
import test_lens_cpu as lc
from redner_b200 import api

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _c2w_scene(scene_fn, clip_near=1e-2, lens=None):
    """scene_fn's scene seen through lc.lens_camera: cam_to_world from (0, 0, -5) towards the origin, 45 degrees."""
    def make(dev, resolution):
        sc = scene_fn(dev, resolution[0], None)
        sc.camera = lc.lens_camera(resolution[0], lc._c2w([0.0, 0.0, -5.0], [0.0, 0.0, 0.0]), lc._intrinsic(45.0), lens, clip_near=clip_near)
        return sc
    return make


CASES = {
    "c2_look_at": (lambda dev, resolution: scenes.shadow_blocker(dev, resolution=resolution, grad_all=True), 64, 16),
    "single_triangle_look_at": (lambda dev, resolution: scenes.single_triangle(dev, resolution=resolution), 48, 8),
    "room_cam_to_world": (lambda dev, resolution: lc.room_scene(dev, resolution[0], None), 40, 4),
    "fisheye_room": (scenes.fisheye_room, 40, 4),
    "panorama_room": (scenes.panorama_room, 40, 4),
    "ortho_room": (scenes.ortho_room, 40, 4),
    "distort_room": (scenes.distort_room, 40, 4),
    # the triangle's vertices lie 4.7 - 5.3 in front of the camera: its edges cross the near plane at 4.9
    "glow_clip_near": (_c2w_scene(lc.glow_scene, clip_near=4.9), 48, 8),
    "glow_lens": (_c2w_scene(lc.glow_scene, lens=(torch.tensor([0.2]), torch.tensor([5.0]))), 48, 8),
}


def prepare(rb, dev, name):
    """(unpacked call, d(loss)/d(image)) of a case: primary-edge sampling alone, one bounce, loss = sum(image^2)."""
    make, res, spp = CASES[name]
    sc = make(dev, resolution=(res, res))
    args = api.RenderFunction.serialize_scene(sc, spp, 1, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb, use_primary_edge_sampling=True,
                                              use_secondary_edge_sampling=False)
    c = api.RenderFunction._unpack((3, 3 + 1000003), args)
    c.keep = args
    h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
    img = torch.zeros(h, w, 3, device=dev)
    rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
    return c, (2 * img).contiguous()


def backward(rb, c, d_img, deterministic, parts=1):
    """{position: float64 buffer} of the backward pass, summed over the `parts` stripes of a partition with 4-row stripes."""
    opts = api.RenderFunction.backward_options(c)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic, warn_only=True)
    total = {}
    try:
        for k in range(parts):
            c.scene.set_partition(k, parts, 4)
            g = api.RenderFunction.gradient_buffers(c)
            rb.render(c.scene, opts, rb.float_ptr(0), xc._fp(rb, d_img), g.d_scene, rb.float_ptr(0), rb.float_ptr(0))
            for pos, t in g.grads.items():
                total[pos] = total.get(pos, 0) + t.cpu().numpy().astype(np.float64)
    finally:
        torch.use_deterministic_algorithms(prev)
        c.scene.set_partition(0, 1, 4)
    return total


def assert_close(ref, got, c):
    """Every buffer within TOL relative L2; the camera pose's and some vertices' gradients must be nonzero, so that both are compared."""
    assert ref.keys() == got.keys()
    ca = c.pos.camera_args
    cam = [p for p in (ca.position, ca.look_at, ca.cam_to_world, ca.world_to_cam) if p is not None and p in ref]
    vert = [s.vertices for s in c.pos.shape_args if s.vertices in ref]
    assert any(ref[p].any() for p in cam), "no nonzero camera-pose gradient to compare"
    assert any(ref[p].any() for p in vert), "no nonzero vertex gradient to compare"
    for pos in ref:
        a, b = ref[pos], got[pos]
        n = np.linalg.norm(a)
        err = np.linalg.norm(a - b) / n if n > 0 else np.linalg.norm(b)
        assert err < TOL, (pos, err, n)


@pytest.mark.parametrize("name", sorted(CASES))
def test_per_edge_projection_matches_per_sample(rb, dev, name):
    c, d_img = prepare(rb, dev, name)
    assert_close(backward(rb, c, d_img, True), backward(rb, c, d_img, False), c)


def test_clipped_edge_contributes(rb, dev):
    """Vertex 1 of the glow triangle lies behind the near plane: the two edges that end there are clipped, and its gradient is nonzero."""
    c, d_img = prepare(rb, dev, "glow_clip_near")
    pos = c.pos.shape_args[0].vertices
    for deterministic in (True, False):
        g = backward(rb, c, d_img, deterministic)[pos]
        assert np.abs(g[1]).max() > 0, (deterministic, g)


def test_projection_kernel_runs(rb, dev):
    """The default sets launch k_prim_edge_project without a lens, and only then: one launch more than with a lens.  The deterministic set
    projects every sample itself and launches the same kernels with and without a lens."""
    launches = {}
    for name in ("glow_clip_near", "glow_lens"):
        c, d_img = prepare(rb, dev, name)
        for deterministic in (True, False):
            backward(rb, c, d_img, deterministic)
            launches[name, deterministic] = c.scene.last_stats()[0]
    assert launches["glow_clip_near", False] == launches["glow_lens", False] + 1, launches
    assert launches["glow_clip_near", True] == launches["glow_lens", True], launches


def test_two_stripes_match_one_image(rb, dev):
    c, d_img = prepare(rb, dev, "c2_look_at")
    assert_close(backward(rb, c, d_img, True), backward(rb, c, d_img, False, parts=2), c)
