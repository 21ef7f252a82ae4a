"""Cost of the thin-lens camera (rb_camera::lens_radius), the measurements behind DESIGN.md section 6 "thin-lens camera".

    python tools/lens_timing.py [--reps 5] [--out result.json]

The teapot (bench workload c3: same scene, size, samples and bounces, Sobol, both edge samplers, loss = sum(img^2)) three ways:
    pinhole        no lens, the kernels rb_render picks (the lean set)
    pinhole-gen    no lens with RB_NO_LEAN=1 (the general set, which carries the lens code)
    lens           lens_radius 2 % of the distance to the look-at point, focused on it (the general set)
Arms run one after the other, alternating, `reps` times each after one warm-up round; per arm the median milliseconds of the forward call
(scene build included) and of the backward call (host clock, both end in a synchronisation) and the library's stage times of the last
backward pass are printed as one JSON line.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def with_lens(make, frac):
    def build(dev):
        sc = make(dev)
        cam = sc.camera
        d = float(torch.linalg.norm(cam.look_at.detach().cpu() - cam.position.detach().cpu()))
        cam.lens_radius, cam.focus_distance = torch.tensor([frac * d]), torch.tensor([d])
        return sc
    return build


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "lens_timing measures on the GPU; there is nothing to measure without one"
    import bench
    from ggx_timing import card, time_arms
    from redner_b200 import _lib
    lib = _lib.load()
    wl = bench.WORKLOADS["c3"]
    teapot = lambda dev: bench.make_scene(wl, dev)  # noqa: E731
    r = time_arms(wl["label"], {"pinhole": (teapot, lib, False), "pinhole-gen": (teapot, lib, True), "lens": (with_lens(teapot, 0.02), lib, False)},
                  wl["spp"], wl["mb"], a.reps)
    r["gpu"] = card()
    print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump([r], f, indent=1)


if __name__ == "__main__":
    main()
