"""Cost of an emission texture on an area light (rb_area_light::emission), the measurement behind DESIGN.md section 6 "Emission textures".

    python tools/emission_timing.py [--reps 5] [--out result.json]

The shadow blocker (bench workload c2: same scene, size, samples and bounces, Sobol, both edge samplers, loss = sum(img^2)) two ways, both on
the general kernels (RB_NO_LEAN=1, the set that carries the emission code):
    plain      the scene's light as it is
    textured   the same light with a 256 x 256 x 3 emission texture (values in [0.5, 1.5], requiring grad)
Arms run one after the other, alternating, `reps` times each after one warm-up round; per arm the median milliseconds of the forward call
(scene build included) and of the backward call (host clock, both end in a synchronisation) and the library's stage times of the last
backward pass are printed as one JSON line.  `pyramid_ms` is the part of the textured arm's backward call that runs in PyTorch, timed on
its own: autograd carrying one gradient per level of api.Texture's mip pyramid back to the texels (median milliseconds of `reps` rounds
after a warm-up, host clock ending in a synchronisation).  The card's name and power limit are read in the
same run."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def with_emission(make, size=256):
    g = torch.Generator().manual_seed(1)
    texels = 0.5 + torch.rand(size, size, 3, generator=g)

    def build(dev):
        from redner_b200 import api
        sc = make(dev)
        for light in sc.area_lights:
            light.emission = api.Texture(texels.to(dev).requires_grad_())
        return sc
    return build


def pyramid_ms(dev, reps, size=256):
    from redner_b200 import api
    g = torch.Generator().manual_seed(1)
    texels = (0.5 + torch.rand(size, size, 3, generator=g)).to(dev)
    times = []
    for rep in range(reps + 1):
        tex = api.Texture(texels.clone().requires_grad_())  # (built with the scene, before the timed calls)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.autograd.backward(tex.mipmap, [torch.ones_like(m) for m in tex.mipmap])
        torch.cuda.synchronize()
        if rep > 0:
            times.append(1e3 * (time.perf_counter() - t0))
    return round(statistics.median(times), 2)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "emission_timing measures on the GPU; there is nothing to measure without one"
    import bench
    from ggx_timing import card, time_arms
    from redner_b200 import _lib
    lib = _lib.load()
    wl = bench.WORKLOADS["c2"]
    blocker = lambda dev: bench.make_scene(wl, dev)  # noqa: E731
    r = time_arms(wl["label"], {"plain": (blocker, lib, True), "textured": (with_emission(blocker), lib, True)}, wl["spp"], wl["mb"], a.reps)
    r["pyramid_ms"] = pyramid_ms(torch.device("cuda:0"), a.reps)
    r["gpu"] = card()
    print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump([r], f, indent=1)


if __name__ == "__main__":
    main()
