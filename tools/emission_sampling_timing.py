"""Cost and gain of emission sampling (rb_area_light::emission_sampling), the measurement behind DESIGN.md section 6 "Emission sampling".

    python tools/emission_sampling_timing.py [--reps 5] [--out result.json]

- tables: the light-table step of rb_scene_update (rb_scene_build_ms "lights", host clock ending in a synchronisation) on the floor-and-lamp
  scene of tests/test_emission_sampling_cpu.py with a 256^2, 1024^2 and 2048^2 window texture, the option off and on, alternating, `reps`
  updates per arm after one warm-up; medians in milliseconds.  The option-on arm rebuilds every emission-sampling table on every update.
- c2: the shadow blocker (bench workload c2: its scene, size, samples and bounces, both edge samplers) with a 256 x 256 x 3 window
  texture on its light, on the general kernels, area against texture strategy: median forward and backward milliseconds of alternating
  rounds (tools/ggx_timing.time_arms).
- efficiency: on the floor-and-lamp scene with the 256^2 window texture, the image variance over `runs` renders and the variance of the
  texel gradient of the window's centre texel per strategy, times the forward (backward) milliseconds: variance x time, lower is better.
- rejection: the fraction of texture-branch samples that the quad's two triangles reject (rb_light_sample_test, 10^6 samples).
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def window(size, ch=3):
    import test_emission_sampling_cpu as es
    return es.window_image(size, size, ch)


def table_times(rb, dev, reps):
    import test_emission_sampling_cpu as es
    out = {}
    for size in (256, 1024, 2048):
        tex = window(size)
        natives = {s: es.native(rb, dev, es.light_scene(dev, tex, sampling=s)) for s in ("area", "texture")}
        scene = natives["area"][0].scene
        times = {s: [] for s in natives}
        for rep in range(reps + 1):
            for s, (c, keep) in natives.items():
                scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False)
                if rep > 0:
                    times[s].append(scene.build_ms()["lights"])
        out["%d^2" % size] = {s: round(statistics.median(t), 3) for s, t in times.items()}
    return out


def with_window(make, sampling, size=256):
    texels = window(size)

    def build(dev):
        from redner_b200 import api
        sc = make(dev)
        for light in sc.area_lights:
            light.emission = api.Texture(texels.to(dev).requires_grad_())
            light.emission_sampling = sampling
        return sc
    return build


def efficiency(rb, dev, runs, spp=16):
    import test_emission_sampling_cpu as es
    from redner_b200 import api
    tex = window(256)
    out = {}
    for s in ("area", "texture"):
        imgs, grads, fwd, bwd = [], [], [], []
        for k in range(runs + 1):
            sc = es.light_scene(dev, tex, sampling=s, res=64)
            t = sc.area_lights[0].emission.texels
            sc.area_lights[0].emission.texels = t.requires_grad_()  # (setting the texels rebuilds the mip pyramid from them)
            args = api.RenderFunction.serialize_scene(sc, spp, 1, device=dev, backend=rb, use_primary_edge_sampling=False,
                                                      use_secondary_edge_sampling=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            img = api.RenderFunction.apply(100 + k, *args)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            img.sum().backward()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if k == 0:
                continue
            fwd.append(1e3 * (t1 - t0))
            bwd.append(1e3 * (t2 - t1))
            imgs.append(img.detach().cpu().numpy())
            g = sc.area_lights[0].emission.texels.grad
            grads.append(float(g[int(0.6 * 256), int(0.3 * 256)].sum()))
        v_img, v_g = float(np.stack(imgs).var(0, ddof=1).sum()), float(np.var(grads, ddof=1))
        out[s] = dict(forward_ms=round(statistics.median(fwd), 2), backward_ms=round(statistics.median(bwd), 2), image_variance=v_img,
                      texel_grad_variance=v_g, image_variance_x_ms=v_img * statistics.median(fwd),
                      texel_grad_variance_x_ms=v_g * statistics.median(bwd))
    return out


def rejection(rb, dev, n=1000000):
    import test_emission_sampling_cpu as es
    c, keep = es.native(rb, dev, es.light_scene(dev, window(256)))
    smp = torch.rand(n, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    smp[:, 0] = 0.125 + 0.875 * smp[:, 0]  # (the texture branch only)
    ints, _, _ = c.scene.light_sample_test(0, smp.to(dev))
    return round(float(ints[:, 2].float().mean()), 4)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "emission_sampling_timing measures on the GPU; there is nothing to measure without one"
    import bench
    from ggx_timing import card, time_arms
    from redner_b200 import _lib
    from redner_b200 import redner as rb
    lib = _lib.load()
    dev = torch.device("cuda:0")
    r = {"gpu": card()}
    r["tables_lights_ms"] = table_times(rb, dev, a.reps)
    wl = bench.WORKLOADS["c2"]
    blocker = lambda d: bench.make_scene(wl, d)  # noqa: E731
    r["c2"] = time_arms(wl["label"], {"area": (with_window(blocker, "area"), lib, True), "texture": (with_window(blocker, "texture"), lib, True)},
                        wl["spp"], wl["mb"], a.reps)
    r["efficiency"] = efficiency(rb, dev, a.runs)
    r["rejection_on_a_quad"] = rejection(rb, dev)
    print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump([r], f, indent=1)


if __name__ == "__main__":
    main()
