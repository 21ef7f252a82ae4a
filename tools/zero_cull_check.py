#!/usr/bin/env python
"""C2 at bench size (512 x 512 x 64 spp, max_bounces 1, both edge samplers, loss sum(img^2), bench.py's seeds) in deterministic mode, with and
without RB_NO_ZERO_CULL=1: every gradient must be bit-identical.  Also reports how many samples the backward pass skipped (pixels whose
adjoint is exactly zero, times spp) against the primary hits it traces without the skip, and the stage times of both runs.

    python tools/zero_cull_check.py [resolution] [spp]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import scenes  # noqa: E402
from redner_b200 import api  # noqa: E402
from redner_b200 import redner as rb  # noqa: E402

res = int(sys.argv[1]) if len(sys.argv) > 1 else 512
spp = int(sys.argv[2]) if len(sys.argv) > 2 else 64
dev = torch.device("cuda:0")
torch.use_deterministic_algorithms(True, warn_only=True)


def run(skip):
    if skip:
        os.environ.pop("RB_NO_ZERO_CULL", None)
    else:
        os.environ["RB_NO_ZERO_CULL"] = "1"
    args = api.RenderFunction.serialize_scene(scenes.shadow_blocker(dev, resolution=(res, res)), spp, 1, sampler_type=rb.SamplerType.sobol, device=dev,
                                              backend=rb)
    c = api.RenderFunction._unpack((1, 1000004), args)
    img = api._render(c)
    d = (2 * img).contiguous()
    grads = [g.detach().cpu().numpy() for g in api._backward(c, d) if isinstance(g, torch.Tensor)]
    stages, vertices, hits = c.scene.last_stage_stats()
    return img.cpu().numpy(), d, grads, dict(stages_ms=stages, path_vertices=vertices, primary_hits=hits)


run(True)  # (warm-up: module loading and the first growth of the scratch land here, not in the stage times below)
img_s, d, g_s, st_s = run(True)
img_f, _, g_f, st_f = run(False)
os.environ.pop("RB_NO_ZERO_CULL", None)
zero_px = int((d == 0).all(-1).sum())
same = [a.tobytes() == b.tobytes() for a, b in zip(g_s, g_f)]
out = dict(device=torch.cuda.get_device_name(0), res=res, spp=spp, images_identical=img_s.tobytes() == img_f.tobytes(), gradients=len(same),
           gradients_bit_identical=sum(same), zero_pixels=zero_px, zero_pixel_fraction=zero_px / (res * res), skipped_samples=zero_px * spp,
           primary_hits_without_skip=st_f["primary_hits"], primary_hits_with_skip=st_s["primary_hits"],
           skipped_share_of_hits=(st_f["primary_hits"] - st_s["primary_hits"]) / max(st_f["primary_hits"], 1),
           with_skip=st_s, without_skip=st_f)
print(json.dumps(out, default=float))
assert all(same) and out["images_identical"], "gradients differ with and without the skip"
