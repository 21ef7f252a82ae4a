"""Multi-GPU rendering: one process per GPU (torch.distributed), no reference counterpart (the reference only lets the
caller pick a device: pyredner/device.py:26-33, src/pathtracer.cpp:184-192).

Two ways to use N GPUs (SURVEY.md section 8e):

* `render_tiles`  -- ONE image, split into round-robin stripes of viewport rows (rb_scene_set_partition).  Samplers stay
  seeded by the full-viewport pixel index, so the union over ranks equals the single-GPU image bit for bit; primary-edge
  samples are sharded by sample index.  One collective at the end of each pass: all_reduce(sum) of the framebuffer
  (ranks hold zeros outside their stripes) after forward, and of the packed gradient buffers after backward.  Under
  torch.use_deterministic_algorithms(True) the backward pass exchanges the exact accumulators instead (redner.render_exact, an integer
  all_reduce, redner.round_exact), so every gradient is the one-GPU deterministic gradient bit for bit, for any number of ranks.
* `render_poses` -- a batch of independent scenes / camera poses (BASELINE config 5): rank r renders poses r, r+N, ...;
  the only exchange is the all_reduce of the parameter gradients (the usual data-parallel multi-view optimisation).

Both functions take the process group as argument, so the host logic is testable on CPU with the gloo backend.
"""
from typing import Callable, List, Sequence

import torch
import torch.distributed as dist

from . import api


def pack(tensors: Sequence[torch.Tensor]) -> torch.Tensor:
    """Flatten a list of tensors into one contiguous buffer (one collective instead of one per tensor)."""
    return torch.cat([t.reshape(-1) for t in tensors]) if len(tensors) else torch.zeros(0)


def unpack(flat: torch.Tensor, like: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    out, o = [], 0
    for t in like:
        n = t.numel()
        out.append(flat[o:o + n].reshape(t.shape))
        o += n
    return out


def all_reduce_packed(tensors: Sequence[torch.Tensor], group=None) -> List[torch.Tensor]:
    """Sum a list of same-device tensors across ranks with a single all_reduce."""
    if len(tensors) == 0:
        return []
    flat = pack(tensors)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return unpack(flat, tensors)


def owned_rows(height: int, rank: int, world: int, rows_per_stripe: int = 4) -> List[int]:
    """Rows of the viewport rendered by `rank` (mirrors count_owned_rows / owned_row_to_row in csrc/rb_render.cuh)."""
    return [r for r in range(height) if (r // rows_per_stripe) % world == rank]


def check_records_agree(count: int, fingerprint: int, device, group=None):
    """Raises on every rank unless all ranks of `group` have the same record count and layout fingerprint (one all_gather)."""
    mine = torch.tensor([count, fingerprint - (1 << 64) if fingerprint >= 1 << 63 else fingerprint], dtype=torch.int64, device=device)
    every = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(every, mine, group=group)
    every = [tuple(int(v) for v in t.cpu()) for t in every]
    if any(e != every[0] for e in every):
        raise RuntimeError("redner_b200.dist: the ranks' gradient records do not line up (count, fingerprint per rank: %s); every rank must "
                           "render the same scene structure" % every)


def _exact_backward(c, grad_img, group):
    """Deterministic backward pass of one sharded image: each rank's exact accumulators as records, one integer all_reduce, one rounding.
    Integer sums do not depend on the order of the ranks or of NCCL's algorithm, so the gradients are the one-GPU deterministic ones."""
    rb = c.backend
    g = api.RenderFunction.gradient_buffers(c)
    opts = api.RenderFunction.backward_options(c)
    count, fingerprint = rb.exact_record_count(c.scene, opts, g.d_scene)
    check_records_agree(count, fingerprint, c.device, group)
    records = rb.render_exact(c.scene, opts, api._ptr(rb, grad_img.contiguous()), g.d_scene)
    dist.all_reduce(records, op=dist.ReduceOp.SUM, group=group)
    rb.round_exact(c.scene, opts, g.d_scene, None, records)  # (render_exact wrote none of g's buffers: they are still zero)
    return api.RenderFunction.gradient_outputs(c, g)


class TileRenderFunction(torch.autograd.Function):
    """RenderFunction for one image sharded over the ranks of a process group."""

    @staticmethod
    def forward(ctx, seed, group, rows_per_stripe, *args):
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        if not isinstance(seed, tuple):
            seed = (seed, seed + 1000003)
        c = api.RenderFunction._unpack(seed, args)
        c.scene.set_partition(rank, world, rows_per_stripe)
        img = api._render(c)
        dist.all_reduce(img, op=dist.ReduceOp.SUM, group=group)  # disjoint stripes: a sum is a gather
        ctx.c, ctx.args, ctx.group = c, args, group
        return img

    @staticmethod
    def backward(ctx, grad_img):
        # every rank holds the full d_image (the loss is computed on the all-reduced image on every rank)
        if torch.are_deterministic_algorithms_enabled():
            grad_img = grad_img.contiguous()
            assert torch.isfinite(grad_img).all()
            return (None, None, None) + _exact_backward(ctx.c, grad_img, ctx.group)[1:]
        grads = api._backward(ctx.c, grad_img)
        reduced = iter(all_reduce_packed([g.to(ctx.c.device) for g in grads if isinstance(g, torch.Tensor)], ctx.group))
        out = [next(reduced).to(g.device) if isinstance(g, torch.Tensor) else g for g in grads]
        return (None, None, None) + tuple(out[1:])


def render_tiles(scene, num_samples, max_bounces, seed, group=None, rows_per_stripe: int = 4, **kw):
    args = api.RenderFunction.serialize_scene(scene, num_samples, max_bounces, **kw)
    return TileRenderFunction.apply(seed, group, rows_per_stripe, *args)


def render_poses(render_one: Callable[[int], torch.Tensor], num_poses: int, params: Sequence[torch.Tensor], loss_fn, group=None):
    """Data-parallel loop over poses: rank r handles poses r, r+world, ...; returns (local loss sum, reduced grads)."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    total = None
    for p in range(rank, num_poses, world):
        loss = loss_fn(render_one(p), p)
        loss.backward()
        total = loss.detach() if total is None else total + loss.detach()
    grads = [(q.grad if q.grad is not None else torch.zeros_like(q)) for q in params]
    devs = [g.device for g in grads]
    dev0 = grads[0].device if len(grads) else torch.device("cpu")
    if any(d.type == "cuda" for d in devs):
        dev0 = next(d for d in devs if d.type == "cuda")
    reduced = all_reduce_packed([g.to(dev0) for g in grads], group)
    return total, [r.to(d) for r, d in zip(reduced, devs)]
