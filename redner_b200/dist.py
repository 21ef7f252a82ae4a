"""Multi-GPU rendering: one process per GPU (torch.distributed), no reference counterpart (the reference only lets the
caller pick a device: pyredner/device.py:26-33, src/pathtracer.cpp:184-192).

Two ways to use N GPUs (SURVEY.md section 8e):

* `render_tiles`  -- ONE image, split into round-robin stripes of viewport rows (rb_scene_set_partition).  Samplers stay
  seeded by the full-viewport pixel index, so the union over ranks equals the single-GPU image bit for bit; primary-edge
  samples are sharded by sample index.  One collective at the end of each pass: all_reduce(sum) of the framebuffer
  (ranks hold zeros outside their stripes) after forward, and of the packed gradient buffers after backward.
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


class TileRenderFunction(torch.autograd.Function):
    """RenderFunction for one image sharded over the ranks of a process group."""

    @staticmethod
    def forward(ctx, seed, group, rows_per_stripe, *args):
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        if not isinstance(seed, tuple):
            seed = (seed, seed + 1000003)
        c = api.RenderFunction._unpack(seed, args)
        rb = c.backend
        c.scene.set_partition(rank, world, rows_per_stripe)
        nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
        h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
        img = torch.zeros(h, w, nch, device=c.device)
        rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
        dist.all_reduce(img, op=dist.ReduceOp.SUM, group=group)  # disjoint stripes: a sum is a gather
        ctx.c, ctx.args, ctx.group = c, args, group
        return img

    @staticmethod
    def backward(ctx, grad_img):
        # every rank holds the full d_image (the loss is computed on the all-reduced image on every rank)
        ctx_like = type("C", (), {})()
        ctx_like.c, ctx_like.args = ctx.c, ctx.args
        grads = api.RenderFunction.backward(ctx_like, grad_img)
        tens = [g for g in grads if isinstance(g, torch.Tensor)]
        dev = ctx.c.device
        moved = [t.to(dev) for t in tens]
        reduced = all_reduce_packed(moved, ctx.group)
        it = iter(reduced)
        out = []
        for g in grads:
            if isinstance(g, torch.Tensor):
                r = next(it)
                out.append(r.to(g.device))
            else:
                out.append(g)
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
