"""GPU suite: exact records (rb_exact_record_count, rb_render_exact, rb_exact_round) on the CUDA library.

- Partition sums: for every case of the deterministic suite, the records of the stripes of a 2-, 3- and 8-way partition (1- and 4-row
  stripes), each stripe's gradient descriptor in an address order of its own, summed as int64 and rounded once, equal the
  unpartitioned deterministic rb_render bit for bit in every buffer, camera and screen-gradient image included; once more with many
  small bands (RB_BAND_BYTES).
- One render's records, rounded, equal that render; crafted records (non-finite counts, carries, a zero sum) round as they should on
  the device; a wrong count, NULL records and overlapping buffers are refused.
- With two visible GPUs: dist.render_tiles over NCCL at world size 2 gives the one-GPU deterministic gradients bit for bit."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import exact_records_check as xc
from test_deterministic_gpu import REPEAT_CASES

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("name", list(REPEAT_CASES))
def test_partition_records_summed_and_rounded_equal_one_deterministic_render(rb, dev, name):
    cfg, kind = REPEAT_CASES[name]
    xc.partition_sums(rb, dev, cfg, kind, (2, 3, 8))


@pytest.mark.parametrize("name", list(REPEAT_CASES))
def test_partition_records_with_small_bands(rb, dev, name, monkeypatch):
    monkeypatch.setenv("RB_BAND_BYTES", str(1 << 20))
    cfg, kind = REPEAT_CASES[name]
    xc.partition_sums(rb, dev, cfg, kind, (2, 3, 8), rows=(4,))


def test_records_of_one_render_rounded_equal_the_deterministic_render(rb, dev):
    cfg, kind = REPEAT_CASES["glossy_room_both_edges"]
    xc.partition_sums(rb, dev, cfg, kind, (1,), rows=(4,))


def test_crafted_records_sum_non_finite_counts_and_carries(rb, dev):
    xc.crafted_records(rb, dev)


def test_wrong_count_null_records_and_overlapping_buffers_are_refused(rb, dev):
    xc.refusals(rb, dev)


# ---------------------------------------------------------------------------------------------------- NCCL
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _render(rb, dev, render):
    import parity_utils as pu
    import scenes
    torch.use_deterministic_algorithms(True, warn_only=True)
    sc = scenes.glossy_room(dev, resolution=(64, 48))
    img = render(sc, dict(sampler_type=rb.SamplerType.sobol, device=dev, backend=rb, use_primary_edge_sampling=True, use_secondary_edge_sampling=True))
    img.pow(2).sum().backward()
    torch.cuda.synchronize(dev)
    return img.detach().cpu().numpy(), pu.collect_grads(sc)


def _nccl_worker(rank, world, port, out_path):
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import dist as rdist, redner as rb
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        img, g = _render(rb, torch.device("cuda", rank), lambda sc, kw: rdist.render_tiles(sc, 8, 2, seed=7, rows_per_stripe=4, **kw))
        if rank == 0:
            np.savez(out_path, image=img, **{k: v.numpy() for k, v in g.items()})
    finally:
        dist.destroy_process_group()


def test_nccl_world_size_2_gives_the_one_gpu_deterministic_gradients(rb, dev, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs (found %d)" % torch.cuda.device_count())
    import torch.multiprocessing as mp
    from redner_b200 import api
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        img1, g1 = _render(rb, dev, lambda sc, kw: api.RenderFunction.apply((7, 7 + 1000003), *api.RenderFunction.serialize_scene(sc, 8, 2, **kw)))
    finally:
        torch.use_deterministic_algorithms(prev)
    path = str(tmp_path / "w2.npz")
    mp.spawn(_nccl_worker, args=(2, _free_port(), path), nprocs=2, join=True)
    out = dict(np.load(path))
    assert out["image"].tobytes() == img1.tobytes()
    assert set(out) - {"image"} == set(g1) and len(g1) > 5
    for k, v in g1.items():
        assert out[k].tobytes() == v.numpy().tobytes(), k
