"""Chunk-parallel sampler on 2 and 3 ranks (gloo, CPU): the exact mode (per-step x0 all-gather) must be
bit-identical to the single-process chunk loop; the literal north-star mode (no per-step exchange)
must run and -- as SURVEY 8e predicts -- differ from it on multi-chunk inputs."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.util import FakeDenoiser, make_inputs

CHUNKS = [(0, 8), (4, 12), (8, 20)]


def _run(diffusion, mode, seed=77, chunks=CHUNKS, frames=20, model=None):
    x, hint, y = make_inputs(21, 1, frames, 10, 8)
    _, _, ny = make_inputs(22, 1, frames, 10, 8)
    g = torch.Generator().manual_seed(seed)
    return diffusion.sample_sr(noise=x.clone(), model=model or FakeDenoiser(), model_kwargs=[{"y": y}, {"y": ny}, {"hint": hint}],
                               guide_scale=7.5, guide_rescale=0.2, solver="dpmpp_2m_sde", solver_mode="normal", steps=3,
                               t_max=899, t_min=0, discretization="trailing", chunk_inds=list(chunks),
                               noise_sampler=lambda a, b: torch.randn(x.shape, generator=g), chunk_parallel=mode)


def _make_diffusion():
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    from star_b200.video_to_video.diffusion.schedules_sdedit import noise_schedule
    return GaussianDiffusion(noise_schedule(schedule="logsnr_cosine_interp", n=1000, zero_terminal_snr=True,
                                            scale_min=2.0, scale_max=4.0))


def _worker(rank, world, port, q, chunks, frames):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        d = _make_diffusion()
        exact = _run(d, "exact", chunks=chunks, frames=frames)
        literal = _run(d, "literal", chunks=chunks, frames=frames)
        q.put((rank, exact.numpy(), literal.numpy()))      # by value: the worker may exit before the parent reads
    finally:
        dist.destroy_process_group()


def test_two_rank_chunk_parallel():
    """2 ranks over 3 chunks; and 3 ranks over 2 chunks, where rank 2 owns no chunk and sends an empty share"""
    for world, chunks, frames in ((2, CHUNKS, 20), (3, CHUNKS[:2], 12)):
        single = _run(_make_diffusion(), "auto", chunks=chunks, frames=frames)      # no process group -> serial chunk loop
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        procs = [ctx.Process(target=_worker, args=(r, world, port, q, chunks, frames)) for r in range(world)]
        for p in procs:
            p.start()
        res = [q.get(timeout=120) for _ in procs]
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
        for rank, exact, literal in res:
            exact, literal = torch.from_numpy(exact), torch.from_numpy(literal)
            assert torch.equal(exact, single), f"{world} ranks, rank {rank}: exact chunk-parallel result differs from the serial loop"
            assert literal.shape == single.shape
            assert not torch.equal(literal, single), "literal mode unexpectedly equals the stitched result"
            if len(chunks) > 2:       # with two chunks the fake denoiser's literal result stays within ~1e-5 of it
                assert not torch.allclose(literal, single, atol=1e-3), "literal mode unexpectedly equals the stitched result"


class _HalfDenoiser(FakeDenoiser):
    """returns fp16 like the .half() UNet: the CFG combine then runs in fp16 (ref :89), the wire dtype must follow"""

    def forward(self, *a, **k):
        return super().forward(*a, **k).half()


C3_CHUNKS = [(0, 8), (4, 12), (8, 18)]        # config 3 in miniature: 3 chunks, stretched last chunk


def _worker_split(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        d = _make_diffusion()
        m = _HalfDenoiser()
        out = _run(d, "auto", chunks=C3_CHUNKS, frames=18, model=m)
        q.put((rank, out.numpy(), len(m.calls)))
    finally:
        dist.destroy_process_group()


def test_cfg_branch_split_six_ranks():
    """3 chunks on 6 ranks: one (chunk, CFG branch) unit per rank, one all-gather of raw model outputs per step;
    bit-identical to the serial loop, one model call per rank per step instead of six."""
    single_model = _HalfDenoiser()
    single = _run(_make_diffusion(), "auto", chunks=C3_CHUNKS, frames=18, model=single_model)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world = 7                                    # 6 active ranks + 1 idle rank (8 GPUs with 3 chunks leave 2 idle)
    procs = [ctx.Process(target=_worker_split, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    steps = len(single_model.calls) // 6
    for rank, out, calls in res:
        out = torch.from_numpy(out)
        assert torch.equal(out, single), f"rank {rank}: CFG-split result differs from the serial loop"
        assert calls == (steps if rank < 6 else 0), f"rank {rank}: {calls} model calls for {steps} steps"


def test_stitch_slices():
    from star_b200.video_to_video.diffusion.diffusion_sdedit import stitch_slices
    keep = stitch_slices([(0, 32), (16, 48), (32, 72)])
    assert keep == [(0, 24), (8, 24), (8, 40)]
    assert sum(hi - lo for lo, hi in keep) == 72
