"""Tiled sampling under a process group, without a GPU: chunk_parallel="literal" with tiles is refused before the sampler
touches its model or inputs, the wire buffer of a round of windows is padded to its longest window, and the round's
all-gather (gloo, CPU tensors, 2 and 3 ranks) hands every rank each window's outputs cropped back to the window."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_stream_cpu import Forbidden


def _diffusion():
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    from star_b200.video_to_video.diffusion.schedules_sdedit import noise_schedule
    return GaussianDiffusion(noise_schedule(schedule="logsnr_cosine_interp", n=1000, zero_terminal_snr=True,
                                            scale_min=2.0, scale_max=4.0))


def test_literal_with_tiles_refused_before_any_work(monkeypatch):
    from star_b200.video_to_video.diffusion import diffusion_sdedit as D
    monkeypatch.setattr(D, "_dist_info", lambda: (2, 0))
    with pytest.raises(NotImplementedError, match="literal"):
        _diffusion().sample_sr(noise=Forbidden("noise"), model=Forbidden("model"), model_kwargs=Forbidden("model_kwargs"),
                               guide_scale=7.5, solver="dpmpp_2m_sde", steps=2, discretization="trailing",
                               chunk_parallel="literal", tile_inds=Forbidden("tile_inds"))


def _windows(frames, chunks, h, w, tile, overlap):
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    from star_b200.video_to_video.video_to_video_model import make_tiles
    noise = torch.zeros(1, 4, frames, h, w)
    kwargs = [{"y": None}, {"y": None}, {"hint": noise}]
    return GaussianDiffusion._windows(noise, chunks, make_tiles(h, w, tile, overlap), kwargs, 7.5, None, None), noise


UNEQUAL = [(0, 8), (4, 12), (8, 18)]          # make_chunks(18, 0, 8): the last chunk is stretched to 10 frames


@pytest.mark.parametrize("world,want", [
    (2, [(2, 1, 4, 8, 26, 32), (2, 1, 4, 8, 26, 32), (2, 1, 4, 10, 26, 32)]),
    (3, [(2, 1, 4, 8, 26, 32), (2, 1, 4, 10, 26, 32)]),             # round 1 mixes an 8- and a 10-frame chunk
    (4, [(2, 1, 4, 8, 26, 32), (2, 1, 4, 10, 26, 32)]),             # round 1: two windows, two idle ranks
    (8, [(2, 1, 4, 10, 26, 32)]),                                   # one round holds every window
])
def test_round_shape_pads_to_the_longest_window(world, want):
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    wins, noise = _windows(18, UNEQUAL, 26, 48, (26, 32), 8)
    assert len(wins) == 6
    got = [GaussianDiffusion._round_shape(wins[k:k + world], noise, True) for k in range(0, len(wins), world)]
    assert got == want
    assert GaussianDiffusion._round_shape(wins[:world], noise, False)[0] == 1


def _gather_worker(rank, world, port, q, pair):
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        wins, noise = _windows(18, UNEQUAL, 26, 48, (26, 32), 8)
        got = []
        for k in range(0, len(wins), world):
            rnd = wins[k:k + world]
            out = _window_outputs(k + rank, rnd[rank], pair) if rank < len(rnd) else None
            got.append([tuple(o.numpy() for o in (x if pair else (x,))) for x in
                        GaussianDiffusion._gather_round(out, rnd, pair, noise)])
        q.put((rank, got))
    finally:
        dist.destroy_process_group()


def _window_outputs(i, win, pair):
    """distinct fp16 outputs of window i, shaped like the window"""
    s, e, _, _, r0, r1, c0, c1 = win[:8]
    g = torch.Generator().manual_seed(100 + i)
    outs = tuple(torch.randn(1, 4, e - s, r1 - r0, c1 - c0, generator=g).half() for _ in range(2 if pair else 1))
    return outs if pair else outs[0]


@pytest.mark.parametrize("world,pair", [(2, True), (3, True), (3, False)])
def test_gather_round_returns_every_window_cropped(world, pair):
    wins, _ = _windows(18, UNEQUAL, 26, 48, (26, 32), 8)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gather_worker, args=(r, world, port, q, pair)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = [q.get(timeout=120) for _ in procs]
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    for rank, rounds in res:
        flat = [w for rnd in rounds for w in rnd]
        assert len(flat) == len(wins)
        for i, (win, got) in enumerate(zip(wins, flat)):
            want = _window_outputs(i, win, pair)
            for g, w in zip(got, want if pair else (want,)):
                assert torch.equal(torch.from_numpy(g), w), f"rank {rank}, window {i}"
