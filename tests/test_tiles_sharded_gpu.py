"""Tiled sampling and enhance_frames under a process group of 2 and 3 ranks, all on the one GPU (gloo carries the CUDA
tensors of all_gather and broadcast; NCCL refuses two ranks on one device).  Reduced UNet, small temporal VAE, synthetic
weights, seeded inputs:

* every rank's tiled denoised latent equals the single-process tiled run byte for byte, and each rank ran the model on
  its own windows only (windows r, r + W, ... of each evaluation): one chunk x 4 tiles, 3 chunks of unequal length x 2
  tiles, an idle rank in every round, guide_scale 1.0 (one branch) and CUDA graphs;
* the single-process tiled run equals a transcription of the tile loop before sharding, byte for byte;
* round-wise enhance_frames equals _test_on_device + ops.adain_color_fix on the same ranks byte for byte, and its peak
  device memory grows by less than one decoded frame per added frame."""
import datetime
import os
import pickle
import socket
import traceback
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_spatial_tiles_gpu import latents, pinned_sampler
from tests.util import SMALL_KW, synth_model

pytestmark = pytest.mark.gpu

DECODED_FRAME = 3 * 720 * 1280 * 2           # bytes of one decoded fp16 canvas frame (5.5 MB)

# name: (ranks, frames, latent h x w, max_chunk_len, tile, overlap, guide_scale, cuda_graph)
TILE_CASES = {
    "1 chunk x 4 tiles": (2, 8, (42, 48), 32, (26, 32), 8, 7.5, False),
    "guide_scale 1.0": (2, 8, (42, 48), 32, (26, 32), 8, 1.0, False),
    "cuda graph, 3 unequal chunks x 2 tiles": (2, 18, (26, 48), 8, (26, 32), 8, 7.5, True),
    "3 unequal chunks x 2 tiles": (3, 18, (26, 48), 8, (26, 32), 8, 7.5, False),     # rounds mix 8- and 10-frame chunks
    "2 windows on 3 ranks": (3, 8, (26, 48), 32, (26, 32), 8, 7.5, False),
}


def _pipe(net, vae=object(), cuda_graph=False):
    from star_b200.video_to_video.video_to_video_model import VideoToVideo_sr
    ny = -torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(4))
    return VideoToVideo_sr(SimpleNamespace(model_path=None), device=torch.device("cuda"), text_encoder=lambda s: ny, vae=vae,
                           generator=net, cuda_graph=cuda_graph)


def _record_windows(calls):
    """log the window of every model call of tiled sampling (in this process)"""
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    real = GaussianDiffusion._window_out

    def recording(self, xt, t, win, *a, **k):
        calls.append(tuple(win[:8]))
        return real(self, xt, t, win, *a, **k)
    GaussianDiffusion._window_out = recording
    return real


def _denoise(net, case):
    _, F, (H, W), mcl, tile, overlap, gs, graphed = TILE_CASES[case]
    feat, y, ny, noise = latents(F, H, W, seed=51)
    pipe = _pipe(net, cuda_graph=graphed)
    z = pipe.denoise_latents(feat, y, ny, steps=2, solver_mode="normal", guide_scale=gs, max_chunk_len=mcl, noise=noise,
                             noise_sampler=pinned_sampler(feat.shape, 5), tile_size=tile, tile_overlap=overlap)
    if graphed:
        assert pipe._graphed.replays > 0
    return z


def _port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _spawn(world, target, *args):
    """run target(rank, world, *args) -> result on `world` gloo ranks in fresh processes; returns the results by rank.
    No process outlives the call."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, target, args)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(pickle.loads(q.get(timeout=600)) for _ in procs)
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    errors = [res[r][1] for r in sorted(res) if res[r][1] is not None]
    assert not errors, "\n".join(errors)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [res[r][0] for r in range(world)]


def _worker(rank, world, port, q, target, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        res = (target(rank, world, *args), None)
    except BaseException:
        res = (None, f"rank {rank}:\n{traceback.format_exc()}")
    finally:
        dist.destroy_process_group()
    q.put(pickle.dumps((rank, res)))             # by value: the worker exits before the parent reads


# -- tiled sampling ---------------------------------------------------------------------------------------------------
def _tiles_on_ranks(rank, world, cases):
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    out = {}
    for case in cases:
        calls = []
        real = _record_windows(calls)
        try:
            z = _denoise(net, case)
        finally:
            GaussianDiffusion._window_out = real
        out[case] = (z.cpu(), calls)
    return out


@pytest.fixture(scope="module")
def single():
    """the single-process tiled runs: (denoised latent, windows of the model calls) per case"""
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    out = {}
    for case in TILE_CASES:
        calls = []
        real = _record_windows(calls)
        try:
            out[case] = (_denoise(net, case).cpu(), calls)
        finally:
            GaussianDiffusion._window_out = real
    return out


@pytest.fixture(scope="module", params=[2, 3])
def sharded(request):
    world = request.param
    cases = [c for c, spec in TILE_CASES.items() if spec[0] == world]
    return world, cases, _spawn(world, _tiles_on_ranks, cases)


def test_sharded_tiles_equal_single_process(single, sharded):
    world, cases, per_rank = sharded
    for case in cases:
        want, calls = single[case]
        assert torch.isfinite(want).all()
        windows = sorted(set(calls), key=calls.index)                   # one evaluation's windows, in window order
        assert len(calls) % len(windows) == 0
        for rank, res in enumerate(per_rank):
            got, rank_calls = res[case]
            diff = (got - want).abs().max().item()
            print(f"{case}, {world} ranks, rank {rank}: max |sharded - single| {diff:.3e}, {len(rank_calls)} model calls")
            assert torch.equal(got, want), f"{case}: rank {rank} of {world} differs from the single-process run"
            mine = [w for w in calls if windows.index(w) % world == rank]
            assert rank_calls == mine, f"{case}: rank {rank} ran the model on windows other than its own"


def _eval_x0_tiled_serial(self, xt, t, alphas, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale,
                          variant_info, world=1, rank=0):
    """the tile loop before sharding: one model call and one blend per window, in window order"""
    from star_b200 import ops
    assert (world, rank) == (1, 0)
    xt = xt.float().contiguous()
    x0 = torch.zeros_like(xt)
    rescale = None if guide_scale == 1.0 else guide_rescale
    for win in windows:
        out = self._window_out(xt, t, win, model, model_kwargs, guide_scale, variant_info)[1]
        y_out, u_out = out if isinstance(out, tuple) else (out, out)
        s, _, lo, hi, r0, _, c0, _, wy, wx = win
        ops.cfg_x0(y_out.contiguous(), u_out.contiguous(), xt, alphas, sigmas, guide_scale, rescale,
                   blend=ops.TileBlend(x0, s, lo, hi, r0, c0, wy, wx))
    return x0


def test_single_process_tiles_unchanged(single, monkeypatch):
    from star_b200.video_to_video.diffusion.diffusion_sdedit import GaussianDiffusion
    monkeypatch.setattr(GaussianDiffusion, "_eval_x0_tiled", _eval_x0_tiled_serial)
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    for case in TILE_CASES:
        assert torch.equal(_denoise(net, case).cpu(), single[case][0]), case


# -- enhance_frames ---------------------------------------------------------------------------------------------------
STEPS = dict(steps=2, solver_mode="normal", guide_scale=7.5)
# name: (frames, LR size, uint8, tile_size)
ENHANCE_CASES = {
    "centred F=7, 3 windows": (7, (96, 160), True, None),
    "centred F=4, fp32": (4, (96, 160), False, None),
    "bottom-right pad F=2, 1 window": (2, (188, 336), True, None),       # 752x1344 -> canvas 784x1408
    "tiles F=5": (5, (96, 160), True, (50, 96)),
}


def _clip(F, lr, scale=4, seed=7):
    g = torch.Generator().manual_seed(seed)
    video = torch.rand(F, 3, *lr, generator=g) * 2 - 1
    return {"video_data": video, "y": torch.randn(1, 77, 1024, generator=g), "target_res": (lr[0] * scale, lr[1] * scale)}


def _peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def _enhance_on_ranks(rank, world):
    from star_b200 import ops
    from star_b200.video_to_video.utils.seed import setup_seed
    from tests.test_vae import SMALL, _setup
    net, _ = synth_model(SMALL_KW, seed=1, device="cuda")
    pipe = _pipe(net, vae=_setup(SMALL, device="cuda")[2])
    out = {}
    for case, (F, lr, uint8, tile) in ENHANCE_CASES.items():
        inp = _clip(F, lr)
        kw = dict(STEPS, tile_size=tile)
        setup_seed(666)
        got = pipe.enhance_frames(inp, uint8=uint8, **kw)
        setup_seed(666)
        vid = pipe.test(inp, **kw).cuda()              # _test_on_device, in fp32 on the host
        want = ops.adain_color_fix(vid, inp["video_data"].cuda().float(), uint8=uint8).cpu()
        out[case] = (got, want)

    kw = dict(steps=1, solver_mode="normal", guide_scale=7.5, max_chunk_len=6)

    def run(F):
        pipe.enhance_frames(_clip(F, (180, 320)), **kw)
    run(6)                                     # lazy weight packing and every window shape, outside the measurement
    out["peaks"] = (_peak_bytes(lambda: run(6)), _peak_bytes(lambda: run(24)))
    return out


@pytest.fixture(scope="module")
def enhanced():
    return _spawn(2, _enhance_on_ranks)


@pytest.mark.parametrize("case", list(ENHANCE_CASES))
def test_round_wise_enhance_frames_equals_whole_clip(enhanced, case):
    F, lr, uint8, _ = ENHANCE_CASES[case]
    for rank, res in enumerate(enhanced):
        got, want = res[case]
        assert got.shape == (F, 4 * lr[0], 4 * lr[1], 3) and got.dtype == (torch.uint8 if uint8 else torch.float32)
        diff = (got.double() - want.double()).abs()
        print(f"{case}, rank {rank}: max |round-wise - whole clip| {diff.max().item()}")
        assert torch.equal(got, want), f"{case}: rank {rank}: {int((diff > 0).sum())} values differ"
        assert torch.equal(got, enhanced[0][case][0])


def test_round_wise_enhance_frames_memory_does_not_grow_with_the_clip(enhanced):
    """720x1280 canvas (LR 180x320, x4), one solver step, 6-frame chunks, 6 and 24 frames: the peak's growth per added
    frame on each rank, against one decoded fp16 frame of the canvas"""
    for rank, res in enumerate(enhanced):
        p6, p24 = res["peaks"]
        grow = (p24 - p6) / 18
        print(f"rank {rank}: peak {p6 / 2 ** 20:.1f} MiB at 6 frames, {p24 / 2 ** 20:.1f} MiB at 24: "
              f"{grow / 1e6:.3f} MB per frame")
        assert grow < DECODED_FRAME, f"rank {rank}: peak grows by {grow / 1e6:.3f} MB per frame"
