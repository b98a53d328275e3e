"""v-prediction diffusion wrapper of STAR: CFG denoise step, sigma/timestep
tables, per-step chunk loop + stitch, and chunk-parallel execution.

Mirrors ``GaussianDiffusion`` of the reference's
video_to_video/diffusion/diffusion_sdedit.py (same method names, argument
meaning and assertion behaviour):
    diffuse      :26-30      denoise    :44-115     sample_sr :265-412
    _sigma_to_t  :415-433    _t_to_sigma :435-443
The legacy ``sample`` (:118-262) dereferences model_kwargs[3] and cannot run
with STAR's 3-entry kwargs; it is not part of the hot path and is not provided.

Multi-GPU (new, SURVEY 8e): when ``torch.distributed`` is initialised with
world_size > 1 and ``chunk_inds`` is given, rank r evaluates chunks r, r+W, ...
and the kept centre slices of x0 are exchanged with ONE all-gather per solver
step ("exact" mode: bit-identical stitching to the single-GPU loop, because
the reference re-stitches all chunks every step, :330-353).  ``chunk_parallel=
"literal"`` is the north-star wording (no per-step collective; each rank
integrates its own chunk for all steps and the slices are gathered once at the
end) -- it only equals the reference for single-chunk inputs.  With spatial tiles (``tile_inds``) the (chunk, tile)
windows are sharded instead, and their raw outputs are all-gathered one round of W windows at a time.
"""
import random

import torch
import torch.distributed as dist

from ..utils.logger import get_logger
from ..utils.sharding import _all_gather_owned, _dist_info
from .solvers_sdedit import sample_dpmpp_2m_sde, sample_heun

logger = get_logger()

__all__ = ["GaussianDiffusion", "stitch_slices"]


def _gather_coef(table, t, like):
    """table[t] broadcast against ``like`` (ref ``_i``, :17-19)."""
    return table[t.to(table.device)].view((like.size(0),) + (1,) * (like.ndim - 1)).to(like.device)


def stitch_slices(chunk_inds):
    """Frame ranges each chunk contributes to the stitched x0 (ref :333-350):
    with overlap O = end(chunk0) - start(chunk1) and cut = O // 2, the first
    chunk keeps [0, len-(O-cut)), middle chunks [cut, len-(O-cut)), the last
    chunk [cut, len).  Returns [(lo, hi)] in chunk-local frame indices."""
    overlap = chunk_inds[0][-1] - chunk_inds[1][0]
    cut = overlap // 2
    out = []
    for i, (s, e) in enumerate(chunk_inds):
        n = e - s
        lo = 0 if i == 0 else cut
        hi = n if i == len(chunk_inds) - 1 else n + cut - overlap
        out.append((lo, hi))
    return out


class GaussianDiffusion(object):

    def __init__(self, sigmas):
        self.sigmas = sigmas
        self.alphas = torch.sqrt(1 - sigmas ** 2)
        self.num_timesteps = len(sigmas)

    # -- forward process ------------------------------------------------------
    def diffuse(self, x0, t, noise=None):
        noise = torch.randn_like(x0) if noise is None else noise
        return _gather_coef(self.alphas, t, x0) * x0 + _gather_coef(self.sigmas, t, x0) * noise

    # -- one denoise evaluation (2 model calls under CFG) -----------------------
    def denoise(self, xt, t, s, model, model_kwargs={}, guide_scale=None, guide_rescale=None,
                clamp=None, percentile=None, variant_info=None):
        s = t - 1 if s is None else s
        sigmas = _gather_coef(self.sigmas, t, xt)
        alphas = _gather_coef(self.alphas, t, xt)
        alphas_s = _gather_coef(self.alphas, s.clamp(0), xt)
        alphas_s[s < 0] = 1.0
        sigmas_s = torch.sqrt(1 - alphas_s ** 2)
        betas = 1 - (alphas / alphas_s) ** 2
        coef1 = betas * alphas_s / sigmas ** 2
        coef2 = (alphas * sigmas_s ** 2) / (alphas_s * sigmas ** 2)
        var = betas * (sigmas_s / sigmas) ** 2
        log_var = torch.log(var).clamp_(-20, 20)

        out = self._model_out(xt, t, model, model_kwargs, guide_scale, variant_info)
        x0 = self._x0(xt, out, alphas, sigmas, guide_scale, guide_rescale, clamp, percentile)
        eps = (xt - alphas * x0) / sigmas
        mu = coef1 * x0 + coef2 * xt
        return mu, var, log_var, x0, eps

    def _model_out(self, xt, t, model, model_kwargs, guide_scale, variant_info, branch=None):
        """The model call(s) of one denoise evaluation: the output, or the (conditional, unconditional) pair under CFG;
        ``branch`` (0 = conditional, 1 = unconditional) runs that CFG branch alone (ref :76-88)."""
        if guide_scale is None:
            assert isinstance(model_kwargs, dict)
            return model(xt, t=t, **model_kwargs)
        assert isinstance(model_kwargs, list)
        extra = {}
        for kw in model_kwargs[2:]:
            extra.update(kw)
        if len(model_kwargs) <= 3:
            extra["variant_info"] = variant_info
        if branch is not None or guide_scale == 1.0:
            return model(xt, t=t, **model_kwargs[branch or 0], **extra)
        pair = getattr(model, "forward_cfg_pair", None)
        if pair is not None and set(model_kwargs[0]) == set(model_kwargs[1]) == {"y"}:
            # the two branches differ only in the text embedding: the model evaluates their common, text-independent
            # prefix once (bit-identical to two calls, tests/test_unet_gpu.py::test_cfg_pair_equals_two_forwards)
            return pair(xt, t, (model_kwargs[0]["y"], model_kwargs[1]["y"]), **extra)
        return model(xt, t=t, **model_kwargs[0], **extra), model(xt, t=t, **model_kwargs[1], **extra)

    def _x0(self, xt, out, alphas, sigmas, guide_scale, guide_rescale, clamp=None, percentile=None):
        """x0 of one evaluation on xt from the model output, or from the (conditional, unconditional) pair under CFG:
        CFG combine + std-ratio rescale + v -> x0 (ref :89-99).  An fp16 CUDA pair (the .half() UNet) takes the fused
        device path -- two launches (star_cfg_x0) instead of ~20 eager tensor ops; anything else (CPU tests, fp32 fakes)
        runs the reference's tensor arithmetic."""
        if not isinstance(out, tuple):
            return self._x0_from_out(xt, alphas, sigmas, out, clamp, percentile)
        y_out, u_out = out
        if y_out.is_cuda and y_out.dtype == torch.float16 and u_out.dtype == torch.float16 and clamp is None \
                and percentile is None:
            from ... import ops
            return ops.cfg_x0(y_out.contiguous(), u_out.contiguous(), xt, alphas, sigmas, guide_scale, guide_rescale)
        return self._x0_from_out(xt, alphas, sigmas, self._guided(y_out, u_out, guide_scale, guide_rescale), clamp, percentile)

    @staticmethod
    def _x0_from_out(xt, alphas, sigmas, out, clamp=None, percentile=None):
        """v-prediction -> x0 (ref :99).  The reference's dynamic-threshold / clamp options (:100-107) are never
        set by VideoToVideo_sr.test (:110-123) and are not carried over."""
        if clamp is not None or percentile is not None:
            raise NotImplementedError("clamp / percentile are not used on STAR's path (ref video_to_video_model.py:110-123)")
        return alphas * xt - sigmas * out

    @staticmethod
    def _guided(y_out, u_out, guide_scale, guide_rescale):
        """CFG combine + std-ratio rescale in the model's output dtype (fp16 in
        the reference, :89-97)."""
        out = u_out + guide_scale * (y_out - u_out)
        if guide_rescale is not None:
            assert 0 <= guide_rescale <= 1
            ratio = (y_out.flatten(1).std(dim=1) / (out.flatten(1).std(dim=1) + 1e-12)
                     ).view((-1,) + (1,) * (y_out.ndim - 1))
            out = out * (guide_rescale * ratio + (1 - guide_rescale) * 1.0)
        return out

    def _t_coefs(self, xt, sigma):
        """The timestep of a solver evaluation at k-diffusion ``sigma``, one per sample of xt, and alphas / sigmas there."""
        t = self._sigma_to_t(sigma).repeat(len(xt)).round().long()
        return t, _gather_coef(self.alphas, t, xt), _gather_coef(self.sigmas, t, xt)

    # -- sampler ---------------------------------------------------------------
    @torch.no_grad()
    def sample_sr(self, noise, model, model_kwargs={}, condition_fn=None, guide_scale=None,
                  guide_rescale=None, clamp=None, percentile=None, solver='euler_a',
                  solver_mode='fast', steps=20, t_max=None, t_min=None, discretization=None,
                  discard_penultimate_step=None, return_intermediate=None, show_progress=False,
                  seed=-1, chunk_inds=None, variant_info=None, chunk_parallel="auto", tile_inds=None, **kwargs):
        """Every solver-step evaluation runs the model on the windows of _windows -- the whole clip, or each chunk of
        ``chunk_inds`` -- and stitches the frames each window keeps into the clip's x0.  ``tile_inds`` (the output of
        video_to_video_model.make_tiles) turns on spatially tiled sampling: the windows are the (chunk, tile) pairs and
        their x0 are blended into the clip's x0 with the tiles' weights (see _eval_x0_tiled).

        Under a process group of W > 1 ranks with ``chunk_parallel`` "auto" or "exact", tiled sampling shards the (chunk,
        tile) windows round-robin, also for a single chunk, and exchanges their outputs round by round (_eval_x0_tiled): x0
        is byte-identical to the single-process loop on every rank.  Every rank then applies the same solver update from
        the same start: the SDE noise stream is seeded from rank 0 below, and denoise_latents broadcasts rank 0's diffused
        latent.  "literal" with tiles is refused: it has no per-step exchange to blend with."""
        assert isinstance(steps, (int, torch.LongTensor))
        assert t_max is None or (0 < t_max <= self.num_timesteps - 1)
        assert t_min is None or (0 <= t_min < self.num_timesteps - 1)
        assert discretization in (None, 'linspace', 'trailing')     # 'leading' (ref :360) is never selected by STAR
        assert discard_penultimate_step in (None, True, False)
        assert return_intermediate in (None, 'x0', 'xt')
        solver_fn = {'heun': sample_heun, 'dpmpp_2m_sde': sample_dpmpp_2m_sde}[solver]

        discretization = discretization or 'linspace'
        seed = seed if seed >= 0 else random.randint(0, 2 ** 31)
        if isinstance(steps, torch.LongTensor):
            discard_penultimate_step = False
        if discard_penultimate_step is None:
            discard_penultimate_step = solver == 'dpmpp_2m_sde'      # ref :318-321 (the other names are not selectable)

        # The reference raises IndexError for a single window (F in 33..40,
        # SURVEY App. B); a one-window list is the un-chunked case.
        if chunk_inds is not None and len(chunk_inds) < 2:
            chunk_inds = None
        group = chunk_parallel in ("auto", "exact", "literal") and _dist_info()[0] > 1
        if tile_inds is not None and group and chunk_parallel == "literal":
            raise NotImplementedError("sample_sr(tile_inds=...): chunk_parallel='literal' has no per-step exchange to blend the "
                                      "tiles with; use 'auto' or 'exact'")

        # Ranks of one job must integrate the same SDE path -- also for single-chunk clips, where every rank evaluates the whole
        # clip and the pipeline then shards only the VAE legs: share rank 0's noise seed whenever a process group exists.
        # Tiled sampling shards its (chunk, tile) windows also for a single chunk.
        world, rank = _dist_info() if group and (chunk_inds is not None or tile_inds is not None) else (1, 0)
        mode = "exact" if chunk_parallel == "auto" else chunk_parallel
        if group and solver == 'dpmpp_2m_sde' and kwargs.get('noise_sampler') is None:
            # every rank applies the same solver update: share the SDE noise stream (rank 0's seed)
            from .solvers_sdedit import IntervalNoiseSampler
            sd = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).to(noise.device)
            dist.broadcast(sd, 0)
            kwargs['noise_sampler'] = IntervalNoiseSampler(noise, seed=int(sd.item()))

        windows = self._windows(noise, chunk_inds, tile_inds, model_kwargs, guide_scale, clamp, percentile)
        # CFG-branch split (SURVEY 8e): with at least two ranks per chunk the (chunk, branch) pairs are the units --
        # BASELINE config 3 (3 chunks) then fills 6 of 8 GPUs instead of 3.  With tiles the units are the windows.
        split_cfg = (tile_inds is None and mode == "exact" and world >= 2 * len(windows) and isinstance(model_kwargs, list)
                     and guide_scale not in (None, 1.0))
        wire = {}
        intermediates = []

        def eval_x0(xt, sigma, variant_info=None):
            t, alphas, sigmas = self._t_coefs(xt, sigma)
            if tile_inds is not None:
                x0 = self._eval_x0_tiled(xt, t, alphas, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale,
                                         variant_info, world, rank)
            elif split_cfg:
                x0 = self._eval_x0_cfg_split(xt, t, alphas, sigmas, windows, model, model_kwargs, guide_scale,
                                             guide_rescale, variant_info, world, rank, wire)
            else:
                # the kept frames of each window (ref :337-350); in exact mode rank r evaluates windows r, r+W, ...
                # and ONE all-gather rebuilds the stitched x0 on every rank
                parts = []
                for win in windows[rank::world]:
                    x, out = self._window_out(xt, t, win, model, model_kwargs, guide_scale, variant_info)
                    lo, hi = win[2:4]
                    parts.append(self._x0(x, out, alphas, sigmas, guide_scale, guide_rescale, clamp, percentile)[:, :, lo:hi])
                if world > 1:
                    b, c, _, h, w = xt.shape
                    local = torch.concat(parts, dim=2).to(xt.dtype) if parts else xt.new_empty((b, c, 0, h, w))
                    x0 = _all_gather_owned(local, [hi - lo for _, _, lo, hi, *_ in windows], 2)
                else:
                    x0 = torch.concat(parts, dim=2) if len(parts) > 1 else parts[0]
            if return_intermediate == 'xt':
                intermediates.append(xt)
            elif return_intermediate == 'x0':
                intermediates.append(x0)
            return x0

        # -- timestep / sigma tables (ref :355-406) -----------------------------
        if isinstance(steps, int):
            steps += 1 if discard_penultimate_step else 0
            t_max = self.num_timesteps - 1 if t_max is None else t_max
            t_min = 0 if t_min is None else t_min
            if discretization == 'linspace':
                steps = torch.linspace(t_max, t_min, steps)
            elif discretization == 'trailing':
                steps = torch.arange(t_max, t_min - 1, -((t_max - t_min + 1) / steps))
                if solver_mode == 'fast':
                    t_mid = 500
                    head = torch.arange(t_max, t_mid - 1, -((t_max - t_mid + 1) / 4))
                    tail = torch.arange(t_mid, t_min - 1, -((t_mid - t_min + 1) / 11))
                    steps = torch.concat([head, tail])
            else:
                raise NotImplementedError(f'{discretization} discretization not implemented')
            steps = steps.clamp_(t_min, t_max)
        steps = torch.as_tensor(steps, dtype=torch.float32, device=noise.device)

        sigmas = self._t_to_sigma(steps)
        sigmas = torch.cat([sigmas, sigmas.new_zeros([1])])
        if discard_penultimate_step:
            sigmas = torch.cat([sigmas[:-2], sigmas[-1:]])

        if world > 1 and mode == "literal":
            x0 = self._sample_literal(noise, solver_fn, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale,
                                      clamp, percentile, variant_info, world, rank, show_progress, kwargs)
        else:
            x0 = solver_fn(noise, eval_x0, sigmas, variant_info=variant_info, show_progress=show_progress, **kwargs)
        return (x0, intermediates) if return_intermediate is not None else x0

    # -- windows: the frames, rows and columns of one model call ---------------------------------------------------------
    @staticmethod
    def _windows(noise, chunk_inds, tile_inds, model_kwargs, guide_scale, clamp, percentile):
        """The windows of one evaluation: [(s, e, lo, hi, r0, r1, c0, c1, wy, wx)], frames [s, e) of which the x0 keeps
        [lo, hi) (chunk-local, stitch_slices), rows [r0, r1) and cols [c0, c1).  One whole-frame window per chunk (one for
        the whole clip without chunks), or one per (chunk, tile) with the tile's weights uploaded once per call (else None)."""
        f, h, w = noise.shape[2:]
        chunks, kept = ([(0, f)], [(0, f)]) if chunk_inds is None else (chunk_inds, stitch_slices(chunk_inds))
        rows, cols, row_w, col_w = [(0, h)], [(0, w)], [None], [None]
        if tile_inds is not None:
            if guide_scale is None or not isinstance(model_kwargs, list) or len(model_kwargs) < 3 \
                    or 'hint' not in model_kwargs[2]:
                raise ValueError("sample_sr(tile_inds=...): tiled sampling needs classifier-free guidance (guide_scale) and "
                                 "model_kwargs [{'y': ...}, {'y': ...}, {'hint': ...}]")
            if clamp is not None or percentile is not None:
                raise NotImplementedError("sample_sr(tile_inds=...): clamp / percentile are not supported")
            rows, cols = tile_inds[:2]
            row_w, col_w = ([v.to(noise.device, torch.float32).contiguous() for v in ws] for ws in tile_inds[2:])
        return [(s, e, lo, hi, r0, r1, c0, c1, wy, wx)
                for (s, e), (lo, hi) in zip(chunks, kept)
                for (r0, r1), wy in zip(rows, row_w)
                for (c0, c1), wx in zip(cols, col_w)]

    @staticmethod
    def _crop(x, win):
        s, e, _, _, r0, r1, c0, c1, _, _ = win
        return x[:, :, s:e, r0:r1, c0:c1].contiguous()

    def _window_kwargs(self, model_kwargs, win):
        """The model kwargs of one window: the clip's, with its LR latent cropped to the window as ``hint_chunk``."""
        return [*model_kwargs[:2], dict(model_kwargs[2], hint_chunk=self._crop(model_kwargs[2]['hint'], win)),
                *model_kwargs[3:]]

    def _window_out(self, xt, t, win, model, model_kwargs, guide_scale, variant_info, branch=None):
        """(xt on the window, the model output(s) there; see _model_out).  The model runs on the window's crop of the clip
        latent and of the LR latent; a window that is the whole clip runs on xt and model_kwargs as they are."""
        s, e, _, _, r0, r1, c0, c1, _, _ = win
        if (e - s, r1 - r0, c1 - c0) != tuple(xt.shape[2:]):
            xt, model_kwargs = self._crop(xt, win), self._window_kwargs(model_kwargs, win)
        return xt, self._model_out(xt, t, model, model_kwargs, guide_scale, variant_info, branch)

    def _eval_x0_tiled(self, xt, t, alphas, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale, variant_info,
                       world=1, rank=0):
        """x0 of the clip = sum over (chunk, tile) windows of the tile's blend weight times its x0, restricted to the frames
        the chunk keeps (stitch_slices).  One star_cfg_x0_blend launch pair per window forms the guided x0 (CFG, std-ratio
        rescale over the window, v -> x0) and adds it into the clip's x0 in place.  Needs fp16 CUDA model outputs (the
        .half() UNet).

        On ``world`` ranks the windows run in rounds of ``world``: in round k rank r runs the model on window k * world + r,
        one all-gather carries the round's raw model outputs (_gather_round), and every rank blends the round's windows in
        window order.  The blends are those of the single-process loop, in its order, so x0 is byte-identical to it on every
        rank; an all-reduce of partial sums would reorder them."""
        from ... import ops
        xt = xt.float().contiguous()
        x0 = torch.zeros_like(xt)
        rescale = None if guide_scale == 1.0 else guide_rescale        # as _x0: no rescale without a second branch
        for k in range(0, len(windows), world):
            wins = windows[k:k + world]
            out = None
            if rank < len(wins):
                out = self._window_out(xt, t, wins[rank], model, model_kwargs, guide_scale, variant_info)[1]
                y_out, u_out = out if isinstance(out, tuple) else (out, out)
                if not (y_out.is_cuda and y_out.dtype == torch.float16 and u_out.dtype == torch.float16):
                    raise TypeError("sample_sr(tile_inds=...): tiled sampling blends on the GPU and needs fp16 CUDA model "
                                    f"outputs (the .half() UNet), got {y_out.dtype} on {y_out.device}")
            outs = [out] if world == 1 else self._gather_round(out, wins, guide_scale != 1.0, xt)
            for win, out in zip(wins, outs):
                y_out, u_out = out if isinstance(out, tuple) else (out, out)
                s, _, lo, hi, r0, _, c0, _, wy, wx = win
                ops.cfg_x0(y_out.contiguous(), u_out.contiguous(), xt, alphas, sigmas, guide_scale, rescale,
                           blend=ops.TileBlend(x0, s, lo, hi, r0, c0, wy, wx))
        return x0

    @staticmethod
    def _round_shape(wins, like, pair):
        """The wire buffer of one round of tiled windows: (branches, B, C, frames, rows, cols), the round's largest extent
        on each axis (chunks can differ in length), 2 branches under CFG with two model calls, else 1."""
        b, c = like.shape[:2]
        return ((2 if pair else 1), b, c, max(e - s for s, e, *_ in wins), max(w[5] - w[4] for w in wins),
                max(w[7] - w[6] for w in wins))

    @staticmethod
    def _gather_round(out, wins, pair, like):
        """ONE all-gather of a round of tiled windows' raw fp16 model outputs.  ``out`` is this rank's output -- the
        (conditional, unconditional) pair when ``pair``, else one tensor -- or None when it has no window in the round, in
        which case it sends only padding.  Returns the outputs of the round's windows in window order, cropped to each
        window.  Device memory: one round of padded outputs, independent of the frame size."""
        world, _ = _dist_info()
        send = torch.zeros(GaussianDiffusion._round_shape(wins, like, pair), dtype=torch.float16, device=like.device)
        if out is not None:
            for dst, o in zip(send, out if pair else (out,)):
                dst[:, :, :o.shape[2], :o.shape[3], :o.shape[4]] = o
        recv = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(recv, send)
        outs = []
        for (s, e, _, _, r0, r1, c0, c1, _, _), buf in zip(wins, recv):
            o = tuple(x[:, :, :e - s, :r1 - r0, :c1 - c0] for x in buf)
            outs.append(o if pair else o[0])
        return outs

    # -- chunk-parallel helpers -------------------------------------------------
    def _eval_x0_cfg_split(self, xt, t, alphas, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale,
                           variant_info, world, rank, wire):
        """Exact mode with two ranks per chunk: rank 2i evaluates the conditional branch of chunk i, rank 2i+1 the
        unconditional one (ranks >= 2n idle).  ONE all-gather of the raw model outputs per solver step; every rank
        then forms the guided output (needs both branches: std-ratio rescale, ref :89-97), x0 and the stitch for all
        chunks -- elementwise work on a few MB, identical on every rank and to the serial loop."""
        b, c, _, h, w = xt.shape
        out = None
        if rank < 2 * len(windows):
            i, branch = divmod(rank, 2)
            out = self._window_out(xt, t, windows[i], model, model_kwargs, guide_scale, variant_info, branch)[1]
        if "dtype" not in wire:                      # the model's output dtype (fp16 for the .half() UNet), agreed once
            codes = [torch.float16, torch.bfloat16, torch.float32, torch.float64]
            code = torch.tensor([codes.index(out.dtype) if out is not None else 0], device=xt.device)
            dist.broadcast(code, 0)
            wire["dtype"] = codes[int(code.item())]
        send = torch.zeros((b, c, max(e - s for s, e, *_ in windows), h, w), dtype=wire["dtype"], device=xt.device)
        if out is not None:
            send[:, :, :out.shape[2]] = out
        recv = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(recv, send)
        parts = []
        for (s, e, lo, hi, *_), y_out, u_out in zip(windows, recv[0::2], recv[1::2]):
            x0c = self._x0(xt[:, :, s:e], (y_out[:, :, :e - s], u_out[:, :, :e - s]), alphas, sigmas, guide_scale,
                           guide_rescale)
            parts.append(x0c[:, :, lo:hi])
        return torch.concat(parts, dim=2)

    def _sample_literal(self, noise, solver_fn, sigmas, windows, model, model_kwargs, guide_scale, guide_rescale, clamp,
                        percentile, variant_info, world, rank, show_progress, kwargs):
        """North-star literal mode: every rank integrates its own chunk(s) for
        all solver steps with no exchange; kept slices are gathered once."""
        outs = []
        for win in windows[rank::world]:
            s, e, lo, hi = win[:4]
            kw = self._window_kwargs(model_kwargs, win)

            def fn(xt, sigma, variant_info=None, kw=kw):
                t, al, sg = self._t_coefs(xt, sigma)
                out = self._model_out(xt, t, model, kw, guide_scale, variant_info)
                return self._x0(xt, out, al, sg, guide_scale, guide_rescale, clamp, percentile)
            kw_i = dict(kwargs)
            if kw_i.get('noise_sampler') is not None:       # injected full-clip noise: use this chunk's frames
                full = kw_i['noise_sampler']
                kw_i['noise_sampler'] = lambda a, b, full=full, s=s, e=e: full(a, b)[:, :, s:e]
            xi = solver_fn(noise[:, :, s:e].clone(), fn, sigmas, variant_info=variant_info,
                           show_progress=show_progress, **kw_i)
            outs.append(xi[:, :, lo:hi])
        b, c, _, h, w = noise.shape
        local = torch.concat(outs, dim=2).to(noise.dtype) if outs else noise.new_empty((b, c, 0, h, w))
        return _all_gather_owned(local, [hi - lo for _, _, lo, hi, *_ in windows], 2)

    # -- sigma <-> t in k-diffusion space (ref :415-443) ---------------------------
    def _log_kd_sigmas(self, like):
        return torch.sqrt(self.sigmas ** 2 / (1 - self.sigmas ** 2)).log().to(like)

    def _sigma_to_t(self, sigma):
        if sigma == float('inf'):
            t = torch.full_like(sigma, len(self.sigmas) - 1)
        else:
            table = self._log_kd_sigmas(sigma)
            ls = sigma.log()
            d = ls - table[:, None]
            lo_idx = d.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=table.shape[0] - 2)
            hi_idx = lo_idx + 1
            lo, hi = table[lo_idx], table[hi_idx]
            wgt = ((lo - ls) / (lo - hi)).clamp(0, 1)
            t = ((1 - wgt) * lo_idx + wgt * hi_idx).view(sigma.shape)
        if t.ndim == 0:
            t = t.unsqueeze(0)
        return t

    def _t_to_sigma(self, t):
        t = t.float()
        lo_idx, hi_idx, wgt = t.floor().long(), t.ceil().long(), t.frac()
        table = self._log_kd_sigmas(t)
        ls = (1 - wgt) * table[lo_idx] + wgt * table[hi_idx]
        ls[torch.isnan(ls) | torch.isinf(ls)] = float('inf')
        return ls.exp()
