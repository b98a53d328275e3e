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
end) -- it only equals the reference for single-chunk inputs.
"""
import random

import torch
import torch.distributed as dist

from ..utils.logger import get_logger
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
        if isinstance(out, tuple):
            x0 = self._guided_x0(out[0], out[1], xt, alphas, sigmas, guide_scale, guide_rescale, clamp, percentile)
        else:
            x0 = self._x0_from_out(xt, alphas, sigmas, out, clamp, percentile)
        eps = (xt - alphas * x0) / sigmas
        mu = coef1 * x0 + coef2 * xt
        return mu, var, log_var, x0, eps

    def _model_out(self, xt, t, model, model_kwargs, guide_scale, variant_info):
        """The model call(s) of one denoise evaluation: the output, or the (conditional, unconditional) pair under CFG."""
        if guide_scale is None:
            assert isinstance(model_kwargs, dict)
            return model(xt, t=t, **model_kwargs)
        assert isinstance(model_kwargs, list)
        pair = getattr(model, "forward_cfg_pair", None)
        if guide_scale != 1.0 and pair is not None and set(model_kwargs[0]) == set(model_kwargs[1]) == {"y"}:
            # the two branches differ only in the text embedding: the model evaluates their common, text-independent
            # prefix once (bit-identical to two calls, tests/test_unet_gpu.py::test_cfg_pair_equals_two_forwards)
            extra = {}
            for kw in model_kwargs[2:]:
                extra.update(kw)
            if len(model_kwargs) <= 3:
                extra["variant_info"] = variant_info
            return pair(xt, t, (model_kwargs[0]["y"], model_kwargs[1]["y"]), **extra)
        y_out = self._branch_out(xt, t, model, model_kwargs, 0, variant_info)
        if guide_scale == 1.0:
            return y_out
        u_out = self._branch_out(xt, t, model, model_kwargs, 1, variant_info)
        return (y_out, u_out)

    @staticmethod
    def _branch_out(xt, t, model, model_kwargs, branch, variant_info):
        """One CFG branch (0 = conditional, 1 = unconditional) of the model call (ref :76-88)."""
        extra = {}
        for kw in model_kwargs[2:]:
            extra.update(kw)
        if len(model_kwargs) <= 3:
            extra["variant_info"] = variant_info
        return model(xt, t=t, **model_kwargs[branch], **extra)

    @staticmethod
    def _x0_from_out(xt, alphas, sigmas, out, clamp=None, percentile=None):
        """v-prediction -> x0 (ref :99).  The reference's dynamic-threshold / clamp options (:100-107) are never
        set by VideoToVideo_sr.test (:110-123) and are not carried over."""
        if clamp is not None or percentile is not None:
            raise NotImplementedError("clamp / percentile are not used on STAR's path (ref video_to_video_model.py:110-123)")
        return alphas * xt - sigmas * out

    def _guided_x0(self, y_out, u_out, xt, alphas, sigmas, guide_scale, guide_rescale, clamp=None, percentile=None):
        """CFG combine + std-ratio rescale + v -> x0 (ref :89-99).  fp16 CUDA model outputs (the .half() UNet) take
        the fused device path -- two launches (star_cfg_x0) instead of ~20 eager tensor ops; anything else (CPU tests,
        fp32 fakes) runs the reference's tensor arithmetic."""
        if y_out.is_cuda and y_out.dtype == torch.float16 and u_out.dtype == torch.float16 and clamp is None \
                and percentile is None:
            from ... import ops
            return ops.cfg_x0(y_out.contiguous(), u_out.contiguous(), xt, alphas, sigmas, guide_scale, guide_rescale)
        return self._x0_from_out(xt, alphas, sigmas, self._guided(y_out, u_out, guide_scale, guide_rescale), clamp, percentile)

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

    # -- sampler ---------------------------------------------------------------
    @torch.no_grad()
    def sample_sr(self, noise, model, model_kwargs={}, condition_fn=None, guide_scale=None,
                  guide_rescale=None, clamp=None, percentile=None, solver='euler_a',
                  solver_mode='fast', steps=20, t_max=None, t_min=None, discretization=None,
                  discard_penultimate_step=None, return_intermediate=None, show_progress=False,
                  seed=-1, chunk_inds=None, variant_info=None, chunk_parallel="auto", tile_inds=None, **kwargs):
        """``tile_inds`` (the output of video_to_video_model.make_tiles) turns on spatially tiled sampling: every solver-step
        evaluation runs the model on each (chunk, tile) window and blends the windows' x0 into the clip's x0 with the tiles'
        weights (see _eval_x0_tiled).  Without it, every path below runs on whole frames."""
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
        if tile_inds is not None and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise NotImplementedError("sample_sr: tiled sampling runs in a single process; spatial tiles are not sharded "
                                      "across ranks")

        intermediates = []
        world, rank = 1, 0
        if chunk_inds is not None and chunk_parallel in ("auto", "exact", "literal") \
                and dist.is_available() and dist.is_initialized():
            world, rank = dist.get_world_size(), dist.get_rank()
        mode = "exact" if chunk_parallel == "auto" else chunk_parallel
        # Ranks of one job must integrate the same SDE path -- also for single-chunk clips, where every rank evaluates the whole
        # clip and the pipeline then shards only the VAE legs: share rank 0's noise seed whenever a process group exists.
        group = (chunk_parallel in ("auto", "exact", "literal") and dist.is_available() and dist.is_initialized()
                 and dist.get_world_size() > 1)
        if group and solver == 'dpmpp_2m_sde' and kwargs.get('noise_sampler') is None:
            # every rank applies the same solver update: share the SDE noise stream (rank 0's seed)
            from .solvers_sdedit import IntervalNoiseSampler
            sd = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).to(noise.device)
            dist.broadcast(sd, 0)
            kwargs['noise_sampler'] = IntervalNoiseSampler(noise, seed=int(sd.item()))

        def eval_x0(xt, sigma, variant_info=None):
            t = self._sigma_to_t(sigma).repeat(len(xt)).round().long()
            x0 = self.denoise(xt, t, None, model, model_kwargs, guide_scale, guide_rescale,
                              clamp, percentile, variant_info=variant_info)[-2]
            if return_intermediate == 'xt':
                intermediates.append(xt)
            elif return_intermediate == 'x0':
                intermediates.append(x0)
            return x0

        keep = stitch_slices(chunk_inds) if chunk_inds is not None else None

        def chunk_inputs(xt, i):
            s, e = chunk_inds[i]
            model_kwargs[2]['hint_chunk'] = model_kwargs[2]['hint'][:, :, s:e].clone()
            return xt[:, :, s:e].clone()

        def chunk_x0(xt, t, i, variant_info):
            """x0 of chunk i, cropped to the slice it contributes (ref :337-350)."""
            x0c = self.denoise(chunk_inputs(xt, i), t, None, model, model_kwargs, guide_scale,
                               guide_rescale, clamp, percentile, variant_info=variant_info)[-2]
            lo, hi = keep[i]
            return x0c[:, :, lo:hi]

        # CFG-branch split (SURVEY 8e): with at least two ranks per chunk the (chunk, branch) pairs are the units --
        # BASELINE config 3 (3 chunks) then fills 6 of 8 GPUs instead of 3.
        split_cfg = (world > 1 and chunk_inds is not None and isinstance(model_kwargs, list)
                     and guide_scale not in (None, 1.0) and world >= 2 * len(chunk_inds)
                     and chunk_parallel in ("auto", "exact"))
        wire = {}

        def eval_x0_chunked(xt, sigma, variant_info=None):
            t = self._sigma_to_t(sigma).repeat(len(xt)).round().long()
            if world == 1:
                parts = [chunk_x0(xt, t, i, variant_info) for i in range(len(chunk_inds))]
                return torch.concat(parts, dim=2)
            if split_cfg:
                return self._eval_x0_cfg_split(xt, t, chunk_inds, keep, chunk_inputs, model, model_kwargs, guide_scale,
                                               guide_rescale, variant_info, world, rank, wire)
            return self._eval_x0_sharded(xt, t, chunk_inds, keep, chunk_x0, variant_info, world, rank)

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

        if tile_inds is not None:
            windows = self._tile_windows(noise, chunk_inds, keep, tile_inds, model_kwargs, guide_scale, clamp, percentile)

            def eval_x0_tiled(xt, sigma, variant_info=None):
                t = self._sigma_to_t(sigma).repeat(len(xt)).round().long()
                x0 = self._eval_x0_tiled(xt, t, windows, model, model_kwargs, guide_scale, guide_rescale, variant_info)
                if return_intermediate == 'xt':
                    intermediates.append(xt)
                elif return_intermediate == 'x0':
                    intermediates.append(x0)
                return x0
            x0 = solver_fn(noise, eval_x0_tiled, sigmas, variant_info=variant_info, show_progress=show_progress, **kwargs)
        elif chunk_inds is not None and world > 1 and mode == "literal":
            x0 = self._sample_literal(noise, solver_fn, sigmas, chunk_inds, keep, model, model_kwargs,
                                      guide_scale, guide_rescale, clamp, percentile, variant_info,
                                      world, rank, show_progress, kwargs)
        else:
            fn = eval_x0_chunked if chunk_inds is not None else eval_x0
            x0 = solver_fn(noise, fn, sigmas, variant_info=variant_info, show_progress=show_progress, **kwargs)
        return (x0, intermediates) if return_intermediate is not None else x0

    # -- spatially tiled sampling ------------------------------------------------
    @staticmethod
    def _tile_windows(noise, chunk_inds, keep, tile_inds, model_kwargs, guide_scale, clamp, percentile):
        """The (chunk, tile) windows of one evaluation: [(s, e, lo, hi, r0, r1, c0, c1, wy, wx)], frames [s, e) of which the
        chunk keeps [lo, hi) (chunk-local), rows [r0, r1), cols [c0, c1), and the tile's weights uploaded once per call."""
        if guide_scale is None or not isinstance(model_kwargs, list) or len(model_kwargs) < 3 \
                or 'hint' not in model_kwargs[2]:
            raise ValueError("sample_sr(tile_inds=...): tiled sampling needs classifier-free guidance (guide_scale) and "
                             "model_kwargs [{'y': ...}, {'y': ...}, {'hint': ...}]")
        if clamp is not None or percentile is not None:
            raise NotImplementedError("sample_sr(tile_inds=...): clamp / percentile are not supported")
        rows, cols, row_w, col_w = tile_inds
        f = noise.shape[2]
        chunks = chunk_inds if chunk_inds is not None else [(0, f)]
        kept = keep if keep is not None else [(0, f)]
        row_w = [w.to(noise.device, torch.float32).contiguous() for w in row_w]
        col_w = [w.to(noise.device, torch.float32).contiguous() for w in col_w]
        return [(s, e, lo, hi, r0, r1, c0, c1, wy, wx)
                for (s, e), (lo, hi) in zip(chunks, kept)
                for (r0, r1), wy in zip(rows, row_w)
                for (c0, c1), wx in zip(cols, col_w)]

    def _eval_x0_tiled(self, xt, t, windows, model, model_kwargs, guide_scale, guide_rescale, variant_info):
        """x0 of the clip = sum over (chunk, tile) windows of the tile's blend weight times its x0, restricted to the frames
        the chunk keeps (stitch_slices).  Each window runs the model on the cropped latent and LR latent, with the branch
        logic of ``denoise``; one star_cfg_x0_blend launch pair per window forms the guided x0 (CFG, std-ratio rescale over
        the window, v -> x0) and adds it into the clip's x0 in place.  Needs fp16 CUDA model outputs (the .half() UNet)."""
        from ... import ops
        xt = xt.float().contiguous()
        x0 = torch.zeros_like(xt)
        alphas, sigmas = _gather_coef(self.alphas, t, xt), _gather_coef(self.sigmas, t, xt)
        hint = model_kwargs[2]['hint']                                    # the clip's LR latent; each window gets its crop
        rescale = None if guide_scale == 1.0 else guide_rescale        # as denoise: no rescale without a second branch
        for s, e, lo, hi, r0, r1, c0, c1, wy, wx in windows:
            kw = [model_kwargs[0], model_kwargs[1],
                  dict(model_kwargs[2], hint_chunk=hint[:, :, s:e, r0:r1, c0:c1].contiguous())] + list(model_kwargs[3:])
            out = self._model_out(xt[:, :, s:e, r0:r1, c0:c1].contiguous(), t, model, kw, guide_scale, variant_info)
            y_out, u_out = out if isinstance(out, tuple) else (out, out)
            if not (y_out.is_cuda and y_out.dtype == torch.float16 and u_out.dtype == torch.float16):
                raise TypeError("sample_sr(tile_inds=...): tiled sampling blends on the GPU and needs fp16 CUDA model outputs "
                                f"(the .half() UNet), got {y_out.dtype} on {y_out.device}")
            ops.cfg_x0(y_out.contiguous(), u_out.contiguous(), xt, alphas, sigmas, guide_scale, rescale,
                       blend=ops.TileBlend(x0, s, lo, hi, r0, c0, wy, wx))
        return x0

    # -- chunk-parallel helpers -------------------------------------------------
    @staticmethod
    def _eval_x0_sharded(xt, t, chunk_inds, keep, chunk_x0, variant_info, world, rank):
        """Exact mode: rank r evaluates chunks r, r+W, ...; one all-gather of the
        kept slices (padded to the longest per-rank payload) rebuilds the
        stitched x0 on every rank."""
        n = len(chunk_inds)
        owner = [i % world for i in range(n)]
        lens = [hi - lo for lo, hi in keep]
        per_rank = [sum(l for l, o in zip(lens, owner) if o == r) for r in range(world)]
        pad = max(per_rank)
        mine = [chunk_x0(xt, t, i, variant_info) for i in range(n) if owner[i] == rank]
        b, c, _, h, w = xt.shape
        send = xt.new_zeros((b, c, pad, h, w))
        if mine:
            cat = torch.concat(mine, dim=2)
            send[:, :, :cat.shape[2]] = cat.to(send.dtype)
        recv = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(recv, send.contiguous())
        cursor = [0] * world
        parts = []
        for i in range(n):
            r = owner[i]
            parts.append(recv[r][:, :, cursor[r]:cursor[r] + lens[i]])
            cursor[r] += lens[i]
        return torch.concat(parts, dim=2)

    def _eval_x0_cfg_split(self, xt, t, chunk_inds, keep, chunk_inputs, model, model_kwargs, guide_scale, guide_rescale,
                           variant_info, world, rank, wire):
        """Exact mode with two ranks per chunk: rank 2i evaluates the conditional branch of chunk i, rank 2i+1 the
        unconditional one (ranks >= 2n idle).  ONE all-gather of the raw model outputs per solver step; every rank
        then forms the guided output (needs both branches: std-ratio rescale, ref :89-97), x0 and the stitch for all
        chunks -- elementwise work on a few MB, identical on every rank and to the serial loop."""
        n = len(chunk_inds)
        lens = [e - s for s, e in chunk_inds]
        b, c, _, h, w = xt.shape
        out = None
        if rank < 2 * n:
            i, branch = divmod(rank, 2)
            out = self._branch_out(chunk_inputs(xt, i), t, model, model_kwargs, branch, variant_info)
        if "dtype" not in wire:                      # the model's output dtype (fp16 for the .half() UNet), agreed once
            codes = [torch.float16, torch.bfloat16, torch.float32, torch.float64]
            code = torch.tensor([codes.index(out.dtype) if out is not None else 0], device=xt.device)
            dist.broadcast(code, 0)
            wire["dtype"] = codes[int(code.item())]
        send = torch.zeros((b, c, max(lens), h, w), dtype=wire["dtype"], device=xt.device)
        if out is not None:
            send[:, :, :out.shape[2]] = out
        recv = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(recv, send)
        sig = _gather_coef(self.sigmas, t, xt)
        alp = _gather_coef(self.alphas, t, xt)
        parts = []
        for i, (s, e) in enumerate(chunk_inds):
            y_out, u_out = recv[2 * i][:, :, :lens[i]], recv[2 * i + 1][:, :, :lens[i]]
            x0c = self._guided_x0(y_out, u_out, xt[:, :, s:e], alp, sig, guide_scale, guide_rescale)
            lo, hi = keep[i]
            parts.append(x0c[:, :, lo:hi])
        return torch.concat(parts, dim=2)

    def _sample_literal(self, noise, solver_fn, sigmas, chunk_inds, keep, model, model_kwargs, guide_scale,
                        guide_rescale, clamp, percentile, variant_info, world, rank, show_progress, kwargs):
        """North-star literal mode: every rank integrates its own chunk(s) for
        all solver steps with no exchange; kept slices are gathered once."""
        n = len(chunk_inds)
        b, c, f, h, w = noise.shape
        lens = [hi - lo for lo, hi in keep]
        owner = [i % world for i in range(n)]
        per_rank = [sum(l for l, o in zip(lens, owner) if o == r) for r in range(world)]
        pad = max(per_rank)
        outs = []
        for i in range(n):
            if owner[i] != rank:
                continue
            s, e = chunk_inds[i]
            kw = [model_kwargs[0], model_kwargs[1], {'hint': model_kwargs[2]['hint'][:, :, s:e].clone()}]

            def fn(xt, sigma, variant_info=None, kw=kw):
                t = self._sigma_to_t(sigma).repeat(len(xt)).round().long()
                return self.denoise(xt, t, None, model, kw, guide_scale, guide_rescale, clamp, percentile,
                                    variant_info=variant_info)[-2]
            kw_i = dict(kwargs)
            if kw_i.get('noise_sampler') is not None:       # injected full-clip noise: use this chunk's frames
                full = kw_i['noise_sampler']
                kw_i['noise_sampler'] = lambda a, b, full=full, s=s, e=e: full(a, b)[:, :, s:e]
            xi = solver_fn(noise[:, :, s:e].clone(), fn, sigmas, variant_info=variant_info,
                           show_progress=show_progress, **kw_i)
            lo, hi = keep[i]
            outs.append(xi[:, :, lo:hi])
        send = noise.new_zeros((b, c, pad, h, w))
        if outs:
            cat = torch.concat(outs, dim=2)
            send[:, :, :cat.shape[2]] = cat
        recv = [torch.empty_like(send) for _ in range(world)]
        dist.all_gather(recv, send.contiguous())
        cursor = [0] * world
        parts = []
        for i in range(n):
            r = owner[i]
            parts.append(recv[r][:, :, cursor[r]:cursor[r] + lens[i]])
            cursor[r] += lens[i]
        return torch.concat(parts, dim=2)

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
