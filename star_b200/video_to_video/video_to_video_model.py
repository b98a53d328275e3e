"""Pipeline entry of STAR video super-resolution on star_b200.

Mirrors ``VideoToVideo_sr`` of the reference's video_to_video/video_to_video_model.py
(:20-139: constructor, ``test``; :141-161 VAE helpers; :164-210 ``pad_to_fit`` /
``make_chunks`` / ``sliding_windows_1d``).  What differs:

* the denoiser is star_b200's ``ControlledV2VUNet`` (sm_90a kernels), not autocast PyTorch;
* the diffusion block of ``test`` (ref :98-123) is factored into ``denoise_latents`` so that
  the latent-in / latent-out hot path can be driven (and benchmarked) without the VAE;
* the temporal VAE is star_b200's own ``AutoencoderKLTemporalDecoder`` (modules/temporal_vae.py, same
  checkpoint layout as diffusers', sm_90a kernels), loaded from ``opt.vae_path`` (no hub download);
* the text encoder (open_clip) is an un-vendored third-party package: it is imported lazily, and
  ready-made objects can be injected (``text_encoder=``, ``vae=``, ``generator=``), which is how the
  tests and the benchmark run on boxes without those packages or checkpoints;
* the LR frames are uploaded, upsampled and encoded one at a time, and ``enhance_frames_iter`` yields the finished frames one
  3-frame decode window at a time, so in a single process the device memory of a clip grows only by its latents;
* with ``torch.distributed`` initialised (one process per GPU) the whole entry is sharded (SURVEY 8e):
  - each rank uploads, upsamples and VAE-encodes only its contiguous share of the frames; the latents (0.42 MB per
    frame) are all-gathered, so every rank conditions on the SAME posterior sample (the reference draws it once);
  - frame chunks -- or (chunk, CFG branch) pairs when there are at least two ranks per chunk, or (chunk, spatial tile)
    windows with ``tile_size`` -- are sharded across ranks with all-gathers every solver step
    (diffusion_sdedit.GaussianDiffusion.sample_sr, ``chunk_parallel``);
  - test() decodes each rank's share of the 3-frame VAE windows and ONE all-gather of the decoded, cropped frames
    assembles the clip (the north-star's end collective); enhance_frames decodes and colour-corrects the windows in
    rounds of one window per rank, with one all-gather of the finished frames per round.
"""
from typing import Any, Dict

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import ops
from .diffusion.diffusion_sdedit import GaussianDiffusion
from .diffusion.schedules_sdedit import noise_schedule
from .modules.unet_v2v import ControlledV2VUNet, rearrange
from .utils.config import cfg
from .utils.logger import get_logger
from .utils.sharding import _all_gather_owned, _all_gather_varlen, _dist_info, _shard_bounds

logger = get_logger()

__all__ = ["VideoToVideo_sr", "pad_to_fit", "make_chunks", "make_tiles", "sliding_windows_1d"]


class VideoToVideo_sr():
    def __init__(self, opt, device=torch.device('cuda:0'), text_encoder=None, vae=None, generator=None, cuda_graph=False):
        self.opt = opt
        self.device = device
        self.cuda_graph = cuda_graph           # serve the denoiser's CFG-pair call from CUDA graphs (launch-bound small latents)

        if text_encoder is None:
            from .modules.embedder import FrozenOpenCLIPEmbedder
            # local files instead of the open_clip package when the options name them (weights: open_clip_pytorch_model.bin of
            # laion/CLIP-ViT-H-14-laion2B-s32B-b79K, merges: open_clip's bpe_simple_vocab_16e6.txt.gz)
            text_encoder = FrozenOpenCLIPEmbedder(device=self.device, pretrained="laion2b_s32b_b79k",
                                                  weights_path=getattr(opt, "clip_weights_path", None),
                                                  bpe_path=getattr(opt, "clip_bpe_path", None))
            text_encoder.model.to(self.device)
            logger.info('Build encoder with FrozenOpenCLIPEmbedder')
        self.text_encoder = text_encoder

        if generator is None:
            generator = ControlledV2VUNet().to(self.device).eval()
            cfg.model_path = opt.model_path
            load_dict = torch.load(cfg.model_path, map_location='cpu')
            if 'state_dict' in load_dict:
                load_dict = load_dict['state_dict']
            ret = generator.load_state_dict(load_dict, strict=False)
            logger.info('Load model path {}, with local status {}'.format(cfg.model_path, ret))
        self.generator = generator.half()
        self._graphed = None

        sigmas = noise_schedule(schedule='logsnr_cosine_interp', n=1000, zero_terminal_snr=True,
                                scale_min=2.0, scale_max=4.0)
        self.diffusion = GaussianDiffusion(sigmas=sigmas)

        if vae is None:
            # ref :57-63 downloads stabilityai/stable-video-diffusion-img2vid (subfolder vae, variant fp16) through
            # diffusers; here the same checkpoint is read from a local snapshot into the sm_90a temporal VAE.
            from .modules.temporal_vae import AutoencoderKLTemporalDecoder
            vae_path = _find_vae_dir(opt)
            if vae_path is None:
                raise ValueError("VideoToVideo_sr: no temporal-VAE weights found -- pass opt.vae_path, set STAR_VAE_PATH or "
                                 "keep the snapshot the reference downloads (stabilityai/stable-video-diffusion-img2vid, "
                                 "subfolder vae) in the Hugging Face cache; or pass vae=...  (denoise_latents() needs neither)")
            vae = AutoencoderKLTemporalDecoder.from_pretrained(vae_path, variant="fp16")
            vae.eval()
            vae.requires_grad_(False)
            vae.to(self.device)
        self.vae = vae

        self.negative_prompt = cfg.negative_prompt
        self.positive_prompt = cfg.positive_prompt
        self.negative_y = self._encode_text(self.negative_prompt)

    def _encode_text(self, y):
        """str -> (1,77,1024) via the text encoder; tensors pass through (precomputed embedding)."""
        if torch.is_tensor(y):
            return y.to(self.device)
        return self.text_encoder(y).detach()

    # -- latent-space hot path (ref :98-123) ------------------------------------------------------
    @torch.no_grad()
    def denoise_latents(self, video_data_feature, y, negative_y=None, total_noise_levels=1000, steps=50,
                        solver_mode='fast', guide_scale=7.5, max_chunk_len=32, noise=None, noise_sampler=None,
                        chunk_parallel="auto", tile_size=None, tile_overlap=16):
        """video_data_feature: (1,4,F,h,w) VAE latent of the upsampled LR clip (any device; moved to
        self.device), y / negative_y: (1,77,1024).  Returns the denoised latent (1,4,F,h,w) fp32 on
        self.device.  ``noise`` / ``noise_sampler`` pin the two random inputs (diffuse noise, SDE noise).

        ``tile_size = (th, tw)`` (latent units, th = 2 and tw = 0 mod 8) denoises overlapping spatial tiles of
        ``tile_overlap`` latent pixels and blends their x0 at every solver step (make_tiles), so that the memory and
        attention cost of a step depend on the tile, not the frame.  It approximates the untiled result (GroupNorm
        statistics, attention context and the CFG rescale become per tile) and is never switched on by itself."""
        feat = self._upload_frames(video_data_feature)
        y = y.to(self.device)
        negative_y = (self.negative_y if negative_y is None else negative_y).to(self.device)
        frames_num = feat.shape[2]
        t = torch.LongTensor([total_noise_levels - 1]).to(self.device)
        noised_lr = self.diffusion.diffuse(feat, t, noise=noise).contiguous()
        if noise is None and torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            torch.distributed.broadcast(noised_lr, 0)       # chunk-parallel ranks start from the same sample
        model_kwargs = [{'y': y}, {'y': negative_y}, {'hint': feat}]
        chunk_inds = make_chunks(frames_num, interp_f_num=0, max_chunk_len=max_chunk_len) \
            if frames_num > max_chunk_len else None
        extra = {} if noise_sampler is None else {'noise_sampler': noise_sampler}
        if tile_size is not None:
            extra['tile_inds'] = make_tiles(feat.shape[3], feat.shape[4], tile_size, tile_overlap)
        model = self.generator
        if self.cuda_graph and hasattr(model, "forward_cfg_pair"):
            if self._graphed is None:
                from .cuda_graph import GraphedCFGPair
                self._graphed = GraphedCFGPair(self.generator)
            model = self._graphed
        return self.diffusion.sample_sr(
            noise=noised_lr, model=model, model_kwargs=model_kwargs, guide_scale=guide_scale,
            guide_rescale=0.2, solver='dpmpp_2m_sde', solver_mode=solver_mode, return_intermediate=None,
            steps=steps, t_max=total_noise_levels - 1, t_min=0, discretization='trailing',
            chunk_inds=chunk_inds, chunk_parallel=chunk_parallel, **extra)

    def _upload_frames(self, x, dim=2):
        """Host tensor -> fp32 on self.device.  Under torch.distributed every rank uploads only its share of the
        frames over its own PCIe link and the shares are all-gathered over NVLink (instead of W full uploads)."""
        world, rank = _dist_info()
        if x.is_cuda or world == 1 or x.shape[dim] < world:
            return x.to(self.device, torch.float32)
        bounds = _shard_bounds(x.shape[dim], world)
        lo, hi = bounds[rank]
        local = x.narrow(dim, lo, hi - lo).contiguous().to(self.device, torch.float32)
        return _all_gather_varlen(local, [b - a for a, b in bounds], dim)

    # -- pixel-space entry (ref :75-139) ------------------------------------------------------------
    @torch.no_grad()
    def test(self, input: Dict[str, Any], total_noise_levels=1000, steps=50, solver_mode='fast', guide_scale=7.5,
             max_chunk_len=32, tile_size=None, tile_overlap=16):
        """The reference entry (ref :75-139): (1, 3, F, H, W) fp32 on the CPU.  tile_size / tile_overlap: denoise_latents."""
        return self._test_on_device(input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len,
                                    tile_size, tile_overlap).type(torch.float32).cpu()

    @torch.no_grad()
    def enhance_frames(self, input: Dict[str, Any], total_noise_levels=1000, steps=50, solver_mode='fast', guide_scale=7.5,
                       max_chunk_len=32, uint8=True, tile_size=None, tile_overlap=16):
        """test() + the CLI's post-processing (inference_sr.py:77-80: tensor2vid, adain_color_fix against the LR clip) with the
        post-processing on the GPU: returns (F, H, W, 3) frames in [0, 255] on the CPU -- uint8 by default, i.e. a quarter of the
        device->host traffic of test()'s fp32 tensor.  In a single process the frames come from enhance_frames_iter.  Under a
        process group of W > 1 ranks the 3-frame decode windows run in rounds of W: in round k rank r decodes, crops and
        colour-corrects window k * W + r, and one all-gather of the finished frames per round fills every rank's host tensor.
        Either way the device holds no whole-clip tensor at output resolution."""
        world, rank = _dist_info()
        (h, w) = input['target_res']
        out = torch.empty((input['video_data'].shape[0], h, w, 3), dtype=torch.uint8 if uint8 else torch.float32)
        if world == 1:
            for s, frames in self.enhance_frames_iter(input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len,
                                                      uint8, tile_size, tile_overlap):
                out[s:s + frames.shape[0]] = frames
            return out
        if torch.device(self.device).type != 'cuda':
            raise NotImplementedError("enhance_frames runs the GPU post-processing kernels; use test() + the reference's CPU "
                                      "helpers otherwise")
        gen_vid, (w1, _, h1, _) = self._sample_latents(input, total_noise_levels, steps, solver_mode, guide_scale,
                                                       max_chunk_len, tile_size, tile_overlap)
        z = rearrange(gen_vid, "b c f h w -> (b f) c h w")
        n, chunk_size = z.shape[0], 3
        starts = list(range(0, n, chunk_size))
        for k in range(0, len(starts), world):
            rnd = starts[k:k + world]
            if rank < len(rnd):
                s = rnd[rank]
                local = self._enhance_window(z, input['video_data'], s, min(chunk_size, n - s), (h1, h + h1, w1, w + w1),
                                             uint8)
            else:
                local = torch.empty((0, h, w, 3), dtype=out.dtype, device=self.device)
            frames = _all_gather_owned(local, [min(chunk_size, n - s) for s in rnd], 0)
            out[rnd[0]:rnd[0] + frames.shape[0]] = frames
        return out

    def enhance_frames_iter(self, input: Dict[str, Any], total_noise_levels=1000, steps=50, solver_mode='fast', guide_scale=7.5,
                            max_chunk_len=32, uint8=True, tile_size=None, tile_overlap=16):
        """enhance_frames as a generator of (start, frames) in clip order, one 3-frame VAE decode window at a time: frames
        (k, H, W, 3) of the clip's frames [start, start + k) on the CPU (pinned), uint8 or fp32 in [0, 255], owned by the caller.

        The LR frames are encoded one at a time and the denoised latent is decoded, cropped and colour-corrected one window at
        a time, so the device memory a clip needs grows only by its fp32 latents (0.42 MB per frame each at 240p -> 960p).  The frames
        equal enhance_frames' byte for byte.  The next window is decoded on the GPU while the caller handles the current one.
        Single process only: under a process group of more than one rank use enhance_frames."""
        if _dist_info()[0] > 1:
            raise NotImplementedError("enhance_frames_iter runs in a single process; under torch.distributed with more than one "
                                      "rank use enhance_frames, which shards the decode across the ranks")
        if torch.device(self.device).type != 'cuda':
            raise NotImplementedError("enhance_frames_iter runs the GPU post-processing kernels; use test() + the reference's "
                                      "CPU helpers otherwise")
        return self._enhanced_windows(input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len, uint8,
                                      tile_size, tile_overlap)

    @torch.no_grad()
    def _enhanced_windows(self, input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len, uint8, tile_size,
                          tile_overlap, chunk_size=3):
        video_data = input['video_data']
        (h, w) = input['target_res']
        gen_vid, (w1, _, h1, _) = self._sample_latents(input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len,
                                                       tile_size, tile_overlap)
        z = rearrange(gen_vid, "b c f h w -> (b f) c h w")
        n = z.shape[0]
        stream = torch.cuda.current_stream(self.device)

        def launch(s):
            """enqueue window [s, s + k) (_enhance_window) and its copy into a fresh pinned host tensor; returns (s, host
            tensor, device result, its copy's event)"""
            out = self._enhance_window(z, video_data, s, min(chunk_size, n - s), (h1, h + h1, w1, w + w1), uint8)
            host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
            host.copy_(out, non_blocking=True)
            done = torch.cuda.Event()
            done.record(stream)
            return s, host, out, done

        pending = launch(0) if n else None
        try:
            while pending is not None:
                s, host, staged, done = pending
                pending = launch(s + chunk_size) if s + chunk_size < n else None
                done.synchronize()
                del staged                     # held until its copy to `host` has completed
                yield s, host
        finally:
            stream.synchronize()              # a caller that stops early leaves no work in flight

    def _enhance_window(self, z, video_data, s, k, crop, uint8):
        """Frames [s, s + k) of the clip, finished on the device: LR upload, decode of the latent frames z[s:s + k] ((b f) c h
        w; the windows and autocast of _test_on_device), crop (t0, t1, l0, l1), colour fix against the LR frames.  Returns
        (k, H, W, 3) in [0, 255], uint8 or fp32."""
        t0, t1, l0, l1 = crop
        lr = self._upload_lr(video_data[s:s + k]).float()
        with torch.autocast('cuda'):
            dec = self.temporal_vae_decode(z[s:s + k], k)
        vid = dec[:, :, t0:t1, l0:l1].permute(1, 0, 2, 3).unsqueeze(0).float()
        return ops.adain_color_fix(vid, lr, uint8=uint8)

    def _upload_lr(self, frames):
        """LR frames -> self.device.  A host tensor goes through pinned memory so that the copy is queued behind the work
        already on the stream instead of waiting for it on the host."""
        if frames.device.type == 'cpu' and torch.device(self.device).type == 'cuda':
            frames = frames.pin_memory()
        return frames.to(self.device, non_blocking=True)

    def _encode_frames(self, frames, target_h, target_w, padding):
        """LR frames (n, 3, h, w) -> their VAE latent (1, 4, n, H/8, W/8) on self.device, one frame at a time: upload,
        upsample_pad, vae_encode (posterior sample times the scaling factor), written into the clip's latent.  Only one
        canvas-sized frame exists at a time.  vae_encode draws one posterior sample per frame, like the reference (ref :141-161),
        so the random draws and the latent are those of encoding the whole upsampled clip."""
        n = frames.shape[0]
        feat = None
        for i in range(n):
            z = self.vae_encode(self.upsample_pad(self._upload_lr(frames[i:i + 1]), target_h, target_w, padding).unsqueeze(0))
            if feat is None:
                feat = z.new_empty((1, z.shape[1], n, *z.shape[3:]))
            feat[:, :, i:i + 1] = z
        if feat is None:
            w1, w2, h1, h2 = padding
            feat = torch.zeros((1, 4, 0, (target_h + h1 + h2) // 8, (target_w + w1 + w2) // 8), device=self.device)
        return feat

    def _sample_latents(self, input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len, tile_size=None,
                        tile_overlap=16):
        """encode (this rank's share of the frames, latents all-gathered) + denoise_latents: (denoised latent, padding)"""
        video_data = input['video_data']
        (target_h, target_w) = input['target_res']
        world, rank = _dist_info()
        frames_num = video_data.shape[0]
        bounds = _shard_bounds(frames_num, world)
        lo, hi = bounds[rank]
        padding = pad_to_fit(target_h, target_w)
        logger.info(f'video_data shape: {(frames_num, video_data.shape[1], target_h, target_w)}')
        feat_local = self._encode_frames(video_data[lo:hi], target_h, target_w, padding)
        video_data_feature = feat_local if world == 1 else \
            _all_gather_varlen(feat_local.float(), [b - a for a, b in bounds], 2)
        del feat_local
        y = self._encode_text(input['y'])
        tiles = {} if tile_size is None else {'tile_size': tile_size, 'tile_overlap': tile_overlap}
        gen_vid = self.denoise_latents(video_data_feature, y, None, total_noise_levels, steps, solver_mode,
                                       guide_scale, max_chunk_len, **tiles)
        logger.info('sampling, finished.')
        return gen_vid, padding

    def _test_on_device(self, input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len, tile_size=None,
                        tile_overlap=16):
        (h, w) = input['target_res']
        bs = 1
        gen_vid, padding = self._sample_latents(input, total_noise_levels, steps, solver_mode, guide_scale, max_chunk_len,
                                                tile_size, tile_overlap)
        world, _ = _dist_info()
        w1, w2, h1, h2 = padding
        with torch.autocast('cuda', enabled=torch.cuda.is_available()):
            if world == 1:
                vid_tensor_gen = self.vae_decode_chunk(gen_vid, chunk_size=3)[:, :, h1:h + h1, w1:w + w1]
            else:
                vid_tensor_gen = self._decode_sharded(gen_vid, 3, (h1, h + h1, w1, w + w1))
        logger.info('temporal vae decoding, finished.')
        return rearrange(vid_tensor_gen, '(b f) c h w -> b c f h w', b=bs)

    def upsample_pad(self, frames, target_h, target_w, padding):
        """(f,3,h,w) -> bilinear resize to (target_h, target_w) (F.interpolate semantics, align_corners=False) and
        constant-1 padding (w1, w2, h1, h2), ref :81-87 -- one kernel on the GPU, eager torch for CPU tensors."""
        if frames.is_cuda:
            return ops.bilinear_pad(frames.float(), target_h, target_w, padding, 1.0)
        return F.pad(F.interpolate(frames, [target_h, target_w], mode='bilinear'), padding, 'constant', 1)

    def _decode_sharded(self, z, chunk_size, crop):
        """3-frame VAE windows (ref :144-151) round-robin over the ranks; ONE all-gather of the decoded, cropped
        frames.  Window w covers frames [3w, 3w+3) of the full clip on every rank, so the windows -- and therefore
        the decoder's per-window GroupNorm / temporal-conv context -- are exactly the single-GPU ones."""
        world, rank = _dist_info()
        t0, t1, l0, l1 = crop
        zf = rearrange(z, "b c f h w -> (b f) c h w")
        n = zf.shape[0]
        starts = list(range(0, n, chunk_size))
        mine = starts[rank::world]
        outs = [self.temporal_vae_decode(zf[s:s + chunk_size], min(chunk_size, n - s))[:, :, t0:t1, l0:l1] for s in mine]
        if outs:
            local = torch.cat(outs)
        else:
            local = torch.zeros((0, 3, t1 - t0, l1 - l0), device=self.device, dtype=torch.float16)
        dtype_code = torch.tensor([0 if local.dtype == torch.float16 else 1], device=self.device)
        dist.all_reduce(dtype_code, op=dist.ReduceOp.MAX)
        local = local.to(torch.float16 if int(dtype_code.item()) == 0 else torch.float32)
        return _all_gather_owned(local, [min(chunk_size, n - s) for s in starts], 0)

    # -- VAE helpers (ref :141-161): exact 3-frame decode windows, 1-frame encode ----------------------
    def temporal_vae_decode(self, z, num_f):
        return self.vae.decode(z / self.vae.config.scaling_factor, num_frames=num_f).sample

    def vae_decode_chunk(self, z, chunk_size=3):
        z = rearrange(z, "b c f h w -> (b f) c h w")
        video = []
        for ind in range(0, z.shape[0], chunk_size):
            num_f = z[ind:ind + chunk_size].shape[0]
            video.append(self.temporal_vae_decode(z[ind:ind + chunk_size], num_f))
        return torch.cat(video)

    def vae_encode(self, t, chunk_size=1):
        num_f = t.shape[1]
        t = rearrange(t, "b f c h w -> (b f) c h w")
        z_list = []
        for ind in range(0, t.shape[0], chunk_size):
            z_list.append(self.vae.encode(t[ind:ind + chunk_size]).latent_dist.sample())
        z = rearrange(torch.cat(z_list, dim=0), "(b f) c h w -> b c f h w", f=num_f)
        return z * self.vae.config.scaling_factor


def _find_vae_dir(opt):
    """opt.vae_path / cfg.vae_path / $STAR_VAE_PATH, else the snapshot the reference's from_pretrained call (ref :57-59)
    leaves in the Hugging Face cache -- so that the reference's unmodified CLI, which only sets model_path, keeps working."""
    import glob
    import os
    for cand in (getattr(opt, 'vae_path', None), getattr(cfg, 'vae_path', None), os.environ.get('STAR_VAE_PATH')):
        if cand:
            return cand
    hub = os.environ.get('HF_HUB_CACHE') or os.path.join(os.environ.get('HF_HOME', os.path.expanduser('~/.cache/huggingface')), 'hub')
    hits = sorted(glob.glob(os.path.join(hub, 'models--stabilityai--stable-video-diffusion-img2vid', 'snapshots', '*', 'vae')))
    return hits[-1] if hits else None


def _centre_pad(size, target):
    lo = int((target - size) // 2)
    return lo, target - lo - size


def pad_to_fit(h, w):
    """(w1, w2, h1, h2) for F.pad (ref :164-187): small inputs are centred in 720x1280; larger ones
    are padded bottom/right so that H = 16 (mod 64) and W = 0 (mod 64) -> latent H = 2 (mod 8)."""
    best_h, best_w = 720, 1280
    if h < best_h:
        h1, h2 = _centre_pad(h, best_h)
    elif h == best_h:
        h1 = h2 = 0
    else:
        h1, h2 = 0, int((h + 48) // 64 * 64) + 64 - 48 - h
    if w < best_w:
        w1, w2 = _centre_pad(w, best_w)
    elif w == best_w:
        w1 = w2 = 0
    else:
        w1, w2 = 0, int(w // 64 * 64) + 64 - w
    return (w1, w2, h1, h2)


def sliding_windows_1d(length, window_size, overlap_size):
    """Windows of ``window_size`` with stride window-overlap; the last window absorbs the remainder
    when fewer than 1.25 windows are left (ref :199-210)."""
    stride = window_size - overlap_size
    coords, ind = [], 0
    while ind < length:
        if ind + window_size * 1.25 >= length:
            coords.append((ind, length))
            break
        coords.append((ind, ind + window_size))
        ind += stride
    return coords


def make_chunks(f_num, interp_f_num, max_chunk_len, chunk_overlap_ratio=0.5):
    """Chunk index list for a clip of f_num frames (ref :190-196)."""
    max_o_len = max_chunk_len * chunk_overlap_ratio
    chunk_len = int((max_chunk_len - 1) // (1 + interp_f_num) * (interp_f_num + 1) + 1)
    o_len = int((max_o_len - 1) // (1 + interp_f_num) * (interp_f_num + 1) + 1)
    return sliding_windows_1d(f_num, chunk_len, o_len)


def _tile_axis(length, tile, overlap):
    """Tile ranges along one axis and their blend weights (fp64 ramps, normalised to a partition of unity)."""
    if length <= tile:
        return [(0, length)], [torch.ones(length, dtype=torch.float64)]
    n = -(-(length - tile) // (tile - overlap)) + 1
    starts = [k * (length - tile) // (n - 1) for k in range(n)]        # even spread: consecutive tiles overlap >= `overlap`
    ramp = torch.arange(1, tile + 1, dtype=torch.float64) / (overlap + 1)
    raw = []
    for k in range(n):
        w = torch.ones(tile, dtype=torch.float64)
        if k > 0:                                                        # inner edges only: no ramp at the frame's border
            w = torch.minimum(w, ramp)
        if k < n - 1:
            w = torch.minimum(w, ramp.flip(0))
        raw.append(w)
    total = torch.zeros(length, dtype=torch.float64)
    for s, w in zip(starts, raw):
        total[s:s + tile] += w
    return [(s, s + tile) for s in starts], [w / total[s:s + tile] for s, w in zip(starts, raw)]


def make_tiles(h, w, tile_size, overlap=16):
    """Spatial tiles of an h x w latent for tiled sampling (``GaussianDiffusion.sample_sr(tile_inds=...)``).

    tile_size = (th, tw) in latent units, with th = 2 (mod 8) and tw = 0 (mod 8) so that the UNet's down/up-sampling closes
    on every tile; an axis no longer than its tile is one tile of the full extent.  Along an axis of length L > T there are
    ceil((L - T) / (T - overlap)) + 1 tiles of size T whose starts are spread evenly over [0, L - T], so neighbours overlap
    by at least `overlap`.  Every tile has the same shape (one CUDA graph per chunk length).

    Returns (row_ranges, col_ranges, row_weights, col_weights): [(start, end)] per axis and, per tile, fp32 CPU weights of its
    extent.  A tile's raw weight ramps linearly over `overlap` pixels up from each inner edge (none at the frame's border) and
    is divided by the sum over all tiles covering the pixel: the weights along an axis sum to 1, a pixel covered by one tile
    has weight exactly 1.0, and the 2-D weight of tile (i, j) at (r, c) is row_weights[i][r] * col_weights[j][c]."""
    th, tw = (int(v) for v in tile_size)
    if th <= 0 or tw <= 0 or th % 8 != 2 or tw % 8 != 0:
        raise ValueError(f"tile size {th}x{tw}: the tile height must be 2 (mod 8) and the width 0 (mod 8), both positive, "
                         "for the UNet's down/up-sampling to close")
    overlap = int(overlap)
    if not (0 <= overlap < min(th, tw)):
        raise ValueError(f"tile overlap {overlap} outside [0, {min(th, tw)}) for tiles of {th}x{tw}")
    rows, row_w = _tile_axis(int(h), th, overlap)
    cols, col_w = _tile_axis(int(w), tw, overlap)
    return rows, cols, [v.float() for v in row_w], [v.float() for v in col_w]
