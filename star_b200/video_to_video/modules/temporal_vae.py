"""Temporal VAE (SVD `AutoencoderKLTemporalDecoder`) on the sm_90a kernels -- SURVEY rows a3 / a16.

The reference builds this module from diffusers (video_to_video/video_to_video_model.py:57-63) and uses exactly
three things of it (:141-161): ``vae.config.scaling_factor``, ``vae.encode(x).latent_dist.sample()`` per frame and
``vae.decode(z, num_frames=n).sample`` on 3-frame windows.  This class offers that surface and the checkpoint's
parameter tree (same keys and shapes as diffusers 0.30.0, so ``diffusion_pytorch_model*.safetensors`` loads with
``load_state_dict``); ``nn`` only stores the parameters.  Execution keeps every activation as an fp16 token matrix
X[(frame h w), C] and is a sequence of C-ABI calls (star_b200/ops.py):

* all 3x3 / (3,1,1) / 1x1 convolutions -> wgmma implicit GEMM with bias + residual epilogues; the stride-2
  encoder convs (F.pad (0,1,0,1) + stride 2) through the parity-plane split; stems with Cin <= 4 through im2col;
* GroupNorm(+SiLU) -> the two-pass GroupNorm kernels, per frame for the spatial blocks, per clip for the temporal ones;
* AlphaBlender: out = a*x_s + (1-a)*(x_s + h) = x_s + sigmoid(mix_factor)*h, i.e. the second temporal conv with its
  weights pre-scaled by sigmoid(mix_factor) and x_s as the residual operand -- no blend kernel;
* the single-head (d = C = 512) mid-block attention as three GEMMs around a row-softmax kernel (S = Q K^T with
  1/sqrt(d) folded into W_q, P = softmax_rows(S), O = P V against V^T = W_v X^T produced directly by a GEMM whose
  "weight" operand is the activation matrix); the V bias commutes with the softmax (rows of P sum to 1) and is folded
  into the output projection's bias;
* quant_conv (1x1) is composed into the encoder's conv_out at pack time; time_conv_out + the tokens -> NCHW layout
  change are one small kernel (star_vae_head).

PARITY UNPINNED (diffusers is not in the reference tree nor in this image): checked against oracle/temporal_vae_ref.py,
a restatement of the published architecture.
"""
import json
import math
import os
from types import SimpleNamespace
from typing import NamedTuple

import torch
import torch.nn as nn

from ... import ops

HALF = torch.float16

__all__ = ["AutoencoderKLTemporalDecoder", "DecodePlan", "DiagonalGaussianDistribution", "decode_plan", "decode_peak_bytes"]


# ---- decode plan ---------------------------------------------------------------------------------------------------------
# A 3-frame window at 1080p -> 4x holds 26 GB per 128-channel full-resolution tensor, so decode() runs its full-resolution
# stages a few frames at a time, each up block's upsample + conv a band of rows at a time, and its temporal convs a pixel
# band at a time.  The window-sized tensors that the temporal GroupNorm statistics need (each st-resnet's input and output)
# are not split; the plan bounds what one pass allocates on top of them.  It depends on the window's shape only, never on free
# device memory, so a clip decodes the same way on any card.
PASS_BYTES = 26 << 30           # one spatial pass's transient tensors: one 1080p -> 4x frame (24.2 GiB) fits, a 720p -> 4x window does not
BAND_BYTES = 1 << 30            # one band of the normalised window / of an upsampled frame (split plans only)


class DecodePlan(NamedTuple):
    """frames: frames per pass of the spatial stages; band: pixels per band of the temporal stages; rows: output rows per band
    of the upsample + conv (>= a stage's H*W / H: one band)."""
    frames: int
    band: int
    rows: int


def _stages(H, W, ch, layers):
    """The decoder's st-resnets in order: (cin, cout, H, W of the input, upsample first?); the mid block's come first."""
    top = ch[-1]
    out = [(top, top, H, W, False) for _ in range(layers)]
    prev, up = top, False
    for c in reversed(ch):
        for _ in range(layers + 1):
            out.append((prev, c, H, W, up))
            if up:
                H, W, up = 2 * H, 2 * W, False
            prev = c
        up = True
    return out


def _pass_bytes(n, rows, cin, cout, H, W, up):
    """transient bytes of one pass of _spatial over n frames (fp16): (upsample + conv, resnet)"""
    hw2 = H * W * (4 if up else 1)
    u = n * hw2 * cin * 2 if up else 0
    if up:                                                    # the upsampled band: a whole pass, or rows + 4 rows of one frame
        ub = u if rows >= 2 * H else min(2 * H, rows + 4) * 2 * W * cin * 2
    t = n * hw2 * cin * 2 if cin == cout else 0               # GroupNorm output when x is the residual
    return (u + ub if up else 0), u + t + n * hw2 * cout * 2


def decode_plan(bf, num_frames, H, W, ch=(128, 256, 512, 512), layers=2):
    """The plan decode() runs a window of bf latent frames of H x W under: all frames in one pass and one band when a pass
    over the whole window stays within PASS_BYTES (every window up to 1080p outputs), else bands of BAND_BYTES and the most
    frames per pass that stay within it."""
    if bf < 1 or num_frames < 1 or bf % num_frames:
        raise ValueError(f"decode_plan: bf={bf} is not a positive multiple of num_frames={num_frames}")
    stages = _stages(H, W, ch, layers)
    scale = 2 ** (len(ch) - 1)
    full = DecodePlan(bf, H * W * scale * scale, H * scale)
    if max(max(_pass_bytes(bf, full.rows, *s)) for s in stages) <= PASS_BYTES:
        return full
    band = min(full.band, max(128, BAND_BYTES // (2 * bf * max(ch)) // 128 * 128))
    rows = min(full.rows, max(2, BAND_BYTES // (2 * W * scale * max(ch)) // 2 * 2))
    frames = bf
    while frames > 1 and max(max(_pass_bytes(frames, rows, *s)) for s in stages) > PASS_BYTES:
        frames -= 1
    return DecodePlan(frames, band, rows)


def decode_peak_bytes(plan, bf, H, W, ch=(128, 256, 512, 512), layers=2):
    """Predicted peak of the activations decode() allocates under `plan` (fp16 tensors and workspaces; weights and z excluded)."""
    top, hw = ch[-1], H * W
    rgb = bf * hw * 4 ** (len(ch) - 1) * 8 * 2                                        # held from the start
    return rgb + _peak_without_rgb(plan, bf, H, W, ch, layers)


def _peak_without_rgb(plan, bf, H, W, ch, layers):
    top, hw = ch[-1], H * W
    win = bf * hw * top * 2
    peak = bf * hw * 4 * 2 + (bf * hw * 64 + top * 64) * 2 + win                      # conv_in: tokens, im2col, output
    ld = (hw + 7) // 8 * 8
    rb = max(128, min(hw, (1 << 28) // ld // 128 * 128))
    peak = max(peak, 7 * win + (min(rb, hw) + top) * ld * 2)                          # mid-block attention
    for cin, cout, h, w, up in _stages(H, W, ch, layers):
        hw2 = h * w * (4 if up else 1)
        x = bf * h * w * cin * 2
        xs = 0 if not up and cin == cout else bf * hw2 * cout * 2
        p_up, p_res = _pass_bytes(min(plan.frames, bf), plan.rows, cin, cout, h, w, up)
        peak = max(peak, x + (xs if plan.frames < bf else 0) + p_up, x + xs + p_res)      # xs is allocated after pass 0's upsample
        s = bf * hw2 * cout * 2
        peak = max(peak, 2 * s + bf * min(plan.band, hw2) * cout * 2)                  # temporal: xs, t, one band of GN(xs)
    hw = hw * 4 ** (len(ch) - 1)
    return max(peak, bf * hw * (ch[0] + 3) * 2)                                       # tail: h, sample


class DiagonalGaussianDistribution:
    """moments (n, 2c, h, w) -> mean / logvar; sample() = mean + std * randn (diffusers vae.py)."""

    def __init__(self, parameters):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None):
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise

    def mode(self):
        return self.mean


def _res_keys(m, p, cin, cout, temporal=False):
    k = (3, 1, 1) if temporal else (3, 3)
    for n, c in (("norm1", cin), ("norm2", cout)):
        m[f"{p}.{n}.weight"] = (c,)
        m[f"{p}.{n}.bias"] = (c,)
    m[f"{p}.conv1.weight"], m[f"{p}.conv1.bias"] = (cout, cin) + k, (cout,)
    m[f"{p}.conv2.weight"], m[f"{p}.conv2.bias"] = (cout, cout) + k, (cout,)
    if cin != cout:
        m[f"{p}.conv_shortcut.weight"], m[f"{p}.conv_shortcut.bias"] = (cout, cin) + (1,) * len(k), (cout,)


def _param_shapes(ch, layers, latent, cin_img, cout_img):
    """Checkpoint layout of diffusers' AutoencoderKLTemporalDecoder: {dotted key: shape}."""
    m = {}

    def conv(p, co, ci, k=(3, 3)):
        m[p + ".weight"], m[p + ".bias"] = (co, ci) + k, (co,)

    def attn(p, c):
        m[p + ".group_norm.weight"], m[p + ".group_norm.bias"] = (c,), (c,)
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            m[f"{p}.{n}.weight"], m[f"{p}.{n}.bias"] = (c, c), (c,)

    def st_res(p, ci, co):
        _res_keys(m, p + ".spatial_res_block", ci, co)
        _res_keys(m, p + ".temporal_res_block", co, co, temporal=True)
        m[p + ".time_mixer.mix_factor"] = (1,)

    top = ch[-1]
    conv("encoder.conv_in", ch[0], cin_img)
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(layers):
            _res_keys(m, f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        if i + 1 < len(ch):
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", c, c)
        prev = c
    attn("encoder.mid_block.attentions.0", top)
    for j in range(2):
        _res_keys(m, f"encoder.mid_block.resnets.{j}", top, top)
    m["encoder.conv_norm_out.weight"], m["encoder.conv_norm_out.bias"] = (top,), (top,)
    conv("encoder.conv_out", 2 * latent, top)
    conv("quant_conv", 2 * latent, 2 * latent, (1, 1))
    conv("decoder.conv_in", top, latent)
    attn("decoder.mid_block.attentions.0", top)
    for j in range(layers):
        st_res(f"decoder.mid_block.resnets.{j}", top, top)
    prev = top
    for i, c in enumerate(reversed(ch)):
        for j in range(layers + 1):
            st_res(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
        if i + 1 < len(ch):
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", c, c)
        prev = c
    m["decoder.conv_norm_out.weight"], m["decoder.conv_norm_out.bias"] = (ch[0],), (ch[0],)
    conv("decoder.conv_out", cout_img, ch[0])
    conv("decoder.time_conv_out", cout_img, cout_img, (3, 1, 1))
    return m


class AutoencoderKLTemporalDecoder(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, sample_size=768, scaling_factor=0.18215, force_upcast=True, **unused):
        super().__init__()
        if in_channels > 4 or latent_channels != 4 or out_channels != 3:
            raise NotImplementedError("star_b200 temporal VAE: RGB in/out and 4 latent channels only")
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels,
                                      block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      latent_channels=latent_channels, sample_size=sample_size,
                                      scaling_factor=scaling_factor, force_upcast=force_upcast)
        for key, shape in _param_shapes(tuple(block_out_channels), layers_per_block, latent_channels, in_channels,
                                        out_channels).items():
            *path, leaf = key.split(".")
            mod = self
            for name in path:
                if name not in mod._modules:
                    mod.add_module(name, nn.Module())
                mod = mod._modules[name]
            mod.register_parameter(leaf, nn.Parameter(torch.zeros(shape), requires_grad=False))
        self._pk = None

    # ---- loading ---------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path, subfolder=None, variant=None, torch_dtype=None, **unused):
        """Local directory in the diffusers layout: config.json + diffusion_pytorch_model[.variant].safetensors|.bin.
        (No hub download: the reference's "stabilityai/stable-video-diffusion-img2vid" must be fetched beforehand.)"""
        root = os.path.join(path, subfolder) if subfolder else path
        if not os.path.isdir(root):
            raise FileNotFoundError(f"temporal VAE directory not found: {root!r} (hub ids are not downloaded; "
                                    "pass a local snapshot of stabilityai/stable-video-diffusion-img2vid/vae)")
        kw = {}
        cfg_path = os.path.join(root, "config.json")
        if os.path.exists(cfg_path):
            with open(cfg_path) as f:
                raw = json.load(f)
            kw = {k: v for k, v in raw.items() if not k.startswith("_") and k != "down_block_types"}
        model = cls(**kw)
        stems = [f"diffusion_pytorch_model.{variant}" if variant else None, "diffusion_pytorch_model"]
        for stem in filter(None, stems):
            st = os.path.join(root, stem + ".safetensors")
            if os.path.exists(st):
                from safetensors.torch import load_file
                model.load_state_dict(load_file(st))
                break
            pt = os.path.join(root, stem + ".bin")
            if os.path.exists(pt):
                model.load_state_dict(torch.load(pt, map_location="cpu"))
                break
        else:
            raise FileNotFoundError(f"no diffusion_pytorch_model weights under {root!r}")
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()

    def _apply(self, fn, *a, **k):
        self._pk = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._pk = None
        return super().load_state_dict(*a, **k)

    # ---- weight repacking ----------------------------------------------------------------------------------
    def _pack(self):
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        dev = next(self.parameters()).device
        pk = {}

        def h(t):
            return t.to(HALF).contiguous().to(dev)

        def w9(key, scale=1.0):                      # [co, ci, 3, 3] -> [co, 3, 3, ci]
            w = sd[key + ".weight"] * scale
            if w.shape[1] < 4:                       # RGB stem: zero 4th input channel
                w = torch.cat([w, w.new_zeros(w.shape[0], 4 - w.shape[1], 3, 3)], dim=1)
            return h(w.permute(0, 2, 3, 1)), h(sd[key + ".bias"] * scale)

        def w3(key, scale=1.0):                      # [co, ci, 3, 1, 1] -> [co, 3, ci]
            return h((sd[key + ".weight"][:, :, :, 0, 0] * scale).permute(0, 2, 1)), h(sd[key + ".bias"] * scale)

        def norm(key):
            return h(sd[key + ".weight"]), h(sd[key + ".bias"])

        def res2d(p):
            r = {"n1": norm(p + ".norm1"), "c1": w9(p + ".conv1"), "n2": norm(p + ".norm2"), "c2": w9(p + ".conv2")}
            if p + ".conv_shortcut.weight" in sd:
                r["sc"] = (h(sd[p + ".conv_shortcut.weight"].flatten(1)), h(sd[p + ".conv_shortcut.bias"]))
            return r

        def st_res(p):
            mix = torch.sigmoid(sd[p + ".time_mixer.mix_factor"]).item()      # = 1 - alpha (switch_spatial_to_temporal_mix)
            t = p + ".temporal_res_block"
            return {"s": res2d(p + ".spatial_res_block"), "tn1": norm(t + ".norm1"), "tc1": w3(t + ".conv1"),
                    "tn2": norm(t + ".norm2"), "tc2": w3(t + ".conv2", mix)}

        def attn(p):
            c = sd[p + ".to_q.weight"].shape[0]
            s = 1.0 / math.sqrt(c)
            wo, bv = sd[p + ".to_out.0.weight"], sd[p + ".to_v.bias"]
            return {"gn": norm(p + ".group_norm"), "q": (h(sd[p + ".to_q.weight"] * s), h(sd[p + ".to_q.bias"] * s)),
                    "k": (h(sd[p + ".to_k.weight"]), h(sd[p + ".to_k.bias"])), "v": h(sd[p + ".to_v.weight"]),
                    "o": (h(wo), h(sd[p + ".to_out.0.bias"] + wo @ bv))}

        ch, L = self.config.block_out_channels, self.config.layers_per_block
        enc = {"in": w9("encoder.conv_in"), "down": [], "mid": [res2d("encoder.mid_block.resnets.0"),
                                                                  res2d("encoder.mid_block.resnets.1")],
               "attn": attn("encoder.mid_block.attentions.0"), "nout": norm("encoder.conv_norm_out")}
        for i in range(len(ch)):
            blk = {"res": [res2d(f"encoder.down_blocks.{i}.resnets.{j}") for j in range(L)]}
            if i + 1 < len(ch):
                blk["down"] = w9(f"encoder.down_blocks.{i}.downsamplers.0.conv")
            enc["down"].append(blk)
        wq = sd["quant_conv.weight"][:, :, 0, 0]                                # moments = Wq (conv_out(h)) + bq
        wco = torch.einsum("om,mcxy->ocxy", wq, sd["encoder.conv_out.weight"])
        bco = wq @ sd["encoder.conv_out.bias"] + sd["quant_conv.bias"]
        enc["out"] = (h(wco.permute(0, 2, 3, 1)), h(bco))
        dec = {"in": w9("decoder.conv_in"), "mid": [st_res(f"decoder.mid_block.resnets.{j}") for j in range(L)],
               "attn": attn("decoder.mid_block.attentions.0"), "up": [], "nout": norm("decoder.conv_norm_out"),
               "out": w9("decoder.conv_out"),
               "head": (h(sd["decoder.time_conv_out.weight"].reshape(27)), h(sd["decoder.time_conv_out.bias"]))}
        for i in range(len(ch)):
            blk = {"res": [st_res(f"decoder.up_blocks.{i}.resnets.{j}") for j in range(L + 1)]}
            if i + 1 < len(ch):
                blk["up"] = w9(f"decoder.up_blocks.{i}.upsamplers.0.conv")
            dec["up"].append(blk)
        pk["enc"], pk["dec"] = enc, dec
        self._pk = pk
        return pk

    def _packed(self):
        return self._pk if self._pk is not None else self._pack()

    # ---- blocks (x: [n*H*W, C] fp16 tokens) ------------------------------------------------------------------
    @staticmethod
    def _res2d(r, x, n, H, W, out=None, eps=1e-6):
        """x [n*H*W, cin] is consumed: with a shortcut conv the shortcut goes straight to out and x is then normalised in
        place; without one x is the residual and out defaults to x itself (the last conv reads and writes the same element)."""
        cin, cout = x.shape[1], r["c1"][0].shape[0]
        if out is None:
            out = x if "sc" not in r else torch.empty((x.shape[0], cout), dtype=HALF, device=x.device)
        if "sc" in r:
            res = ops.linear(x, r["sc"][0], r["sc"][1], out=out)
            t = ops.groupnorm(x, r["n1"][0], r["n1"][1], n, eps, True, out=x)
        else:
            res = x
            t = ops.groupnorm(x, r["n1"][0], r["n1"][1], n, eps, True)
        t = ops.conv2d_3x3(t.view(n, H, W, cin), r["c1"][0], r["c1"][1])
        t = ops.groupnorm(t, r["n2"][0], r["n2"][1], n, eps, True, out=t)
        return ops.conv2d_3x3(t.view(n, H, W, cout), r["c2"][0], r["c2"][1], residual=res, out=out)

    @classmethod
    def _spatial(cls, r, x, bf, H, W, frames, rows, up=None):
        """Spatial half of a SpatioTemporalResBlock over the window x [bf*H*W, cin], `frames` frames per pass, preceded by the
        previous up block's nearest-x2 upsample and conv (`rows` output rows per band) when `up` is given.  x is consumed.
        Returns (xs, H', W')."""
        cin, cout = x.shape[1], r["c1"][0].shape[0]
        H2, W2 = (2 * H, 2 * W) if up is not None else (H, W)
        hw, hw2 = H * W, H2 * W2
        xs = x if up is None and "sc" not in r else None
        for f0 in range(0, bf, frames):
            n = min(frames, bf - f0)
            xf = x[f0 * hw:(f0 + n) * hw]
            if up is not None:
                xf = cls._upconv(up, xf, n, H, W, rows)
            if xs is None:              # after the first upsample: one pass over the window never holds xs and the upsample at once
                xs = torch.empty((bf * hw2, cout), dtype=HALF, device=x.device)
            cls._res2d(r, xf, n, H2, W2, out=xs[f0 * hw2:(f0 + n) * hw2])
        return xs, H2, W2

    @staticmethod
    def _upconv(up, x, n, H, W, rows):
        """conv3x3(nearest_x2(x)) of n frames x [n*H*W, C] -> [n*2H*2W, C].  With rows < 2H each frame is done in bands of
        `rows` output rows (rows even): the band's input rows, plus one halo row on each side, are upsampled from x and the
        conv computes only the band's rows, so at most rows + 4 upsampled rows of one frame exist at once."""
        C, H2, W2 = x.shape[1], 2 * H, 2 * W
        u = torch.empty((n * H2 * W2, C), dtype=HALF, device=x.device)
        g = n if rows >= H2 else 1                  # frames per band
        for j in range(0, n, g):
            for r0 in range(0, H2, rows):
                r1 = min(H2, r0 + rows)
                a, b = max(0, r0 // 2 - 1), min(H, r1 // 2 + 1)         # low-res rows holding upsampled rows r0 - 1 .. r1
                xu = ops.upsample2x(x[(j * H + a) * W:((j + g - 1) * H + b) * W], g, b - a, W)
                kw = {} if r1 - r0 == H2 else {"rows": (r0 - 2 * a, r1 - r0)}      # a whole frame is the plain conv
                ops.conv2d_3x3(xu.view(g, 2 * (b - a), W2, C), up[0], up[1], out=u[(j * H2 + r0) * W2:((j + g - 1) * H2 + r1) * W2],
                               **kw)
                del xu
        return u

    @staticmethod
    def _temporal(r, xs, B, T, HW, band):
        """Temporal half + AlphaBlender, in place on xs [B*T*HW, C].  The first GroupNorm's clip statistics are taken once;
        its apply and the first (3,1,1) conv then run `band` pixels of every frame at a time, so only a band of the
        normalised clip exists at once.  The second GroupNorm is in place and the second conv writes over its residual."""
        t = torch.empty_like(xs)
        if band >= HW:                  # one band: the same statistics and apply launches as the banded path
            g = ops.groupnorm(xs, r["tn1"][0], r["tn1"][1], B, 1e-5, True)
            ops.conv_t3(g, r["tc1"][0], r["tc1"][1], B=B, T=T, HW=HW, out=t)
            del g
        else:
            for p01, g in ops.groupnorm(xs, r["tn1"][0], r["tn1"][1], B, 1e-5, True, bands=(HW, band)):
                ops.conv_t3(g, r["tc1"][0], r["tc1"][1], B=B, T=T, HW=HW, band=p01, out=t)
                del g
        t = ops.groupnorm(t, r["tn2"][0], r["tn2"][1], B, 1e-5, True, out=t)
        return ops.conv_t3(t, r["tc2"][0], r["tc2"][1], residual=xs, B=B, T=T, HW=HW, out=xs)

    @staticmethod
    def _attention(a, x, n, HW):
        C = x.shape[1]
        xn = ops.groupnorm(x, a["gn"][0], a["gn"][1], n, 1e-6, False)
        q = ops.linear(xn, a["q"][0], a["q"][1])
        k = ops.linear(xn, a["k"][0], a["k"][1])
        ld = (HW + 7) // 8 * 8
        # a row of logits is spread over as many CTAs as its keys need (one CTA stages <= 102 400 of them, a 2 560 x 2 560-pixel
        # frame; 234 576 at 720p -> 4x take 3).  Rows that fit one CTA make the default call, which is also the signature of
        # the emulated kernel in oracle/kernel_ref.py.  Logits are materialised for a block of query rows at a time (<= 0.6 GB
        # up to 819 200 key columns, the most 8 CTAs hold); columns HW..ld of S are zeroed by star_softmax_rows
        cluster = {} if HW <= 102400 else {"ctas_per_row": -(-HW // 102400)}
        rb = max(128, min(HW, (1 << 28) // ld // 128 * 128))
        S = torch.empty((min(rb, HW), ld), dtype=HALF, device=x.device)
        vt = torch.zeros((C, ld), dtype=HALF, device=x.device)
        o = torch.empty_like(x)
        for f in range(n):
            rows = slice(f * HW, (f + 1) * HW)
            ops.linear(a["v"], xn[rows], out=vt[:, :HW])                    # V^T = W_v X^T  [C, HW]
            for r0 in range(0, HW, rb):
                r1 = min(HW, r0 + rb)
                Sb = S[: r1 - r0]
                ops.linear(q[f * HW + r0:f * HW + r1], k[rows], out=Sb[:, :HW])   # logits, 1/sqrt(C) already in W_q
                ops.softmax_rows(Sb, HW, **cluster)
                ops.linear(Sb, vt, out=o[f * HW + r0:f * HW + r1])          # P V
        return ops.linear(o, a["o"][0], a["o"][1], residual=x)

    # ---- public surface ----------------------------------------------------------------------------------
    @torch.no_grad()
    def encode(self, x, return_dict=True):
        """x (n, 3, H, W) in [-1, 1], H and W multiples of 8 -> latent_dist over (n, 4, H/8, W/8)."""
        pk = self._packed()["enc"]
        n, c, H, W = x.shape
        if H % 8 or W % 8:
            raise ValueError("temporal VAE encode: H and W must be multiples of 8")
        x = x.float()
        if c < 4:
            x = torch.cat([x, x.new_zeros(n, 4 - c, H, W)], dim=1)
        h = ops.nchw5_to_tokens(x.unsqueeze(2))                              # [(n H W), 4]
        h = ops.conv2d_3x3_c4(h.view(n, H, W, 4), pk["in"][0], pk["in"][1])
        for blk in pk["down"]:
            for r in blk["res"]:
                h = self._res2d(r, h, n, H, W)
            if "down" in blk:
                h, H, W = ops.conv2d_3x3_s2p(h.view(n, H, W, h.shape[1]), blk["down"][0], blk["down"][1], (0, 1, 0, 1))
        h = self._res2d(pk["mid"][0], h, n, H, W)
        h = self._attention(pk["attn"], h, n, H * W)
        h = self._res2d(pk["mid"][1], h, n, H, W)
        h = ops.groupnorm(h, pk["nout"][0], pk["nout"][1], n, 1e-6, True, out=h)
        m = ops.conv2d_3x3(h.view(n, H, W, h.shape[1]), pk["out"][0], pk["out"][1])         # conv_out o quant_conv
        moments = ops.tokens_to_nchw5(m, n, m.shape[1], 1, H, W)[:, :, 0].float()
        dist = DiagonalGaussianDistribution(moments)
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z, num_frames, return_dict=True, plan=None):
        """z (b*num_frames, 4, h, w) -> sample (b*num_frames, 3, 8h, 8w) fp16.  Runs under decode_plan() of the window's
        shape unless a DecodePlan is given; every plan computes the same function."""
        pk = self._packed()["dec"]
        bf, c, H, W = z.shape
        T = int(num_frames)
        if bf % T:
            raise ValueError("temporal VAE decode: batch is not a multiple of num_frames")
        B = bf // T
        ch, L = self.config.block_out_channels, self.config.layers_per_block
        plan = plan or decode_plan(bf, T, H, W, ch, L)
        if plan.frames < 1 or plan.band < 1 or plan.rows < 2 or plan.rows % 2:
            raise ValueError(f"temporal VAE decode: bad plan {plan}")

        def stages():                   # (resnet, upsampler of the previous up block or None); "attn" = mid-block attention
            yield pk["mid"][0], None
            for r in pk["mid"][1:]:
                yield "attn", None
                yield r, None
            up = None
            for blk in pk["up"]:
                for r in blk["res"]:
                    yield r, up
                    up = None
                up = blk.get("up")

        # A split plan's window-sized tensors come and go in caching-allocator segments of tens of GiB.  A small tensor carved
        # from a freed one (this window's RGB or output, or the caller's post-processing of it) would pin it, and the next
        # window could not place its own, so under a split plan the free cached segments are released before the small
        # tensors are allocated and before returning.
        scale = 2 ** (len(ch) - 1)
        split = plan.frames < bf or plan.band < H * W * scale * scale or plan.rows < H * scale
        if split:
            torch.cuda.empty_cache()
        rgb = torch.empty((bf * H * W * scale * scale, 8), dtype=HALF, device=z.device)
        h = ops.nchw5_to_tokens(z.float().unsqueeze(2))
        h = ops.conv2d_3x3_c4(h.view(bf, H, W, 4), pk["in"][0], pk["in"][1])
        for r, up in stages():
            if isinstance(r, str):
                h = self._attention(pk["attn"], h, bf, H * W)
                continue
            h, H, W = self._spatial(r["s"], h, bf, H, W, plan.frames, plan.rows, up)
            h = self._temporal(r, h, B, T, H * W, plan.band)
        HW = H * W
        for f0 in range(0, bf, plan.frames):
            n = min(plan.frames, bf - f0)
            x = h[f0 * HW:(f0 + n) * HW]
            x = ops.groupnorm(x, pk["nout"][0], pk["nout"][1], n, 1e-6, True, out=x)
            ops.conv2d_3x3(x.view(n, H, W, h.shape[1]), pk["out"][0], pk["out"][1], out=rgb[f0 * HW:(f0 + n) * HW, :3])
        del h
        if split:
            torch.cuda.empty_cache()
        sample = ops.vae_head(rgb, pk["head"][0], pk["head"][1], B, T, H, W)
        del rgb
        if split:
            torch.cuda.empty_cache()
        return SimpleNamespace(sample=sample) if return_dict else (sample,)

    def forward(self, sample, sample_posterior=False, generator=None, num_frames=1):
        post = self.encode(sample).latent_dist
        z = post.sample(generator=generator) if sample_posterior else post.mode()
        return self.decode(z, num_frames=num_frames)
