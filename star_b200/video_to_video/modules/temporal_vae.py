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

import torch
import torch.nn as nn

from ... import ops

HALF = torch.float16

__all__ = ["AutoencoderKLTemporalDecoder", "DiagonalGaussianDistribution"]


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
    def _res2d(r, x, n, H, W, eps=1e-6):
        cin = x.shape[1]
        t = ops.groupnorm(x, r["n1"][0], r["n1"][1], n, eps, True)
        t = ops.conv2d_3x3(t.view(n, H, W, cin), r["c1"][0], r["c1"][1])
        cout = t.shape[1]
        t = ops.groupnorm(t, r["n2"][0], r["n2"][1], n, eps, True, out=t)
        sc = ops.linear(x, r["sc"][0], r["sc"][1]) if "sc" in r else x
        return ops.conv2d_3x3(t.view(n, H, W, cout), r["c2"][0], r["c2"][1], residual=sc)

    @classmethod
    def _st_res(cls, r, x, B, T, H, W):
        xs = cls._res2d(r["s"], x, B * T, H, W)
        t = ops.groupnorm(xs, r["tn1"][0], r["tn1"][1], B, 1e-5, True)
        t = ops.conv_t3(t, r["tc1"][0], r["tc1"][1], B=B, T=T, HW=H * W)
        t = ops.groupnorm(t, r["tn2"][0], r["tn2"][1], B, 1e-5, True, out=t)
        return ops.conv_t3(t, r["tc2"][0], r["tc2"][1], residual=xs, B=B, T=T, HW=H * W)

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
    def decode(self, z, num_frames, return_dict=True):
        """z (b*num_frames, 4, h, w) -> sample (b*num_frames, 3, 8h, 8w) fp16."""
        pk = self._packed()["dec"]
        bf, c, H, W = z.shape
        T = int(num_frames)
        if bf % T:
            raise ValueError("temporal VAE decode: batch is not a multiple of num_frames")
        B = bf // T
        h = ops.nchw5_to_tokens(z.float().unsqueeze(2))
        h = ops.conv2d_3x3_c4(h.view(bf, H, W, 4), pk["in"][0], pk["in"][1])
        h = self._st_res(pk["mid"][0], h, B, T, H, W)
        for r in pk["mid"][1:]:
            h = self._attention(pk["attn"], h, bf, H * W)
            h = self._st_res(r, h, B, T, H, W)
        for blk in pk["up"]:
            for r in blk["res"]:
                h = self._st_res(r, h, B, T, H, W)
            if "up" in blk:
                C = h.shape[1]
                h = ops.upsample2x(h, bf, H, W)
                H, W = 2 * H, 2 * W
                h = ops.conv2d_3x3(h.view(bf, H, W, C), blk["up"][0], blk["up"][1])
        h = ops.groupnorm(h, pk["nout"][0], pk["nout"][1], bf, 1e-6, True, out=h)
        rgb = torch.empty((bf * H * W, 8), dtype=HALF, device=h.device)
        ops.conv2d_3x3(h.view(bf, H, W, h.shape[1]), pk["out"][0], pk["out"][1], out=rgb[:, :3])
        sample = ops.vae_head(rgb, pk["head"][0], pk["head"][1], B, T, H, W)
        return SimpleNamespace(sample=sample) if return_dict else (sample,)

    def forward(self, sample, sample_posterior=False, generator=None, num_frames=1):
        post = self.encode(sample).latent_dist
        z = post.sample(generator=generator) if sample_posterior else post.mode()
        return self.decode(z, num_frames=num_frames)
