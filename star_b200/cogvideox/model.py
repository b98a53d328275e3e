"""STAR's CogVideoX-5B DiT (cogvideox-based/sat/dit_video_concat.py:602-817 ``DiffusionTransformer``) on the star_b200 kernels.

Parameter tree = the reference checkpoint's (sat) key layout, so ``load_state_dict`` of the `model.diffusion_model.*` part of a
STAR CogVideoX checkpoint works unchanged:
    mixins.patch_embed.{proj_sr,text_proj}.*                      ImagePatchEmbeddingMixin          (:23-82)
    mixins.adaln_layer.{adaLN_modulations.i.1,query_layernorm_list.i,key_layernorm_list.i}.*        AdaLNMixin (:416-480)
    mixins.final_layer.{norm_final,linear,adaLN_modulation.1}.*   FinalLayerMixin                   (:372-414)
    transformer.layers.i.{input_layernorm,post_attention_layernorm,attention.*,mlp.*,spa_local,temp_local}.*
                                                                  cogvideox-based/transformer.py:368-490
    transformer.layers.i.attention.{query_key_value,dense}.{original.*,matrix_A.k,matrix_B.k}       LoRA r = 512 (yaml :70-73)
    transformer.final_layernorm.*, time_embed.{0,2}.*             transformer.py:629-631, dit_video_concat.py:680-687
``nn`` only stores the parameters.  Execution: everything is a token matrix X[(b s), 3072]; patch embedding is an im2col view +
one GEMM; LoRA is merged into the dense weights at pack time (W + (alpha / r) B A -- inference only); the 42 layers are
``DiTLayer`` (dit_block.py); final LayerNorm -> LayerNorm + adaLN modulate (folded into its affine) -> Linear -> unpatchify.
Precision follows the dtype the model is built with: torch.bfloat16 (the reference config, yaml :11) runs on the bf16 build of
the kernel library, torch.float16 on the default one; fp32 accumulation in both.
"""
import math

import torch
import torch.nn as nn

from .. import ops
from .dit_block import DiTLayer


def rope_tables(frames, height, width, head_dim=64, theta=10000.0):
    """freqs_cos / freqs_sin (t*h*w, head_dim) of Rotary3DPositionEmbeddingMixin.__init__ (dit_video_concat.py:269-297)."""
    dim_t, dim_h, dim_w = head_dim // 4, head_dim // 8 * 3, head_dim // 8 * 3

    def axis(n, dim):
        fr = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))
        f = torch.arange(n, dtype=torch.float32)[:, None] * fr[None, :]
        return f.repeat_interleave(2, dim=-1)                                     # "... n -> ... (n r)", r = 2

    ft, fh, fw = axis(frames, dim_t), axis(height, dim_h), axis(width, dim_w)
    freqs = torch.cat([ft[:, None, None, :].expand(frames, height, width, dim_t),
                       fh[None, :, None, :].expand(frames, height, width, dim_h),
                       fw[None, None, :, :].expand(frames, height, width, dim_w)], dim=-1).reshape(-1, head_dim)
    return freqs.cos().contiguous(), freqs.sin().contiguous()


def dit_manifest(num_layers=42, hidden=3072, heads=48, time_embed_dim=512, in_channels=16, out_channels=16, patch=2,
                 text_hidden=4096, lora_r=512):
    """{key: shape} of DiffusionTransformer's state dict (buffers excluded)."""
    hd, m = hidden // heads, {}
    m["mixins.patch_embed.proj_sr.weight"] = (hidden, 2 * in_channels, patch, patch)
    m["mixins.patch_embed.proj_sr.bias"] = (hidden,)
    m["mixins.patch_embed.text_proj.weight"] = (hidden, text_hidden)
    m["mixins.patch_embed.text_proj.bias"] = (hidden,)
    for i in range(num_layers):
        m[f"mixins.adaln_layer.adaLN_modulations.{i}.1.weight"] = (12 * hidden, time_embed_dim)
        m[f"mixins.adaln_layer.adaLN_modulations.{i}.1.bias"] = (12 * hidden,)
        for n in ("query", "key"):
            m[f"mixins.adaln_layer.{n}_layernorm_list.{i}.weight"] = (hd,)
            m[f"mixins.adaln_layer.{n}_layernorm_list.{i}.bias"] = (hd,)
        p = f"transformer.layers.{i}."
        for n in ("input_layernorm", "post_attention_layernorm"):
            m[p + n + ".weight"], m[p + n + ".bias"] = (hidden,), (hidden,)
        lo = ".original" if lora_r else ""
        m[p + f"attention.query_key_value{lo}.weight"], m[p + f"attention.query_key_value{lo}.bias"] = (3 * hidden, hidden), (3 * hidden,)
        m[p + f"attention.dense{lo}.weight"], m[p + f"attention.dense{lo}.bias"] = (hidden, hidden), (hidden,)
        if lora_r:
            for k in range(3):
                m[p + f"attention.query_key_value.matrix_A.{k}"] = (lora_r, hidden)
                m[p + f"attention.query_key_value.matrix_B.{k}"] = (hidden, lora_r)
            m[p + "attention.dense.matrix_A.0"], m[p + "attention.dense.matrix_B.0"] = (lora_r, hidden), (hidden, lora_r)
        m[p + "mlp.dense_h_to_4h.weight"], m[p + "mlp.dense_h_to_4h.bias"] = (4 * hidden, hidden), (4 * hidden,)
        m[p + "mlp.dense_4h_to_h.weight"], m[p + "mlp.dense_4h_to_h.bias"] = (hidden, 4 * hidden), (hidden,)
        m[p + "spa_local.conv1.weight"], m[p + "temp_local.conv1.weight"] = (1, 2, 7, 7), (1, 2)
    m["mixins.final_layer.norm_final.weight"], m["mixins.final_layer.norm_final.bias"] = (hidden,), (hidden,)
    m["mixins.final_layer.linear.weight"] = (patch * patch * out_channels, hidden)
    m["mixins.final_layer.linear.bias"] = (patch * patch * out_channels,)
    m["mixins.final_layer.adaLN_modulation.1.weight"], m["mixins.final_layer.adaLN_modulation.1.bias"] = (2 * hidden, time_embed_dim), (2 * hidden,)
    m["transformer.final_layernorm.weight"], m["transformer.final_layernorm.bias"] = (hidden,), (hidden,)
    m["time_embed.0.weight"], m["time_embed.0.bias"] = (time_embed_dim, hidden), (time_embed_dim,)
    m["time_embed.2.weight"], m["time_embed.2.bias"] = (time_embed_dim, time_embed_dim), (time_embed_dim,)
    return m


class DiffusionTransformer(nn.Module):
    """``forward(x, timesteps, context)``: x (b, t, 2*in_channels, h, w) = noisy latent || LQ latent (sample_sr concat),
    timesteps (b,), context (b, text_length, text_hidden) -> (b, t, out_channels, h, w)."""

    def __init__(self, num_layers=42, hidden_size=3072, num_attention_heads=48, num_frames=49, time_compressed_rate=4,
                 latent_height=60, latent_width=90, patch_size=2, in_channels=16, out_channels=16, time_embed_dim=512,
                 text_length=226, text_hidden_size=4096, lora_r=512, lora_alpha=1.0, layernorm_epsilon=1e-5,
                 dtype=torch.bfloat16):
        super().__init__()
        self.cfg = dict(num_layers=num_layers, hidden=hidden_size, heads=num_attention_heads, time_embed_dim=time_embed_dim,
                        in_channels=in_channels, out_channels=out_channels, patch=patch_size, text_hidden=text_hidden_size,
                        lora_r=lora_r)
        self.frames = (num_frames - 1) // time_compressed_rate + 1
        self.gh, self.gw = latent_height // patch_size, latent_width // patch_size
        self.text_length, self.lora_alpha, self.ln_eps, self.dtype = text_length, lora_alpha, layernorm_epsilon, dtype
        for key, shape in dit_manifest(**self.cfg).items():
            *path, leaf = key.split(".")
            mod = self
            for name in path:
                if name not in mod._modules:
                    mod.add_module(name, nn.Module())
                mod = mod._modules[name]
            mod.register_parameter(leaf, nn.Parameter(torch.zeros(shape), requires_grad=False))
        self._pk = None

    def _apply(self, fn, *a, **k):
        self._pk = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, sd, *a, **k):
        self._pk = None
        sd = {key: v for key, v in sd.items() if not key.startswith("mixins.pos_embed.freqs_") and key != "transformer.position_embeddings.weight"}
        return super().load_state_dict(sd, *a, **k)

    # ---- packing: LoRA merge, per-layer weight dicts, rope tables ---------------------------------------------------
    def _pack(self):
        c, dt = self.cfg, self.dtype
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        dev = next(self.parameters()).device
        d, r = c["hidden"], c["lora_r"]

        def h(t):
            return t.to(dev, dt).contiguous()

        def merged(p, parts):
            if not r:
                return sd[p + ".weight"].float(), sd[p + ".bias"].float()
            w = sd[p + ".original.weight"].float().clone()
            rows = w.shape[0] // parts
            for k in range(parts):
                w[k * rows:(k + 1) * rows] += (self.lora_alpha / r) * (sd[p + f".matrix_B.{k}"].float() @ sd[p + f".matrix_A.{k}"].float())
            return w, sd[p + ".original.bias"].float()

        cos, sin = rope_tables(self.frames, self.gh, self.gw, d // c["heads"])
        layers = []
        for i in range(c["num_layers"]):
            p = f"transformer.layers.{i}."
            wqkv, bqkv = merged(p + "attention.query_key_value", 3)
            wo, bo = merged(p + "attention.dense", 1)
            lsd = {"adaLN_modulation.1.weight": sd[f"mixins.adaln_layer.adaLN_modulations.{i}.1.weight"],
                   "adaLN_modulation.1.bias": sd[f"mixins.adaln_layer.adaLN_modulations.{i}.1.bias"],
                   "attention.query_key_value.weight": wqkv, "attention.query_key_value.bias": bqkv,
                   "attention.dense.weight": wo, "attention.dense.bias": bo}
            for n in ("input_layernorm", "post_attention_layernorm", "mlp.dense_h_to_4h", "mlp.dense_4h_to_h"):
                lsd[n + ".weight"], lsd[n + ".bias"] = sd[p + n + ".weight"], sd[p + n + ".bias"]
            lsd["spa_local.conv1.weight"], lsd["temp_local.conv1.weight"] = sd[p + "spa_local.conv1.weight"], sd[p + "temp_local.conv1.weight"]
            for n in ("query", "key"):
                lsd[n + "_layernorm.weight"] = sd[f"mixins.adaln_layer.{n}_layernorm_list.{i}.weight"]
                lsd[n + "_layernorm.bias"] = sd[f"mixins.adaln_layer.{n}_layernorm_list.{i}.bias"]
            layers.append(DiTLayer(lsd, d, c["heads"], self.text_length, self.frames, self.gh, self.gw, self.ln_eps, 1e-6,
                                   cos, sin, device=dev, dtype=dt, time_embed_dim=c["time_embed_dim"]))
        pk = {"layers": layers,
              "patch": (h(sd["mixins.patch_embed.proj_sr.weight"].flatten(1)), h(sd["mixins.patch_embed.proj_sr.bias"])),
              "text": (h(sd["mixins.patch_embed.text_proj.weight"]), h(sd["mixins.patch_embed.text_proj.bias"])),
              "te0": (h(sd["time_embed.0.weight"]), h(sd["time_embed.0.bias"])),
              "te2": (h(sd["time_embed.2.weight"]), h(sd["time_embed.2.bias"])),
              "ln_f": (h(sd["transformer.final_layernorm.weight"]), h(sd["transformer.final_layernorm.bias"])),
              "norm_final": (sd["mixins.final_layer.norm_final.weight"].to(dev, torch.float32), sd["mixins.final_layer.norm_final.bias"].to(dev, torch.float32)),
              "ada_f": (h(sd["mixins.final_layer.adaLN_modulation.1.weight"]), h(sd["mixins.final_layer.adaLN_modulation.1.bias"])),
              "lin_f": (h(sd["mixins.final_layer.linear.weight"]), h(sd["mixins.final_layer.linear.bias"]))}
        self._pk = pk
        return pk

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, shard=None, **unused):
        """shard: this rank's parallel.SeqShard to run the layers token-sharded over its group (see parallel.py); the
        returned output is the whole one on every rank of the group"""
        if shard is not None:
            return self._forward_shard(x, timesteps, context, shard)
        pk = self._pk if self._pk is not None else self._pack()
        c, dt = self.cfg, self.dtype
        b, t, cin, hh, ww = x.shape
        p, d, tl = c["patch"], c["hidden"], self.text_length
        gh, gw = hh // p, ww // p
        assert (t, gh, gw) == (self.frames, self.gh, self.gw) and cin == 2 * c["in_channels"] and context.shape[1] == tl
        n_img = t * gh * gw
        S = tl + n_img
        # ---- embeddings: patch conv (kernel = stride = patch) as a GEMM over (c, p, q) columns; text projection
        cols = x.to(dt).reshape(b, t, cin, gh, p, gw, p).permute(0, 1, 3, 5, 2, 4, 6).reshape(b * n_img, cin * p * p).contiguous()
        hidden = torch.empty((b, S, d), dtype=dt, device=x.device)
        h2 = hidden.view(b * S, d)
        ctx2 = context.to(dt).reshape(b * tl, -1).contiguous()
        for bi in range(b):
            ops.linear(ctx2[bi * tl:(bi + 1) * tl], *pk["text"], out=h2[bi * S:bi * S + tl])
            ops.linear(cols[bi * n_img:(bi + 1) * n_img], *pk["patch"], out=h2[bi * S + tl:(bi + 1) * S])
        # ---- time embedding: sinusoidal (cos || sin, sgm timestep_embedding) -> Linear -> SiLU -> Linear
        e = ops.sinusoidal(timesteps.to(x.device), d, dtype=dt)
        e = ops.linear(e, *pk["te0"], flags=ops.FLAG_SILU_OUT)
        emb = ops.linear(e, *pk["te2"])
        # ---- 42 layers
        for layer in pk["layers"]:
            hidden = layer.forward(hidden, emb)
        # ---- final LayerNorm (transformer.py:629) -> final layer (dit_video_concat.py:397-412) on the image tokens
        h2 = hidden.reshape(b * S, d)
        mod = ops.linear(ops.silu(emb), *pk["ada_f"])                               # (b, 2 d): shift | scale
        out = torch.empty((b * n_img, p * p * c["out_channels"]), dtype=dt, device=x.device)
        g, be = pk["norm_final"]
        for bi in range(b):
            img = ops.layernorm(h2[bi * S + tl:(bi + 1) * S], *pk["ln_f"], eps=self.ln_eps)
            shift, scale = mod[bi, :d].float(), mod[bi, d:].float()
            img = ops.layernorm(img, (g * (1 + scale)).to(dt), (be * (1 + scale) + shift).to(dt), eps=1e-6)
            ops.linear(img, *pk["lin_f"], out=out[bi * n_img:(bi + 1) * n_img])
        co = c["out_channels"]                                                     # "b (t h w) (c p q) -> b t c (h p) (w q)"
        return out.view(b, t, gh, gw, co, p, p).permute(0, 1, 4, 2, 5, 3, 6).reshape(b, t, co, gh * p, gw * p)

    def _forward_shard(self, x, timesteps, context, sp):
        """``forward`` with the token rows sp.me of every sample on this rank; one all-gather of the image-token outputs at
        the end hands every rank the whole output"""
        pk = self._pk if self._pk is not None else self._pack()
        c, dt, me = self.cfg, self.dtype, sp.me
        b, t, cin, hh, ww = x.shape
        p, d, tl = c["patch"], c["hidden"], self.text_length
        gh, gw = hh // p, ww // p
        assert (t, gh, gw) == (self.frames, self.gh, self.gw) and cin == 2 * c["in_channels"] and context.shape[1] == tl
        n_img, n, nt, ni = t * gh * gw, me.rows, me.text_rows, me.image_rows
        i0 = me.start + nt - tl                                                     # first image token of the shard
        # ---- embeddings of the shard's text and image tokens
        cols = x.to(dt).reshape(b, t, cin, gh, p, gw, p).permute(0, 1, 3, 5, 2, 4, 6).reshape(b * n_img, cin * p * p).contiguous()
        hidden = torch.empty((b, n, d), dtype=dt, device=x.device)
        h2 = hidden.view(b * n, d)
        ctx2 = context.to(dt).reshape(b * tl, -1).contiguous()
        for bi in range(b):
            if nt:
                ops.linear(ctx2[bi * tl + me.start:bi * tl + me.start + nt], *pk["text"], out=h2[bi * n:bi * n + nt])
            if ni:
                ops.linear(cols[bi * n_img + i0:bi * n_img + i0 + ni], *pk["patch"], out=h2[bi * n + nt:(bi + 1) * n])
        e = ops.sinusoidal(timesteps.to(x.device), d, dtype=dt)
        e = ops.linear(e, *pk["te0"], flags=ops.FLAG_SILU_OUT)
        emb = ops.linear(e, *pk["te2"])
        for layer in pk["layers"]:
            hidden = layer.forward_shard(hidden, emb, sp)
        # ---- final layer on the shard's image tokens, then one all-gather of them
        h2 = hidden.reshape(b * n, d)
        mod = ops.linear(ops.silu(emb), *pk["ada_f"])
        out = torch.empty((b, ni, p * p * c["out_channels"]), dtype=dt, device=x.device)
        g, be = pk["norm_final"]
        for bi in range(b):
            if not ni:
                continue
            img = ops.layernorm(h2[bi * n + nt:(bi + 1) * n], *pk["ln_f"], eps=self.ln_eps)
            shift, scale = mod[bi, :d].float(), mod[bi, d:].float()
            img = ops.layernorm(img, (g * (1 + scale)).to(dt), (be * (1 + scale) + shift).to(dt), eps=1e-6)
            ops.linear(img, *pk["lin_f"], out=out[bi])
        out = sp.gather_image_rows(out.transpose(0, 1)).transpose(0, 1)             # (b, n_img, p*p*co)
        co = c["out_channels"]
        return out.reshape(b, t, gh, gw, co, p, p).permute(0, 1, 4, 2, 5, 3, 6).reshape(b, t, co, gh * p, gw * p)
