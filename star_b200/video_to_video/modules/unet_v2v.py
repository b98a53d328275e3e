"""STAR denoiser (3-D UNet + VideoControlNet with LIEM gates) on sm_90a kernels.

Drop-in for the model surface of the reference's
video_to_video/modules/unet_v2v.py: the classes below keep the reference's
names, constructor meaning and -- crucially -- its parameter tree, so a
reference checkpoint loads with ``load_state_dict`` unchanged (2 247 tensors
for the default config, including the ``temopral_conv`` spelling, ref :651).

Execution is completely different from the reference.  ``nn`` layers are only
parameter containers; the forward pass keeps every activation as an fp16
channels-last token matrix X[(b t h w), C] and is a sequence of calls into
libstar_sm100.so (star_b200/ops.py): wgmma implicit-GEMM convolutions /
linears with fused bias + time-embedding + residual + GEGLU epilogues, a
wgmma flash attention for the H*W-token spatial attention, a temporal
attention kernel over T, and 128-bit-vectorised GroupNorm / LayerNorm(+LIEM)
kernels.  The (b t)(h w) c <-> (b h w) t c rearranges of the reference
(ref :307,:314,:1045-1086) do not exist: both are stride views of the same
buffer.

Weights are repacked once after loading (``_pack``): conv kernels to
[Cout, kh, kw, Cin], q/k/v concatenated, all time-embedding projections and
all text K/V projections concatenated into one GEMM each.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F  # noqa: F401  (re-exported: callers of the reference rely on it)
from einops import rearrange  # noqa: F401  (re-exported, see SURVEY 8b)

from ... import ops

HALF = torch.float16

__all__ = [
    "sinusoidal_embedding", "zero_module", "exists", "default", "MemoryEfficientCrossAttention",
    "SpatialTransformer", "SpatialAttention", "TemporalLocalAttention", "BasicTransformerBlock", "GEGLU",
    "FeedForward", "Upsample", "ResBlock", "Downsample", "TemporalTransformer", "TemporalConvBlock_v2",
    "Vid2VidSDUNet", "ControlledV2VUNet", "VideoControlNet", "TimestepBlock", "TimestepEmbedSequential",
    "rearrange", "math", "torch", "nn", "F",
]


def exists(x):
    return x is not None


def default(val, d):
    if exists(val):
        return val
    return d() if callable(d) else d


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def sinusoidal_embedding(timesteps, dim):
    """cos || sin embedding (ref :96-108); host-side helper kept for API parity.
    The model itself uses the fused device kernel (ops.sinusoidal)."""
    half = dim // 2
    timesteps = timesteps.float()
    freqs = torch.pow(10000, -torch.arange(half).to(timesteps).div(half))
    ang = torch.outer(timesteps, freqs)
    x = torch.cat([torch.cos(ang), torch.sin(ang)], dim=1)
    if dim % 2 != 0:
        x = torch.cat([x, torch.zeros_like(x[:, :1])], dim=1)
    return x


def _h(t):
    return t.detach().to(HALF).contiguous()


class _Ctx:
    """Per-forward state shared by the blocks of one network (UNet or ControlNet)."""
    __slots__ = ("B", "T", "temb", "text_kv", "context_rows")

    def __init__(self, B, T):
        self.B, self.T = B, T
        self.temb = None          # [B, sum Cout] fp16: every ResBlock's emb_layers output, one GEMM
        self.text_kv = None       # [B*77, sum 2C] fp16: every spatial block's text K|V, one GEMM
        self.context_rows = 0


# ----------------------------------------------------------------------------------------------
# attention / transformer blocks
# ----------------------------------------------------------------------------------------------
class MemoryEfficientCrossAttention(nn.Module):
    """Parameter layout of ref :134-156 (to_q/to_k/to_v bias-free, to_out.0 biased)."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, max_bs=16384, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = default(context_dim, query_dim)
        self.heads, self.dim_head, self.max_bs = heads, dim_head, max_bs
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))


class SpatialAttention(nn.Module):
    """Spatial LIEM gate (ref :380-394): 7x7 conv over [max_c, mean_c]."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(2, 1, kernel_size=7, padding=3, bias=False)
        self.sigmoid = nn.Sigmoid()


class TemporalLocalAttention(nn.Module):
    """Temporal LIEM gate (ref :396-411): Linear(2->1) over [max_c, mean_c]."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Linear(2, 1, bias=False)
        self.sigmoid = nn.Sigmoid()


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.0):
        super().__init__()
        inner = int(dim * mult)
        dim_out = default(dim_out, dim)
        if not glu:
            raise NotImplementedError("STAR only instantiates the GEGLU feed-forward (ref :438)")
        self.net = nn.Sequential(GEGLU(dim, inner), nn.Dropout(dropout), nn.Linear(inner, dim_out))

    def run(self, x, residual):
        """x = LN3 output; returns ff(x) + residual  (ref :477/:490)."""
        g = ops.linear(x, self._w_in, self._b_in, flags=ops.FLAG_GEGLU)
        return ops.linear(g, self._w_out, self._b_out, residual=residual)

    def _pack(self):
        self._w_in, self._b_in = _h(self.net[0].proj.weight), _h(self.net[0].proj.bias)
        self._w_out, self._b_out = _h(self.net[2].weight), _h(self.net[2].bias)


class BasicTransformerBlock(nn.Module):
    """ref :414-492.  'space': LIEM -> LN -> self-attn, LN -> text cross-attn, LN -> FF.
    'temp': LIEM -> LN -> self-attn(T), LIEM -> LN -> self-attn(T), LN -> FF."""

    def __init__(self, dim, n_heads, d_head, dropout=0.0, context_dim=None, gated_ff=True, checkpoint=True,
                 disable_self_attn=False, local_type=None, is_ctrl=False):
        super().__init__()
        if not is_ctrl or local_type not in ("space", "temp") or disable_self_attn:
            raise NotImplementedError("STAR builds every block with is_ctrl=True and a local_type (ref :1367,:1403)")
        self.local_type, self.is_ctrl, self.disable_self_attn = local_type, is_ctrl, disable_self_attn
        self.dim, self.n_heads = dim, n_heads
        self.attn1 = MemoryEfficientCrossAttention(dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = MemoryEfficientCrossAttention(dim, context_dim=context_dim, heads=n_heads, dim_head=d_head,
                                                   dropout=dropout)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)
        self.checkpoint = checkpoint
        if local_type == "space":
            self.local1 = SpatialAttention()
        else:
            self.local1 = TemporalLocalAttention()
            self.local2 = TemporalLocalAttention()

    def _pack(self):
        a1, a2 = self.attn1, self.attn2
        self._qkv1 = _h(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], dim=0))
        self._o1_w, self._o1_b = _h(a1.to_out[0].weight), _h(a1.to_out[0].bias)
        self._o2_w, self._o2_b = _h(a2.to_out[0].weight), _h(a2.to_out[0].bias)
        self._ln = [(_h(n.weight), _h(n.bias)) for n in (self.norm1, self.norm2, self.norm3)]
        if self.local_type == "space":
            self._q2 = _h(a2.to_q.weight)
            self._liem = _h(self.local1.conv1.weight.reshape(-1))           # [2*7*7]
        else:
            self._qkv2 = _h(torch.cat([a2.to_q.weight, a2.to_k.weight, a2.to_v.weight], dim=0))
            w1 = self.local1.conv1.weight.detach().to(HALF).float().reshape(-1).tolist()
            w2 = self.local2.conv1.weight.detach().to(HALF).float().reshape(-1).tolist()
            self._liem_t = (w1, w2)
        self.ff._pack()

    def text_kv_weight(self):
        """[2C, context_dim] rows = to_k | to_v of the text cross-attention."""
        return torch.cat([self.attn2.to_k.weight, self.attn2.to_v.weight], dim=0)

    def run_space(self, ctx, x, H, W, kv):
        return self.run_space_back(ctx, *self.run_space_front(ctx, x, H, W), H, W, kv)

    def run_space_front(self, ctx, x, H, W):
        """Everything of the 'space' block that does not see the text: LIEM -> LN -> self-attention (+x) -> LN -> q of the text
        cross-attention.  Identical for the two CFG branches of a solver step (same x, t, hint; only y differs)."""
        BT, C, heads = ctx.B * ctx.T, self.dim, self.n_heads
        HW = H * W
        gate = ops.liem_spatial_gate(x, self._liem, BT, H, W)
        n = ops.layernorm(x, *self._ln[0], gate_mode=1, gate=gate)
        qkv = ops.linear(n, self._qkv1)
        a = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], BT, heads, HW, HW, 1, 0.125)
        x = ops.linear(a, self._o1_w, self._o1_b, residual=x)
        n = ops.layernorm(x, *self._ln[1])
        return x, ops.linear(n, self._q2)

    def run_space_back(self, ctx, x, q, H, W, kv):
        BT, heads = ctx.B * ctx.T, self.n_heads
        k, v = kv
        a = ops.attention(q, k, v, BT, heads, H * W, ctx.context_rows, ctx.T, 0.125)
        x = ops.linear(a, self._o2_w, self._o2_b, residual=x)
        n = ops.layernorm(x, *self._ln[2])
        return self.ff.run(n, x)

    def run_temp(self, ctx, x, HW):
        C, heads = self.dim, self.n_heads
        (w10, w11), (w20, w21) = self._liem_t
        n = ops.layernorm(x, *self._ln[0], gate_mode=2, w0=w10, w1=w11)
        qkv = ops.linear(n, self._qkv1)
        a = ops.temporal_attention(qkv, ctx.B, ctx.T, HW, heads, C, 0.125)
        x = ops.linear(a, self._o1_w, self._o1_b, residual=x)
        n = ops.layernorm(x, *self._ln[1], gate_mode=2, w0=w20, w1=w21)
        qkv = ops.linear(n, self._qkv2)
        a = ops.temporal_attention(qkv, ctx.B, ctx.T, HW, heads, C, 0.125)
        x = ops.linear(a, self._o2_w, self._o2_b, residual=x)
        n = ops.layernorm(x, *self._ln[2])
        return self.ff.run(n, x)


class SpatialTransformer(nn.Module):
    """ref :242-317 (use_linear=True): GN(eps 1e-6) -> Linear -> block -> Linear -> +x."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None,
                 disable_self_attn=False, use_linear=False, use_checkpoint=True, is_ctrl=False):
        super().__init__()
        if not use_linear or depth != 1:
            raise NotImplementedError("STAR uses use_linear=True, depth=1 (ref :1395-1404)")
        if isinstance(context_dim, list):
            context_dim = context_dim[0]
        inner = n_heads * d_head
        self.in_channels, self.inner = in_channels, inner
        self.norm = nn.GroupNorm(32, in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(
            inner, n_heads, d_head, dropout=dropout, context_dim=context_dim, disable_self_attn=disable_self_attn,
            checkpoint=use_checkpoint, local_type="space", is_ctrl=is_ctrl)])
        self.proj_out = zero_module(nn.Linear(in_channels, inner))
        self.use_linear = use_linear

    def _pack(self):
        self._gn = (_h(self.norm.weight), _h(self.norm.bias))
        self._in = (_h(self.proj_in.weight), _h(self.proj_in.bias))
        self._out = (_h(self.proj_out.weight), _h(self.proj_out.bias))
        self.transformer_blocks[0]._pack()

    def run(self, ctx, x, H, W, kv):
        return self.run_back(ctx, self.run_front(ctx, x, H, W), H, W, kv)

    def run_front(self, ctx, x, H, W):
        h = ops.groupnorm(x, *self._gn, ctx.B * ctx.T, 1e-6, False)
        h = ops.linear(h, *self._in)
        return (x,) + self.transformer_blocks[0].run_space_front(ctx, h, H, W)

    def run_back(self, ctx, front, H, W, kv):
        x, h, q = front
        h = self.transformer_blocks[0].run_space_back(ctx, h, q, H, W, kv)
        return ops.linear(h, *self._out, residual=x)


class TemporalTransformer(nn.Module):
    """ref :970-1092 (use_linear=False, only_self_att=True): 5-D GN over the whole clip ->
    Conv1d k=1 -> block over T -> Conv1d k=1 -> +x."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None,
                 disable_self_attn=False, use_linear=False, use_checkpoint=True, only_self_att=True,
                 multiply_zero=False, is_ctrl=False):
        super().__init__()
        if use_linear or not only_self_att or depth != 1 or multiply_zero:
            raise NotImplementedError("STAR uses the Conv1d, self-attention-only temporal transformer (ref :1358-1368)")
        inner = n_heads * d_head
        self.in_channels, self.inner = in_channels, inner
        self.only_self_att, self.multiply_zero, self.use_linear = only_self_att, multiply_zero, use_linear
        self.norm = nn.GroupNorm(32, in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Conv1d(in_channels, inner, kernel_size=1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(
            inner, n_heads, d_head, dropout=dropout, context_dim=None, checkpoint=use_checkpoint,
            local_type="temp", is_ctrl=is_ctrl)])
        self.proj_out = zero_module(nn.Conv1d(inner, in_channels, kernel_size=1))

    def _pack(self):
        self._gn = (_h(self.norm.weight), _h(self.norm.bias))
        self._in = (_h(self.proj_in.weight.squeeze(-1)), _h(self.proj_in.bias))
        self._out = (_h(self.proj_out.weight.squeeze(-1)), _h(self.proj_out.bias))
        self.transformer_blocks[0]._pack()

    def run(self, ctx, x, HW):
        h = ops.groupnorm(x, *self._gn, ctx.B, 1e-6, False)       # statistics over (C/32, T, H, W)
        h = ops.linear(h, *self._in)
        h = self.transformer_blocks[0].run_temp(ctx, h, HW)
        return ops.linear(h, *self._out, residual=x)


# ----------------------------------------------------------------------------------------------
# convolutional blocks
# ----------------------------------------------------------------------------------------------
def _w9(conv):
    return _h(conv.weight.permute(0, 2, 3, 1))                   # [Cout, kh, kw, Cin]


class Upsample(nn.Module):
    """nearest x2, drop first/last row, conv3x3 (ref :532-567, dims=2.0 path)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels, self.out_channels = channels, out_channels or channels
        self.use_conv, self.dims = use_conv, dims
        if use_conv:
            self.conv = nn.Conv2d(self.channels, self.out_channels, 3, padding=padding)

    def _pack(self):
        self._w, self._b = _w9(self.conv), _h(self.conv.bias)

    def run(self, ctx, x, H, W):
        BT = ctx.B * ctx.T
        up = ops.upsample2x_crop(x, BT, H, W)
        Ho, Wo = 2 * H - 2, 2 * W
        return ops.conv2d_3x3(up.view(BT, Ho, Wo, self.channels), self._w, self._b), Ho, Wo


class Downsample(nn.Module):
    """conv3x3 stride 2 padding (2, 1) (ref :695-729)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=(2, 1)):
        super().__init__()
        if not use_conv:
            raise NotImplementedError("STAR only uses the convolutional Downsample (ref :1435)")
        self.channels, self.out_channels = channels, out_channels or channels
        self.op = nn.Conv2d(self.channels, self.out_channels, 3, stride=2, padding=padding)

    def _pack(self):
        self._w, self._b = _w9(self.op), _h(self.op.bias)

    def run(self, ctx, x, H, W):
        return ops.conv2d_3x3_s2(x.view(ctx.B * ctx.T, H, W, self.channels), self._w, self._b)


class TemporalConvBlock_v2(nn.Module):
    """4 x [5-D GroupNorm + SiLU + Conv3d(3,1,1)] + identity (ref :1194-1278, default branch)."""

    def __init__(self, in_dim, out_dim=None, dropout=0.0, use_image_dataset=False):
        super().__init__()
        out_dim = out_dim or in_dim
        self.in_dim, self.out_dim = in_dim, out_dim
        self.conv1 = nn.Sequential(nn.GroupNorm(32, in_dim), nn.SiLU(),
                                   nn.Conv3d(in_dim, out_dim, (3, 1, 1), padding=(1, 0, 0)))
        for name in ("conv2", "conv3", "conv4"):
            setattr(self, name, nn.Sequential(nn.GroupNorm(32, out_dim), nn.SiLU(), nn.Dropout(dropout),
                                              nn.Conv3d(out_dim, in_dim, (3, 1, 1), padding=(1, 0, 0))))
        nn.init.zeros_(self.conv4[-1].weight)
        nn.init.zeros_(self.conv4[-1].bias)

    def _pack(self):
        self._stages = []
        for seq in (self.conv1, self.conv2, self.conv3, self.conv4):
            gn, conv = seq[0], seq[-1]
            w3 = _h(conv.weight[:, :, :, 0, 0].permute(0, 2, 1))          # [Cout, 3, Cin]
            self._stages.append((_h(gn.weight), _h(gn.bias), w3, _h(conv.bias)))

    def run(self, ctx, x, HW):
        h = x
        for i, (g, b, w3, bias) in enumerate(self._stages):
            h = ops.groupnorm(h, g, b, ctx.B, 1e-5, True)           # clip-wide statistics
            h = ops.conv_t3(h, w3, bias, x if i == 3 else None, ctx.B, ctx.T, HW)
        return h


class ResBlock(nn.Module):
    """ref :570-692 (no up/down, no scale-shift norm, temporal conv on)."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False,
                 use_scale_shift_norm=False, dims=2, up=False, down=False, use_temporal_conv=True,
                 use_image_dataset=False):
        super().__init__()
        if up or down or use_scale_shift_norm or use_conv or not use_temporal_conv:
            raise NotImplementedError("configuration not used by STAR (ref :1384-1391)")
        self.channels, self.emb_channels = channels, emb_channels
        self.out_channels = out_channels or channels
        self.in_layers = nn.Sequential(nn.GroupNorm(32, channels), nn.SiLU(),
                                       nn.Conv2d(channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(nn.GroupNorm(32, self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(nn.Conv2d(self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = nn.Conv2d(channels, self.out_channels, 1)
        self.temopral_conv = TemporalConvBlock_v2(self.out_channels, self.out_channels, dropout=0.1,
                                                  use_image_dataset=use_image_dataset)
        self._temb_slice = None

    def _pack(self):
        self._gn1 = (_h(self.in_layers[0].weight), _h(self.in_layers[0].bias))
        self._c1 = (_w9(self.in_layers[2]), _h(self.in_layers[2].bias))
        self._gn2 = (_h(self.out_layers[0].weight), _h(self.out_layers[0].bias))
        self._c2 = (_w9(self.out_layers[3]), _h(self.out_layers[3].bias))
        if isinstance(self.skip_connection, nn.Conv2d):
            self._skip = (_h(self.skip_connection.weight[:, :, 0, 0]), _h(self.skip_connection.bias))
        else:
            self._skip = None
        self.temopral_conv._pack()

    def run(self, ctx, x, H, W):
        BT, HW = ctx.B * ctx.T, H * W
        lo, hi = self._temb_slice
        temb = ctx.temb[:, lo:hi]                          # column slice of the one time-embedding GEMM: passed with its row pitch
        h = ops.groupnorm(x, *self._gn1, BT, 1e-5, True)
        h = ops.conv2d_3x3(h.view(BT, H, W, self.channels), *self._c1, rowvec=temb, rowvec_div=ctx.T * HW)
        h = ops.groupnorm(h, *self._gn2, BT, 1e-5, True)
        skip = x if self._skip is None else ops.linear(x, *self._skip)
        h = ops.conv2d_3x3(h.view(BT, H, W, self.out_channels), *self._c2, residual=skip)
        return self.temopral_conv.run(ctx, h, HW)


class TimestepBlock(nn.Module):
    pass


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """Wrapper the ControlNet uses around its zero 1x1 convs (ref :2130-2132, :2305-2319)."""


# ----------------------------------------------------------------------------------------------
# networks
# ----------------------------------------------------------------------------------------------
class _UNetBase(nn.Module):
    """Shared builder/runner of the encoder + middle block (identical in Vid2VidSDUNet, ref
    :1351-1488, and VideoControlNet, ref :1983-2118)."""

    def _build_trunk(self, in_dim, dim, context_dim, dim_mult, num_heads, head_dim, num_res_blocks, attn_scales,
                     dropout, use_checkpoint):
        embed_dim = dim * 4
        self.time_embed = nn.Sequential(nn.Linear(dim, embed_dim), nn.SiLU(), nn.Linear(embed_dim, embed_dim))
        enc_dims = [dim * u for u in [1] + list(dim_mult)]
        shortcut_dims, scale = [dim], 1.0

        def tt(c, heads):
            return TemporalTransformer(c, heads, head_dim, depth=1, context_dim=context_dim, use_linear=False,
                                       use_checkpoint=use_checkpoint, multiply_zero=False, is_ctrl=True)

        def st(c):
            return SpatialTransformer(c, c // head_dim, head_dim, depth=1, context_dim=context_dim,
                                      disable_self_attn=False, use_linear=True, use_checkpoint=use_checkpoint,
                                      is_ctrl=True)

        self.input_blocks = nn.ModuleList()
        self.input_blocks.append(nn.ModuleList([nn.Conv2d(in_dim, dim, 3, padding=1), tt(dim, num_heads)]))
        for i, (cin, cout) in enumerate(zip(enc_dims[:-1], enc_dims[1:])):
            for j in range(num_res_blocks):
                block = nn.ModuleList([ResBlock(cin, embed_dim, dropout, out_channels=cout)])
                if scale in attn_scales:
                    block.append(st(cout))
                    block.append(tt(cout, cout // head_dim))
                cin = cout
                self.input_blocks.append(block)
                shortcut_dims.append(cout)
                if i != len(dim_mult) - 1 and j == num_res_blocks - 1:
                    self.input_blocks.append(Downsample(cout, True, dims=2, out_channels=cout))
                    shortcut_dims.append(cout)
                    scale /= 2.0
        self.middle_block = nn.ModuleList([ResBlock(cout, embed_dim, dropout), st(cout), tt(cout, cout // head_dim),
                                           ResBlock(cout, embed_dim, dropout)])
        return shortcut_dims, scale, cout, st, tt

    # -- packing -------------------------------------------------------------------------------
    def _pack_trunk(self):
        te = self.time_embed
        self._te = (_h(te[0].weight), _h(te[0].bias), _h(te[2].weight), _h(te[2].bias))
        conv0 = self.input_blocks[0][0]
        self._stem = (_w9(conv0), _h(conv0.bias))
        res, spatial = [], []
        trunk = [self.input_blocks, self.middle_block]
        if hasattr(self, "output_blocks"):
            trunk.append(self.output_blocks)
        for part in trunk:                    # NOT self.modules(): the UNet owns the ControlNet as a child
            for m in part.modules():
                if isinstance(m, (ResBlock, SpatialTransformer, TemporalTransformer, Upsample, Downsample)):
                    m._pack()
                if isinstance(m, ResBlock):
                    res.append(m)
                if isinstance(m, SpatialTransformer):
                    spatial.append(m)
        # one GEMM for every ResBlock's emb_layers Linear (ref :626-633)
        off, ws, bs = 0, [], []
        for m in res:
            lin = m.emb_layers[1]
            m._temb_slice = (off, off + lin.out_features)
            off += lin.out_features
            ws.append(lin.weight)
            bs.append(lin.bias)
        self._temb_w, self._temb_b = _h(torch.cat(ws, 0)), _h(torch.cat(bs, 0))
        # one GEMM for every spatial block's text to_k | to_v (ref :161-162; the context is identical for all
        # frames of a clip, :1769, so it is projected once per clip instead of once per frame)
        off, ws = 0, []
        self._kv_slices = {}
        for m in spatial:
            w = m.transformer_blocks[0].text_kv_weight()
            c = w.shape[0] // 2
            self._kv_slices[id(m)] = (off, off + c, off + 2 * c)
            off += 2 * c
            ws.append(w)
        self._kv_w = _h(torch.cat(ws, 0))
        self._packed = True

    def _ensure_packed(self):
        if not getattr(self, "_packed", False):
            self._pack_all()

    # any dtype/device move or weight load invalidates the packed copies
    def _apply(self, fn, *a, **k):
        self._packed = False
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._packed = False
        return super()._load_from_state_dict(*a, **k)

    def _begin_time(self, t, B, T):
        """time embedding of every ResBlock of this network (one GEMM); returns ctx without the text part."""
        ctx = _Ctx(B, T)
        e = ops.sinusoidal(t, self.dim)
        w0, b0, w1, b1 = self._te
        e = ops.linear(e, w0, b0, flags=ops.FLAG_SILU_OUT)
        e = ops.linear(e, w1, b1, flags=ops.FLAG_SILU_OUT)         # = SiLU(time_embed(..)), input of every emb_layers
        ctx.temb = ops.linear(e, self._temb_w, self._temb_b)
        return ctx

    def _with_text(self, ctx, y):
        """a copy of ctx carrying the text K/V of every spatial block for the embedding y (one GEMM)"""
        c = _Ctx(ctx.B, ctx.T)
        c.temb = ctx.temb
        y16 = y.to(HALF).reshape(-1, y.shape[-1]).contiguous()
        c.context_rows = y.shape[1]
        c.text_kv = ops.linear(y16, self._kv_w)
        return c

    def _begin(self, t, y, B, T):
        """time embedding + text K/V for this network; returns ctx."""
        return self._with_text(self._begin_time(t, B, T), y)

    # -- the part of the encoder that never sees the text ---------------------------------------------------------------------
    # stem output -> temporal transformer of input_blocks[0] -> ResBlock and the front of the SpatialTransformer of
    # input_blocks[1].  The two CFG branches of a solver step call the network with the same (x, t, hint) and different y
    # (diffusion_sdedit.py:81,88), so this prefix -- incl. one finest-level self-attention -- is evaluated ONCE for both.
    def _prefix_splittable(self):
        b1 = self.input_blocks[1]
        return (isinstance(b1, nn.ModuleList) and len(b1) == 3 and isinstance(b1[0], ResBlock)
                and isinstance(b1[1], SpatialTransformer) and isinstance(b1[2], TemporalTransformer))

    def _run_prefix(self, ctx, h, H, W):
        """h = stem output.  Returns (h0, front): h0 = output of input_blocks[0], front = state of block 1 at the split point."""
        h0 = self.input_blocks[0][1].run(ctx, h, H * W)
        b1 = self.input_blocks[1]
        r = b1[0].run(ctx, h0, H, W)
        return h0, b1[1].run_front(ctx, r, H, W)

    def _finish_block1(self, ctx, front, H, W):
        b1 = self.input_blocks[1]
        h = b1[1].run_back(ctx, front, H, W, self._kv(ctx, b1[1]))
        return b1[2].run(ctx, h, H * W)

    def _kv(self, ctx, m):
        a, b, c = self._kv_slices[id(m)]
        return ctx.text_kv[:, a:b], ctx.text_kv[:, b:c]

    def _run_block(self, ctx, block, x, H, W):
        if isinstance(block, Downsample):
            x, H, W = block.run(ctx, x, H, W)
            return x, H, W
        for m in block:
            if isinstance(m, ResBlock):
                x = m.run(ctx, x, H, W)
            elif isinstance(m, SpatialTransformer):
                x = m.run(ctx, x, H, W, self._kv(ctx, m))
            elif isinstance(m, TemporalTransformer):
                x = m.run(ctx, x, H * W)
            elif isinstance(m, Upsample):
                x, H, W = m.run(ctx, x, H, W)
            else:
                raise TypeError(type(m))
        return x, H, W


class Vid2VidSDUNet(_UNetBase):
    """ref :1281-1709.  Constructor arguments keep the reference's names; only the values STAR
    uses are supported."""

    def __init__(self, in_dim=4, dim=320, y_dim=1024, context_dim=1024, out_dim=4, dim_mult=[1, 2, 4, 4],
                 num_heads=8, head_dim=64, num_res_blocks=2, attn_scales=[1 / 1, 1 / 2, 1 / 4],
                 use_scale_shift_norm=True, dropout=0.1, temporal_attn_times=1, temporal_attention=True,
                 use_checkpoint=True, use_image_dataset=False, use_fps_condition=False, use_sim_mask=False,
                 training=False, inpainting=True):
        super().__init__()
        if not temporal_attention or use_image_dataset or use_fps_condition:
            raise NotImplementedError("configuration not used by STAR")
        self.in_dim, self.dim, self.y_dim, self.context_dim = in_dim, dim, y_dim, context_dim
        self.embed_dim, self.out_dim, self.dim_mult = dim * 4, out_dim, list(dim_mult)
        self.num_heads = num_heads if num_heads else dim // 32
        self.head_dim, self.num_res_blocks, self.attn_scales = head_dim, num_res_blocks, list(attn_scales)
        self.temporal_attention, self.use_checkpoint = temporal_attention, use_checkpoint
        shortcut_dims, scale, cout, st, tt = self._build_trunk(
            in_dim, dim, context_dim, dim_mult, self.num_heads, head_dim, num_res_blocks, attn_scales, dropout,
            use_checkpoint)
        dec_dims = [dim * u for u in [dim_mult[-1]] + list(dim_mult[::-1])]
        self.output_blocks = nn.ModuleList()
        for i, (cin, co) in enumerate(zip(dec_dims[:-1], dec_dims[1:])):
            for j in range(num_res_blocks + 1):
                block = nn.ModuleList([ResBlock(cin + shortcut_dims.pop(), self.embed_dim, dropout, co)])
                if scale in attn_scales:
                    block.append(st(co))
                    block.append(tt(co, co // head_dim))
                cin = co
                if i != len(dim_mult) - 1 and j == num_res_blocks:
                    block.append(Upsample(co, True, dims=2.0, out_channels=co))
                    scale *= 2.0
                self.output_blocks.append(block)
        self.out = nn.Sequential(nn.GroupNorm(32, co), nn.SiLU(), nn.Conv2d(co, self.out_dim, 3, padding=1))
        nn.init.zeros_(self.out[-1].weight)
        self._packed = False

    def _pack_all(self):
        self._pack_trunk()
        self._head = (_h(self.out[0].weight), _h(self.out[0].bias), _w9(self.out[2]), _h(self.out[2].bias))
        cn = getattr(self, "VideoControlNet", None)
        if cn is not None:
            cn._pack_all()


class ControlledV2VUNet(Vid2VidSDUNet):
    """The STAR denoiser: UNet + VideoControlNet (ref :1712-1893).  ``ControlledV2VUNet()`` with no
    arguments is the reference configuration; keyword arguments (dim_mult, num_res_blocks) exist
    for reduced test models."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.VideoControlNet = VideoControlNet(**kw)

    @torch.no_grad()
    def forward(self, x, t, y, hint=None, variant_info=None, hint_chunk=None, t_hint=None, s_cond=None,
                mask_cond=None, x_lr=None, fps=None, mask=None, video_mask=None, focus_present_mask=None,
                prob_focus_present=0.0, mask_last_frame_num=0):
        """x: (B,4,F,h,w) latent (any float dtype), t: (B,) long, y: (B,77,1024) text embedding,
        hint / hint_chunk: (B,4,F,h,w) LR latent.  Returns the v-prediction (B,4,F,h,w) in fp16,
        like the reference's ``.half()`` model under autocast (ref :1717-1809)."""
        if hint_chunk is not None:
            hint = hint_chunk                                              # ref :1743-1744
        return self._forward_branches(x, t, (y,), hint)[0]

    @torch.no_grad()
    def forward_cfg_pair(self, x, t, y_pair, hint=None, hint_chunk=None, variant_info=None):
        """Both classifier-free-guidance branches of one solver step: ``(forward(x, t, y_pair[0], hint), forward(x, t, y_pair[1],
        hint))`` bit for bit, with the text-independent prefix of both networks (stem, first temporal transformer, first ResBlock,
        and the first spatial block up to the query of its text cross-attention -- one finest-level self-attention per network)
        evaluated once.  The reference makes two full calls (diffusion_sdedit.py:81,88)."""
        if hint_chunk is not None:
            hint = hint_chunk
        return tuple(self._forward_branches(x, t, tuple(y_pair), hint))

    def _forward_branches(self, x, t, ys, hint):
        if hint is None:
            raise ValueError("ControlledV2VUNet needs the LR latent (hint / hint_chunk)")
        self._ensure_packed()
        B, _, T, H0, W0 = x.shape
        if H0 % 8 != 2 or W0 % 8 != 0:
            raise ValueError(f"latent {H0}x{W0}: H must be 2 (mod 8) and W 0 (mod 8) for the UNet's "
                             "down/up-sampling to close (ref :709, :564)")
        t = t.to(x.device)
        xt = ops.nchw5_to_tokens(x)
        ht = ops.nchw5_to_tokens(hint)
        BT = B * T
        cn = self.VideoControlNet
        share = len(ys) > 1 and self._prefix_splittable() and cn._prefix_splittable()
        base = self._begin_time(t, B, T)
        cn_shared = cn.run_shared(xt, ht, t, B, T, H0, W0) if share else None
        if share:
            h = ops.conv2d_3x3_c4(xt.view(BT, H0, W0, self.in_dim), *self._stem)
            h0, front = self._run_prefix(base, h, H0, W0)
        outs = []
        for y in ys:
            H, W = H0, W0
            control = cn.run_text(cn_shared, y, H, W) if share else cn.run(xt, ht, t, y, B, T, H, W)      # ref :1746
            ctx = self._with_text(base, y)
            if share:
                xs = [(h0, H, W)]
                h = self._finish_block1(ctx, front, H, W)
                xs.append((h, H, W))
                rest = list(self.input_blocks)[2:]
            else:
                h = ops.conv2d_3x3_c4(xt.view(BT, H, W, self.in_dim), *self._stem)
                h = self.input_blocks[0][1].run(ctx, h, H * W)
                xs = [(h, H, W)]
                rest = list(self.input_blocks)[1:]
            for block in rest:
                h, H, W = self._run_block(ctx, block, h, H, W)
                xs.append((h, H, W))
            h, H, W = self._run_block(ctx, self.middle_block, h, H, W)
            h = ops.add(control.pop(), h)                                      # ref :1784-1785
            for block in self.output_blocks:
                skip, _, _ = xs.pop()
                h = ops.concat_add(h, skip, control.pop())                     # ref :1792
                h, H, W = self._run_block(ctx, block, h, H, W)
            gw, gb, w9, b9 = self._head
            h = ops.groupnorm(h, gw, gb, BT, 1e-5, True)
            h = ops.conv2d_3x3(h.view(BT, H, W, h.shape[1]), w9, b9)          # ref :1805
            outs.append(ops.tokens_to_nchw5(h, B, self.out_dim, T, H, W))     # ref :1808
        return outs


class VideoControlNet(_UNetBase):
    """Copy of the UNet encoder + middle block whose per-block outputs go through zero 1x1 convs
    and are added to the UNet's skips (ref :1896-2206)."""

    def __init__(self, in_dim=4, dim=320, y_dim=1024, context_dim=1024, out_dim=4, dim_mult=[1, 2, 4, 4],
                 num_heads=8, head_dim=64, num_res_blocks=2, attn_scales=[1 / 1, 1 / 2, 1 / 4],
                 use_scale_shift_norm=True, dropout=0.1, temporal_attn_times=1, temporal_attention=True,
                 use_checkpoint=True, use_image_dataset=False, use_fps_condition=False, use_sim_mask=False,
                 training=False, inpainting=True):
        super().__init__()
        self.in_dim, self.dim, self.context_dim, self.embed_dim = in_dim, dim, context_dim, dim * 4
        self.num_heads = num_heads if num_heads else dim // 32
        shortcut_dims, _, cout, _, _ = self._build_trunk(
            in_dim, dim, context_dim, dim_mult, self.num_heads, head_dim, num_res_blocks, attn_scales, dropout,
            use_checkpoint)
        self.zero_convs = nn.ModuleList([self.make_zero_conv(c) for c in shortcut_dims])
        self.middle_block_out = self.make_zero_conv(self.embed_dim)
        self.add_dim = 320
        self.input_hint_block = zero_module(nn.Conv2d(4, self.add_dim, 3, padding=1))
        self._packed = False

    def make_zero_conv(self, in_channels, out_channels=None):
        out_channels = in_channels if out_channels is None else out_channels
        return TimestepEmbedSequential(zero_module(nn.Conv2d(in_channels, out_channels, 1, padding=0)))

    def _pack_all(self):
        self._pack_trunk()
        self._zc = [(_h(z[0].weight[:, :, 0, 0]), _h(z[0].bias)) for z in self.zero_convs]
        self._mid_out = (_h(self.middle_block_out[0].weight[:, :, 0, 0]), _h(self.middle_block_out[0].bias))
        self._hint = (_w9(self.input_hint_block), _h(self.input_hint_block.bias))

    def run(self, xt, ht, t, y, B, T, H, W):
        """Returns the list of 13 control residuals as token matrices (ref :2134-2206)."""
        self._ensure_packed()
        ctx = self._begin(t, y, B, T)
        BT = B * T
        hint = ops.conv2d_3x3_c4(ht.view(BT, H, W, 4), *self._hint)                       # ref :2170-2171
        h = ops.conv2d_3x3_c4(xt.view(BT, H, W, self.in_dim), *self._stem, residual=hint)  # ref :2189-2194
        h = self.input_blocks[0][1].run(ctx, h, H * W)
        outs = [ops.linear(h, *self._zc[0])]
        return self._run_rest(ctx, h, outs, 1, H, W)

    def _run_rest(self, ctx, h, outs, first, H, W):
        for k, block in enumerate(list(self.input_blocks)[first:], start=first):
            h, H, W = self._run_block(ctx, block, h, H, W)
            outs.append(ops.linear(h, *self._zc[k]))
        h, H, W = self._run_block(ctx, self.middle_block, h, H, W)
        outs.append(ops.linear(h, *self._mid_out))
        return outs

    def run_shared(self, xt, ht, t, B, T, H, W):
        """The text-independent prefix of run() (see _UNetBase._run_prefix): evaluated once per solver step for both CFG branches."""
        self._ensure_packed()
        base = self._begin_time(t, B, T)
        BT = B * T
        hint = ops.conv2d_3x3_c4(ht.view(BT, H, W, 4), *self._hint)
        h = ops.conv2d_3x3_c4(xt.view(BT, H, W, self.in_dim), *self._stem, residual=hint)
        h0, front = self._run_prefix(base, h, H, W)
        return base, ops.linear(h0, *self._zc[0]), front

    def run_text(self, shared, y, H, W):
        base, out0, front = shared
        ctx = self._with_text(base, y)
        h = self._finish_block1(ctx, front, H, W)
        return self._run_rest(ctx, h, [out0, ops.linear(h, *self._zc[1])], 2, H, W)
