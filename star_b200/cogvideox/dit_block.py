"""One CogVideoX-5B DiT layer with STAR's LIEM gates on the star_b200 kernels.

Reference (cogvideox-based/): AdaLNMixin.layer_forward (sat/dit_video_concat.py:482-563), the qk-LayerNorm and 3-D
rotary attention_fn mixins (:570-598, :306-346), SpatialAttention / TemporalLocalAttention (transformer.py:316-348) and
sat's default SelfAttention / MLP (transformer.py:35-119, :202-312).  Same kernels as the I2VGen-XL path:
  * fused QKV / dense / MLP GEMMs on the persistent wgmma tap-GEMM, with the adaLN gate and residual
    (``hidden + gate * f(x)``) and the tanh-GELU folded into the epilogue (star_linear_ex),
  * the 3-D full attention over text + T*H*W tokens (48 heads x 64, N = 17 776) on the TMEM-resident flash
    attention kernel (attn4), fed by a fused per-head qk-LayerNorm + rotary kernel,
  * LayerNorm + adaLN modulate as ONE LayerNorm launch per (sample, text|image) segment: the modulation is folded
    into the affine parameters, gamma' = gamma (1 + scale), beta' = beta (1 + scale) + shift,
  * spatial / temporal LIEM gates on the channels-last token matrix (no (b t) c h w <-> (b h w) t c reshuffles).
Precision: ``dtype`` = torch.bfloat16 (the reference config, cogvideox_5b_infer_sr.yaml:11; runs on libstar_sm100_bf16.so,
the same kernel sources built with -DSTAR_BF16) or torch.float16; fp32 accumulation, statistics and softmax in both.
Oracles: oracle/cogvideox_sat.py executes the reference's own transformer.py / dit_video_concat.py behind a shim of the
un-vendored SwissArmyTransformer; oracle/cogvideox_ref.py is the older line-by-line restatement of one layer.
"""
import torch

from .. import ops
from ..ops import LiemPart

HALF = torch.float16


class DiTLayer:
    """Holds the packed fp16 weights of one layer; ``forward(hidden, emb)`` -> new hidden (fp16)."""

    def __init__(self, sd, hidden=3072, heads=48, text_length=226, frames=13, height=30, width=45,
                 ln_eps=1e-5, qk_ln_eps=1e-6, cos=None, sin=None, device="cuda", dtype=HALF, time_embed_dim=512):
        self.d, self.heads, self.tl = hidden, heads, text_length
        self.T, self.H, self.W = frames, height, width
        self.ln_eps, self.qk_eps = ln_eps, qk_ln_eps
        self.dt = dtype
        dev = torch.device(device)
        HALF = dtype                                                             # noqa: N806  (token dtype of this layer)

        def h(k):
            return sd[k].detach().to(dev, HALF).contiguous()

        self.w_ada, self.b_ada = h("adaLN_modulation.1.weight"), h("adaLN_modulation.1.bias")
        self.ln1 = (sd["input_layernorm.weight"].to(dev, torch.float32), sd["input_layernorm.bias"].to(dev, torch.float32))
        self.ln2 = (sd["post_attention_layernorm.weight"].to(dev, torch.float32),
                    sd["post_attention_layernorm.bias"].to(dev, torch.float32))
        self.liem_s = h("spa_local.conv1.weight").reshape(-1)
        wt = sd["temp_local.conv1.weight"].detach().to(HALF).float().reshape(-1).tolist()
        self.liem_t = (wt[0], wt[1])
        self.w_qkv, self.b_qkv = h("attention.query_key_value.weight"), h("attention.query_key_value.bias")
        self.w_o, self.b_o = h("attention.dense.weight"), h("attention.dense.bias")
        self.qg, self.qb = h("query_layernorm.weight"), h("query_layernorm.bias")
        self.kg, self.kb = h("key_layernorm.weight"), h("key_layernorm.bias")
        self.w1, self.b1 = h("mlp.dense_h_to_4h.weight"), h("mlp.dense_h_to_4h.bias")
        self.w2, self.b2 = h("mlp.dense_4h_to_h.weight"), h("mlp.dense_4h_to_h.bias")
        self.cos = cos.to(dev, torch.float32).contiguous()
        self.sin = sin.to(dev, torch.float32).contiguous()

    def _ln_modulate(self, x, out, ln, shift, scale, B, S, segs=None):
        """out <- LN(x) * (1 + scale) + shift per (sample, segment); the modulation is folded into gamma/beta.
        segs: the (text, image) row ranges of a sample's S rows, default the whole sequence's."""
        g, b = ln
        tl = self.tl
        for bi in range(B):
            for seg, (lo, hi) in enumerate(segs or ((0, tl), (tl, S))):
                if lo == hi:
                    continue
                sc, sh = scale[seg][bi].float(), shift[seg][bi].float()
                gp = (g * (1 + sc)).to(self.dt)
                bp = (b * (1 + sc) + sh).to(self.dt)
                rows = slice(bi * S + lo, bi * S + hi)
                out[rows] = ops.layernorm(x[rows], gp, bp, eps=self.ln_eps)
        return out

    @torch.no_grad()
    def forward(self, hidden, emb):
        """hidden (B, text_length + T*H*W, hidden) any float dtype; emb (B, 512).  Returns fp16 (B, S, hidden)."""
        B, S, d = hidden.shape
        tl, T, H, W = self.tl, self.T, self.H, self.W
        assert S == tl + T * H * W and d == self.d
        x = hidden.to(self.dt).reshape(B * S, d).contiguous()
        mod = ops.linear(ops.silu(emb.to(self.dt).contiguous()), self.w_ada, self.b_ada)           # (B, 12 d)
        (sh_msa, sc_msa, g_msa, sh_mlp, sc_mlp, g_mlp, tsh_msa, tsc_msa, tg_msa, tsh_mlp, tsc_mlp, tg_mlp) = mod.chunk(12, dim=1)

        # ---- attention branch
        a_in = torch.empty_like(x)
        self._ln_modulate(x, a_in, self.ln1, (tsh_msa, sh_msa), (tsc_msa, sc_msa), B, S)
        for bi in range(B):                                                                     # LIEM gates on image tokens
            rows = slice(bi * S + tl, (bi + 1) * S)
            img = a_in[rows]
            gate = ops.liem_spatial_gate(img, self.liem_s, T, H, W)
            img = ops.row_gate(img, 1, gate)
            a_in[rows] = ops.row_gate(img, 2, None, *self.liem_t)
        qkv = ops.linear(a_in, self.w_qkv, self.b_qkv)
        ops.qk_ln_rope(qkv, self.heads, d, self.qg, self.qb, self.kg, self.kb, self.cos, self.sin, S, tl, self.qk_eps)
        att = ops.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, self.heads, S, S, 1, 0.125)
        x = self._gated_linear(att, self.w_o, self.b_o, (tg_msa, g_msa), x, B, S)
        # ---- MLP branch
        m_in = torch.empty_like(x)
        self._ln_modulate(x, m_in, self.ln2, (tsh_mlp, sh_mlp), (tsc_mlp, sc_mlp), B, S)
        h4 = ops.linear_ex(m_in, self.w1, self.b1, flags=ops.FLAG_GELU_TANH)
        x = self._gated_linear(h4, self.w2, self.b2, (tg_mlp, g_mlp), x, B, S)
        return x.reshape(B, S, d)

    def _gated_linear(self, a, w, b, gates, resid, B, S, segs=None):
        """resid + gate * (a W^T + b), gate per (sample, text|image segment)"""
        out = torch.empty_like(resid)
        tl = self.tl
        for bi in range(B):
            for seg, (lo, hi) in enumerate(segs or ((0, tl), (tl, S))):
                if lo == hi:
                    continue
                rows = slice(bi * S + lo, bi * S + hi)
                ops.linear_ex(a[rows], w, b, colscale=gates[seg][bi].contiguous(), residual=resid[rows], out=out[rows])
        return out

    def _qkv_by_rank(self, P):
        """the QKV projection split by the rank whose heads each output column feeds: [(W_j, b_j)], W_j = the q, k and v rows
        of heads [j H / P, (j + 1) H / P) stacked, so one GEMM writes rank j's block of the head all-to-all's send buffer"""
        split = self.__dict__.setdefault("_qkv_split", {})
        if P not in split:
            d, c = self.d, self.heads // P * 64
            split[P] = [tuple(torch.cat([t[o + j * c:o + (j + 1) * c] for o in (0, d, 2 * d)]).contiguous()
                              for t in (self.w_qkv, self.b_qkv)) for j in range(P)]
        return split[P]

    @torch.no_grad()
    def forward_shard(self, hidden, emb, sp):
        """``forward`` on this rank's token shard sp.me of every sample (parallel.SeqShard): hidden (B, rows, hidden) ->
        (B, rows, hidden), equal byte for byte to those rows of ``forward`` over the whole sequence.  Collective over
        sp.group: the LIEM map is all-gathered and attention runs over all S tokens on heads / P heads per rank, one
        all-to-all each way per sample."""
        B, n, d = hidden.shape
        me, P = sp.me, sp.P
        tl, T, H, W = self.tl, self.T, self.H, self.W
        S, hp = tl + T * H * W, self.heads // P
        c = hp * 64
        assert n == me.rows and d == self.d
        segs = ((0, me.text_rows), (me.text_rows, n))
        x = hidden.to(self.dt).reshape(B * n, d).contiguous()
        mod = ops.linear(ops.silu(emb.to(self.dt).contiguous()), self.w_ada, self.b_ada)           # (B, 12 d)
        (sh_msa, sc_msa, g_msa, sh_mlp, sc_mlp, g_mlp, tsh_msa, tsc_msa, tg_msa, tsh_mlp, tsc_mlp, tg_mlp) = mod.chunk(12, dim=1)

        # ---- attention branch
        a_in = torch.empty_like(x)
        self._ln_modulate(x, a_in, self.ln1, (tsh_msa, sh_msa), (tsc_msa, sc_msa), B, n, segs)
        img0, ni = me.start + me.text_rows - tl, me.image_rows                                  # image tokens held
        for bi in range(B):                                                                     # LIEM gates on image tokens
            rows = slice(bi * n + me.text_rows, (bi + 1) * n)
            img = a_in[rows]
            mm = torch.empty((T * H * W, 2), dtype=self.dt, device=x.device)
            if ni:
                ops.liem_spatial_gate(img, None, T, H, W, part=LiemPart(mm, img0, ni))     # this shard's max / mean
            mm = sp.gather_image_rows(mm[img0:img0 + ni])                                        # the whole map
            if ni:
                gate = ops.liem_spatial_gate(None, self.liem_s, T, H, W, part=LiemPart(mm, img0, ni))
                img = ops.row_gate(img, 1, gate)
                a_in[rows] = ops.row_gate(img, 2, None, *self.liem_t)
        back = []
        for bi in range(B):
            send = torch.empty((P, n, 3 * c), dtype=self.dt, device=x.device)     # [dest rank][row][q | k | v of its heads]
            for j, (wj, bj) in enumerate(self._qkv_by_rank(P)):
                ops.linear(a_in[bi * n:(bi + 1) * n], wj, bj, out=send[j])
            # qk-LayerNorm + RoPE in place; row r of every block is sequence position me.start + r: with seq = n and the
            # text boundary moved to tl - me.start, qk_ln_rope's position (row % seq) - text_len is exactly that
            ops.qk_ln_rope(send.view(P * n, 3 * c), hp, c, self.qg, self.qb, self.kg, self.kb, self.cos, self.sin, n,
                           tl - me.start, self.qk_eps)
            recv = sp.all_to_all(send.view(P * n, 3 * c), "qkv")                                   # [S][q | k | v of my heads]
            att = ops.attention(recv[:, :c], recv[:, c:2 * c], recv[:, 2 * c:], 1, hp, S, S, 1, 0.125)
            back.append(sp.all_to_all(att, "out").view(P, n, c))                                  # [source rank][my rows][its heads]
        out = torch.empty_like(x)
        gates = (tg_msa, g_msa)
        for bi in range(B):                              # the dense projection reads the head-blocked output in place
            for seg, (lo, hi) in enumerate(segs):
                if lo == hi:
                    continue
                rows = slice(bi * n + lo, bi * n + hi)
                ops.linear_ex(back[bi][:, lo:hi], self.w_o, self.b_o, colscale=gates[seg][bi].contiguous(), residual=x[rows],
                              out=out[rows])
        x = out
        # ---- MLP branch
        m_in = torch.empty_like(x)
        self._ln_modulate(x, m_in, self.ln2, (tsh_mlp, sh_mlp), (tsc_mlp, sc_mlp), B, n, segs)
        h4 = ops.linear_ex(m_in, self.w1, self.b1, flags=ops.FLAG_GELU_TANH)
        x = self._gated_linear(h4, self.w2, self.b2, (tg_mlp, g_mlp), x, B, n, segs)
        return x.reshape(B, n, d)
