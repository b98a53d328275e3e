"""TEST INFRASTRUCTURE -- per-kernel references for every op in star_b200/ops.py.

Same signatures as ``star_b200.ops`` but computed with plain torch in fp32 on
whatever device the inputs live on (CPU in the host-logic tests, CUDA in the
GPU parity tests), rounding to fp16 only where the CUDA kernel does.  Used
 (a) by tests/test_kernels_gpu.py as the expected value of each C-ABI call,
 (b) by tests/test_unet_wiring_cpu.py, which monkeypatches these over
     ``star_b200.ops`` to validate the host graph (weight repacking, op order,
     layouts) against the golden vectors without a GPU.
Never imported by the product.
"""
import torch
import torch.nn.functional as F

HALF = torch.float16          # token dtype the references round to; tests of the bf16 library call set_dtype(torch.bfloat16)
FLAG_GEGLU = 1


def set_dtype(dtype):
    global HALF
    HALF = dtype

FLAG_SILU_OUT = 2
FLAG_GELU_ERF = 4


def _f(t):
    return None if t is None else t.float()


def linear(a, w, bias=None, residual=None, rowvec=None, rowvec_div=1, flags=0, out=None):
    acc = _f(a) @ _f(w).t()
    if bias is not None:
        acc = acc + _f(bias)
    if flags & FLAG_GEGLU:
        val, gate = acc.chunk(2, dim=-1)
        acc = val * F.gelu(gate)
    if flags & FLAG_GELU_ERF:
        acc = F.gelu(acc)
    if rowvec is not None:
        idx = torch.arange(a.shape[0], device=a.device) // rowvec_div
        acc = acc + _f(rowvec)[idx]
    if residual is not None:
        acc = acc + _f(residual)
    if flags & FLAG_SILU_OUT:
        acc = F.silu(acc)
    res = acc.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def attention_causal(q, k, v, batch, heads, N, scale=0.125, out=None):
    def split(t):
        return _f(t)[:, :heads * 64].reshape(batch, N, heads, 64).permute(0, 2, 1, 3)
    s = (split(q) @ split(k).transpose(-1, -2)) * scale
    s = s + torch.full((N, N), float("-inf"), device=q.device).triu(1)
    o = torch.softmax(s, dim=-1) @ split(v)
    res = o.permute(0, 2, 1, 3).reshape(batch * N, heads * 64).to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def conv2d_3x3(x, w9, bias=None, rowvec=None, rowvec_div=1, residual=None, out=None):
    BT, H, W, Cin = x.shape
    y = F.conv2d(_f(x).permute(0, 3, 1, 2), _f(w9).permute(0, 3, 1, 2), _f(bias), padding=1)
    y = y.permute(0, 2, 3, 1).reshape(BT * H * W, -1)
    if rowvec is not None:
        idx = torch.arange(y.shape[0], device=x.device) // rowvec_div
        y = y + _f(rowvec)[idx]
    if residual is not None:
        y = y + _f(residual)
    res = y.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def conv2d_3x3_s2(x, w9, bias=None):
    BT, H, W, Cin = x.shape
    y = F.conv2d(_f(x).permute(0, 3, 1, 2), _f(w9).permute(0, 3, 1, 2), _f(bias), stride=2, padding=(2, 1))
    Ho, Wo = y.shape[2], y.shape[3]
    return y.permute(0, 2, 3, 1).reshape(BT * Ho * Wo, -1).to(HALF), Ho, Wo


def conv_t3(x, w3, bias=None, residual=None, B=1, T=1, HW=1, out=None):
    Cin = x.shape[1]
    x5 = _f(x).reshape(B, T, HW, Cin).permute(0, 3, 1, 2)            # b c t hw
    w = _f(w3).permute(0, 2, 1)[..., None]                          # cout cin 3 1
    y = F.conv2d(x5, w, _f(bias), padding=(1, 0))
    y = y.permute(0, 2, 3, 1).reshape(B * T * HW, -1)
    if residual is not None:
        y = y + _f(residual)
    res = y.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def conv2d_3x3_c4(x, w9, bias=None, residual=None):
    BT, H, W, C = x.shape
    y = F.conv2d(_f(x).permute(0, 3, 1, 2), _f(w9).permute(0, 3, 1, 2), _f(bias), padding=1)
    y = y.permute(0, 2, 3, 1).reshape(BT * H * W, -1)
    if residual is not None:
        y = y.to(HALF).float() + _f(residual)
    return y.to(HALF)


def attention(q, k, v, batch, heads, Nq, Nk, kv_batch_div=1, scale=0.125, out=None):
    d = 64
    qf = _f(q)[:, :heads * d].reshape(batch, Nq, heads, d).permute(0, 2, 1, 3)
    kvb = (batch + kv_batch_div - 1) // kv_batch_div
    kf = _f(k)[:, :heads * d].reshape(kvb, Nk, heads, d).permute(0, 2, 1, 3)
    vf = _f(v)[:, :heads * d].reshape(kvb, Nk, heads, d).permute(0, 2, 1, 3)
    idx = torch.arange(batch, device=q.device) // kv_batch_div
    o = F.scaled_dot_product_attention(qf, kf[idx], vf[idx], scale=scale)
    res = o.permute(0, 2, 1, 3).reshape(batch * Nq, heads * d).to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def attention_exact(q, k, v, batch, heads, Nq, Nk, scale=0.125, budget_bytes=6 << 30):
    """softmax(q k^T * scale) v in true fp32 with plain matmuls over query-row chunks (no fused kernel: a fused fp32
    SDPA may run TF32 tensor ops).  k / v hold ONE kv batch shared by every q batch (kv_batch_div = batch) or `batch`."""
    d = 64
    qf = _f(q)[:, :heads * d].reshape(batch, Nq, heads, d).permute(0, 2, 1, 3)             # b h nq d
    kvb = k.shape[0] // Nk
    kf = _f(k)[:, :heads * d].reshape(kvb, Nk, heads, d).permute(0, 2, 3, 1)               # b h d nk
    vf = _f(v)[:, :heads * d].reshape(kvb, Nk, heads, d).permute(0, 2, 1, 3)
    if kvb != batch:
        kf, vf = kf.expand(batch, -1, -1, -1), vf.expand(batch, -1, -1, -1)
    out = torch.empty(batch, heads, Nq, d, device=q.device, dtype=torch.float32)
    rows = max(1, min(Nq, budget_bytes // (4 * batch * heads * Nk)))
    for r in range(0, Nq, rows):
        s = torch.matmul(qf[:, :, r:r + rows], kf) * scale
        out[:, :, r:r + rows] = torch.matmul(torch.softmax(s, dim=-1), vf)
    return out.permute(0, 2, 1, 3).reshape(batch * Nq, heads * d).to(HALF)


def temporal_attention(qkv, B, T, HW, heads, Ci, scale=0.125):
    d = 64
    x = _f(qkv).reshape(B, T, HW, -1)

    def split(t):
        return t.reshape(B, T, HW, heads, d).permute(0, 2, 3, 1, 4)     # b hw h t d

    q, k, v = split(x[..., :Ci]), split(x[..., Ci:2 * Ci]), split(x[..., 2 * Ci:3 * Ci])
    o = F.scaled_dot_product_attention(q, k, v, scale=scale)
    return o.permute(0, 3, 1, 2, 4).reshape(B * T * HW, Ci).to(HALF)


def groupnorm(x, gamma, beta, nsamples, eps, silu, out=None):
    rows, C = x.shape
    xs = _f(x).reshape(nsamples, rows // nsamples, C).permute(0, 2, 1)          # n c r
    y = F.group_norm(xs, 32, _f(gamma), _f(beta), eps)
    if silu:
        y = F.silu(y)
    res = y.permute(0, 2, 1).reshape(rows, C).to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def layernorm(x, gamma, beta, gate_mode=0, gate=None, w0=0.0, w1=0.0, eps=1e-5):
    xf = _f(x)
    if gate_mode == 1:
        xf = (xf * _f(gate)[:, None]).to(HALF).float()
    elif gate_mode == 2:
        mx = xf.max(dim=-1, keepdim=True)[0]
        mean = xf.mean(dim=-1, keepdim=True).to(HALF).float()
        lin = (w0 * mx + w1 * mean).to(HALF).float()
        g = torch.sigmoid(lin).to(HALF).float()
        xf = (xf * g).to(HALF).float()
    return F.layer_norm(xf, (x.shape[1],), _f(gamma), _f(beta), eps).to(HALF)


def liem_spatial_gate(x, w98, BT, H, W):
    xf = _f(x).reshape(BT, H, W, -1)
    mx = xf.max(dim=-1)[0]
    mean = xf.mean(dim=-1)
    mm = torch.stack([mx, mean], dim=1).to(HALF).float()                       # bt 2 h w
    conv = F.conv2d(mm, _f(w98).reshape(1, 2, 7, 7), padding=3).to(HALF).float()
    return torch.sigmoid(conv).reshape(-1).to(HALF)


def concat_add(a, b, c=None):
    bb = b if c is None else (_f(b) + _f(c)).to(HALF)
    return torch.cat([a, bb], dim=1)


def add(a, b):
    return (_f(a) + _f(b)).to(HALF)


def upsample2x_crop(x, BT, H, W):
    C = x.shape[1]
    x4 = x.reshape(BT, H, W, C)
    up = x4.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)[:, 1:-1]
    return up.reshape(-1, C).contiguous()


def nchw5_to_tokens(x, dtype=None):
    B, C, Fr, H, W = x.shape
    return x.float().permute(0, 2, 3, 4, 1).reshape(B * Fr * H * W, C).to(HALF)


def tokens_to_nchw5(x, B, C, Fr, H, W):
    return x[:, :C].reshape(B, Fr, H, W, C).permute(0, 4, 1, 2, 3).contiguous()


def sinusoidal(t, dim, dtype=None):
    half = dim // 2
    tf = t.float()
    freqs = torch.pow(10000, -torch.arange(half, device=t.device).float().div(half))
    s = torch.outer(tf, freqs)
    return torch.cat([torch.cos(s), torch.sin(s)], dim=1).to(HALF)


def silu(x):
    return F.silu(_f(x)).to(HALF)


FLAG_GELU_TANH = 8


def linear_ex(a, w, bias=None, colscale=None, residual=None, flags=0, out=None):
    acc = _f(a) @ _f(w).t()
    if bias is not None:
        acc = acc + _f(bias)
    if flags & FLAG_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    if colscale is not None:
        acc = acc * _f(colscale)
    if residual is not None:
        acc = acc + _f(residual)
    res = acc.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def row_gate(x, mode, gate=None, w0=0.0, w1=0.0, out=None):
    xf = _f(x)
    if mode == 1:
        g = _f(gate)[:, None]
    else:
        mx = xf.max(dim=-1, keepdim=True)[0]
        mean = xf.mean(dim=-1, keepdim=True).to(HALF).float()
        g = torch.sigmoid((w0 * mx + w1 * mean).to(HALF).float()).to(HALF).float()
    res = (xf * g).to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def qk_ln_rope(qkv, heads, koff, qg, qb, kg, kb, cos, sin, seq, text_len, eps=1e-6):
    rows = qkv.shape[0]
    tok = torch.arange(rows, device=qkv.device) % seq
    img = tok >= text_len
    idx = (tok - text_len).clamp(min=0)
    c, s = cos.to(qkv.device)[idx][:, None, :], sin.to(qkv.device)[idx][:, None, :]
    for off, g, b in ((0, qg, qb), (koff, kg, kb)):
        x = _f(qkv[:, off:off + heads * 64]).reshape(rows, heads, 64)
        x = F.layer_norm(x, (64,), _f(g), _f(b), eps).to(HALF).float()
        xr = x.reshape(rows, heads, 32, 2)
        rot = torch.stack((-xr[..., 1], xr[..., 0]), dim=-1).reshape(rows, heads, 64)
        y = torch.where(img[:, None, None], x * c + rot * s, x)
        qkv[:, off:off + heads * 64] = y.reshape(rows, heads * 64).to(HALF)
    return qkv


def conv2d_3x3_s2p(x, w9, bias=None, pad=(0, 1, 0, 1)):
    BT, H, W, Cin = x.shape
    pt, pb, pl, pr = pad
    xp = F.pad(_f(x).permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xp, _f(w9).permute(0, 3, 1, 2), _f(bias), stride=2)
    Ho, Wo = y.shape[2], y.shape[3]
    return y.permute(0, 2, 3, 1).reshape(BT * Ho * Wo, -1).to(HALF), Ho, Wo


def upsample2x(x, BT, H, W, out=None):
    C = x.shape[1]
    up = x.reshape(BT, H, W, C).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    up = up.reshape(-1, C).contiguous()
    if out is not None:
        out.copy_(up)
        return out
    return up


def softmax_rows(s, cols):
    p = torch.softmax(_f(s[:, :cols]), dim=-1).to(HALF)
    s.zero_()
    s[:, :cols] = p
    return s


def vae_head(x, w27, bias3, B, T, H, W):
    x5 = _f(x[:, :3]).reshape(B, T, H, W, 3).permute(0, 4, 1, 2, 3)                 # b c t h w
    y = F.conv3d(x5, _f(w27).reshape(3, 3, 3, 1, 1), _f(bias3), padding=(1, 0, 0))
    return y.permute(0, 2, 1, 3, 4).reshape(B * T, 3, H, W).to(HALF)


def bilinear_pad(x, H, W, padding=(0, 0, 0, 0), value=1.0):
    return F.pad(F.interpolate(x.reshape(-1, 1, *x.shape[-2:]).float(), [H, W], mode="bilinear"), padding, "constant", value
                 ).reshape(*x.shape[:-2], H + padding[2] + padding[3], W + padding[0] + padding[1])


def cfg_x0(y_out, u_out, xt, alphas, sigmas, guide_scale, guide_rescale=None, return_guided=False):
    """the reference's fp16 tensor arithmetic, op by op (diffusion_sdedit.py:89-99)"""
    out = u_out + guide_scale * (y_out - u_out)
    if guide_rescale is not None:
        ratio = (y_out.flatten(1).std(dim=1) / (out.flatten(1).std(dim=1) + 1e-12)).view((-1,) + (1,) * (y_out.ndim - 1))
        out = out * (guide_rescale * ratio + (1 - guide_rescale) * 1.0)
    x0 = alphas * xt - sigmas * out
    return (x0, out) if return_guided else x0


def adain_color_fix(video, source, uint8=False):
    """inference_utils.tensor2vid followed by color_fix.adain_color_fix, op by op (inference_sr.py:77-80)"""
    v = (video.clone() * 0.5 + 0.5).clamp(0, 1) * 255.0                          # tensor2vid
    target = v[0].permute(1, 2, 3, 0)                                             # b c f h w -> f h w c
    target = target.permute(0, 3, 1, 2) / 255                                     # T H W C -> T C H W
    src = (source.to(video.device) + 1) / 2
    outs = []
    for i in range(target.shape[0]):
        c, s = target[i:i + 1], src[i:i + 1]
        cm, cs = c.reshape(1, c.shape[1], -1).mean(2).reshape(1, -1, 1, 1), (c.reshape(1, c.shape[1], -1).var(2) + 1e-5).sqrt().reshape(1, -1, 1, 1)
        sm, ss = s.reshape(1, s.shape[1], -1).mean(2).reshape(1, -1, 1, 1), (s.reshape(1, s.shape[1], -1).var(2) + 1e-5).sqrt().reshape(1, -1, 1, 1)
        outs.append((c - cm) / cs * ss + sm)
    res = torch.cat(outs).clamp_(0.0, 1.0).permute(0, 2, 3, 1) * 255
    return res.round().to(torch.uint8) if uint8 else res


def conv3d_causal(xp, w27, T, H, W, bias=None, residual=None, out=None):
    """xp [(T+2)*H*W, Cin] (two context frames + clip); w27 [Cout, 3(t), 3(h), 3(w), Cin]"""
    Cin = xp.shape[1]
    x5 = _f(xp).reshape(1, T + 2, H, W, Cin).permute(0, 4, 1, 2, 3)
    y = F.conv3d(x5, _f(w27).permute(0, 4, 1, 2, 3), _f(bias), padding=(0, 1, 1))
    y = y.permute(0, 2, 3, 4, 1).reshape(T * H * W, -1)
    if residual is not None:
        y = y + _f(residual)
    res = y.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def spatial_norm_src_index(T, H, W, Tl, Hl, Wl, device):
    """row (t, h, w) -> latent row, the nearest-neighbour rule of SpatialNorm3D.forward (cp_enc_dec.py:492-500): each index
    is F.interpolate(mode="nearest")'s min(floor(dst * s), n_in - 1) with the fp32 scale s = n_in / n_out"""
    def nearest(n_out, n_in):
        s = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
        i = (torch.arange(n_out, device=device, dtype=torch.float32) * s.to(device)).floor().long()
        return i.clamp(max=n_in - 1)
    if T > 1 and T % 2 == 1:
        ts = torch.cat([torch.zeros(1, dtype=torch.long, device=device), 1 + nearest(T - 1, Tl - 1)])
    else:
        ts = nearest(T, Tl)
    hs, ws = nearest(H, Hl), nearest(W, Wl)
    return ((ts[:, None, None] * Hl + hs[None, :, None]) * Wl + ws[None, None, :]).reshape(-1)


def groupnorm_mod(x, gamma, beta, ymod, bmod, T, H, W, Tl, Hl, Wl, eps, silu, out=None):
    rows, C = x.shape
    y = F.group_norm(_f(x).t().reshape(1, C, rows), 32, _f(gamma), _f(beta), eps).reshape(C, rows).t()
    src = spatial_norm_src_index(T, H, W, Tl, Hl, Wl, x.device)
    y = y * _f(ymod)[src] + _f(bmod)[src]
    if silu:
        y = F.silu(y)
    res = y.to(HALF)
    if out is not None:
        out.copy_(res)
        return out
    return res


def time_avgpool2(x, T, HW):
    C = x.shape[1]
    f = _f(x).reshape(T, HW, C)
    if T % 2:
        out = torch.cat([f[:1], 0.5 * (f[1::2] + f[2::2])], 0)
    else:
        out = 0.5 * (f[0::2] + f[1::2])
    return out.reshape(-1, C).to(HALF)
