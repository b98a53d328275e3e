"""Tensor-level wrappers over the C ABI (include/star_sm100.h).

PyTorch is used for device memory (torch.empty) and the current CUDA stream
only; every op below is one call into libstar_sm100.so.  All activations are
fp16 CUDA tensors in the channels-last token layout X[rows, C] with rows
ordered (b, t, h, w).
"""
from typing import NamedTuple

import torch

from . import lib as _L

HALF = torch.float16

FLAG_GEGLU = 1
FLAG_SILU_OUT = 2
FLAG_GELU_ERF = 4
GN_STATS = 1        # star_groupnorm phases
GN_APPLY = 2


# ---- optional per-op tracing (CUDA events on the launching stream) ---------------------------------
_trace = None


def trace_begin():
    """Start recording (name, signature, start_event, end_event) for every op call."""
    global _trace
    _trace = []


def trace_end():
    """Stop recording; returns [(name, signature, milliseconds)] (synchronises the device)."""
    global _trace
    rec, _trace = _trace, None
    torch.cuda.synchronize()
    return [(n, sig, a.elapsed_time(b)) for (n, sig, a, b) in (rec or [])]


def _traced(fn):
    """Every op runs with its first tensor's device current (kernels are launched on the CURRENT device and stream:
    a model on cuda:1 must not launch on cuda:0 with foreign pointers), and is optionally timed."""
    import functools

    def guarded(*args, **kw):
        t = next((a for a in args if torch.is_tensor(a)), None)
        if t is not None and t.is_cuda and t.device.index != torch.cuda.current_device():
            with torch.cuda.device(t.device):
                return fn(*args, **kw)
        return fn(*args, **kw)

    @functools.wraps(fn)
    def wrapper(*args, **kw):
        if _trace is None:
            return guarded(*args, **kw)
        sig = tuple(tuple(a.shape) if torch.is_tensor(a) else a for a in args
                    if torch.is_tensor(a) or isinstance(a, (int, float)))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = guarded(*args, **kw)
        b.record()
        _trace.append((fn.__name__, sig, a, b))
        return out
    return wrapper


def launch_count():
    """Kernels launched by the star_b200 libraries since load."""
    return _L.launch_count()


def _bind(t, dtype=None):
    """(library, token dtype) of an op whose first tensor is t: fp16 tokens run on libstar_sm100.so, bf16 tokens on
    libstar_sm100_bf16.so (same sources).  The dtype is t's (fp16 for other dtypes) or the explicit ``dtype=``; every
    allocation and dtype check of the op follows it.  The library is initialised on t's device."""
    if not t.is_cuda:
        raise _L.StarError("star_b200 ops need CUDA tensors (no CPU fallback)")
    if dtype is None:
        dtype = t.dtype if t.dtype in (torch.float16, torch.bfloat16) else torch.float16
    if dtype not in (torch.float16, torch.bfloat16):
        raise _L.StarError(f"star_b200 ops run on fp16 or bf16 tokens, not {dtype}")
    _L.ensure_init(t.device.index if t.device.index is not None else torch.cuda.current_device(), dtype)
    return _L.get_lib(dtype), dtype


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _h(t, name, dtype):
    if t is not None and t.dtype != dtype:
        raise _L.StarError(f"{name} must be {dtype} like the op's first tensor, got {t.dtype}")
    return t


def _rowmajor(t, name):
    """2-D view whose last dim is contiguous; returns leading dim."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise _L.StarError(f"{name} must be a 2-D tensor with contiguous columns")
    return t.stride(0)


@_traced
def linear(a, w, bias=None, residual=None, rowvec=None, rowvec_div=1, flags=0, out=None):
    """out[r, n] = epi(sum_k a[r, k] w[n, k]); a may be a strided 2-D view."""
    L, dt = _bind(a)
    _h(a, "a", dt); _h(w, "w", dt); _h(bias, "bias", dt); _h(residual, "residual", dt); _h(rowvec, "rowvec", dt)
    lda = _rowmajor(a, "a")
    rows, K = a.shape
    n_w = w.shape[0]
    N = n_w // 2 if (flags & FLAG_GEGLU) else n_w
    assert w.is_contiguous() and w.shape[1] == K
    if out is None:
        out = torch.empty((rows, N), dtype=dt, device=a.device)
    ldo = _rowmajor(out, "out")
    ldres = _rowmajor(residual, "residual") if residual is not None else 0
    if rowvec is not None:
        assert rowvec.is_contiguous() and rowvec.shape[-1] == N
    _L.check(L, L.star_linear(_p(a), lda, _p(w), _p(bias), _p(rowvec), int(rowvec_div), _p(residual), ldres,
                              _p(out), ldo, rows, K, N, flags, _st()), "star_linear")
    return out


@_traced
def conv2d_3x3(x, w9, bias=None, rowvec=None, rowvec_div=1, residual=None, out=None, rows=None):
    """x [BT, H, W, Cin] contiguous; w9 [Cout, 3, 3, Cin]; returns [BT*H*W, Cout].  With rows=(row0, n) only output rows
    row0..row0+n of each frame are computed ([BT*n*W, Cout]), their halo read from x."""
    L, dt = _bind(x)
    BT, H, W, Cin = x.shape
    row0, Ho = (0, H) if rows is None else rows
    Cout = w9.shape[0]
    assert x.is_contiguous() and w9.is_contiguous() and w9.shape[1:] == (3, 3, Cin)
    if out is None:
        out = torch.empty((BT * Ho * W, Cout), dtype=dt, device=x.device)
    ldo = _rowmajor(out, "out")
    ldres = _rowmajor(residual, "residual") if residual is not None else 0
    ldrv = _rowmajor(rowvec, "rowvec") if rowvec is not None else 0           # a column slice of a wider matrix is fine
    _L.check(L, L.star_conv2d_3x3(_p(x), _p(w9), _p(bias), _p(rowvec), int(rowvec_div), ldrv, _p(residual), ldres,
                                  _p(out), ldo, BT, H, W, Cin, Cout, int(row0), int(Ho), _st()), "star_conv2d_3x3")
    return out


@_traced
def conv2d_3x3_s2(x, w9, bias=None):
    """Downsample conv: stride 2, padding (2, 1).  x [BT,H,W,Cin] -> ([BT*Ho*Wo, Cout], Ho, Wo)."""
    L, dt = _bind(x)
    BT, H, W, Cin = x.shape
    Cout = w9.shape[0]
    assert x.is_contiguous() and w9.is_contiguous()
    Ho, Wo = (H + 1) // 2 + 1, (W - 1) // 2 + 1
    ws = torch.empty(L.star_conv2d_s2_workspace_bytes(BT, H, W, Cin), dtype=torch.uint8, device=x.device)
    out = torch.empty((BT * Ho * Wo, Cout), dtype=dt, device=x.device)
    _L.check(L, L.star_conv2d_3x3_s2(_p(x), _p(w9), _p(bias), _p(out), Cout, _p(ws), BT, H, W, Cin, Cout, _st()),
             "star_conv2d_3x3_s2")
    return out, Ho, Wo


@_traced
def conv2d_3x3_s2p(x, w9, bias=None, pad=(0, 1, 0, 1)):
    """Stride-2 3x3 conv with explicit zero padding pad = (top, bottom, left, right).  Returns (out, Ho, Wo)."""
    L, dt = _bind(x)
    BT, H, W, Cin = x.shape
    Cout = w9.shape[0]
    assert x.is_contiguous() and w9.is_contiguous()
    pt, pb, pl, pr = (int(v) for v in pad)
    Ho, Wo = (H + pt + pb - 3) // 2 + 1, (W + pl + pr - 3) // 2 + 1
    ws = torch.empty(L.star_conv2d_s2p_workspace_bytes(BT, H, W, Cin, pt, pb, pl, pr), dtype=torch.uint8, device=x.device)
    out = torch.empty((BT * Ho * Wo, Cout), dtype=dt, device=x.device)
    _L.check(L, L.star_conv2d_3x3_s2p(_p(x), _p(w9), _p(bias), _p(out), Cout, _p(ws), BT, H, W, Cin, Cout, pt, pb, pl, pr,
                                      _st()), "star_conv2d_3x3_s2p")
    return out, Ho, Wo


@_traced
def conv_t3(x, w3, bias=None, residual=None, B=1, T=1, HW=1, out=None, band=None):
    """Temporal conv (3,1,1): x [B*T*HW, Cin]; w3 [Cout, 3, Cin].  With band=(p0, p1), x holds pixels p0..p1 of every frame
    ([B*T*(p1-p0), Cin]) and only those rows of out / residual ([B*T*HW, .], out required) are read / written."""
    L, dt = _bind(x)
    rows, Cin = x.shape
    p0, p1 = (0, HW) if band is None else band
    assert rows == B * T * (p1 - p0) and x.is_contiguous() and w3.is_contiguous()
    Cout = w3.shape[0]
    if out is None:
        assert band is None, "conv_t3: a band is written into a given out"
        out = torch.empty((rows, Cout), dtype=dt, device=x.device)
    assert out.shape[0] == B * T * HW and (residual is None or residual.shape[0] == B * T * HW)
    ldres = _rowmajor(residual, "residual") if residual is not None else 0
    _L.check(L, L.star_conv_t3(_p(x), _p(w3), _p(bias), _p(residual), ldres, _p(out), _rowmajor(out, "out"),
                               B, T, HW, p0, p1 - p0, Cin, Cout, _st()), "star_conv_t3")
    return out


@_traced
def conv3d_causal(xp, w27, T, H, W, bias=None, residual=None, out=None):
    """Causal Conv3d 3x3x3 (CogVideoX VAE).  xp [(T+2)*H*W, Cin]: two context frames + the clip; w27 [Cout, 3, 3, 3, Cin];
    returns [T*H*W, Cout]."""
    L, dt = _bind(xp)
    rows, Cin = xp.shape
    assert rows == (T + 2) * H * W and xp.is_contiguous() and w27.is_contiguous() and tuple(w27.shape[1:]) == (3, 3, 3, Cin)
    _h(w27, "w27", dt); _h(bias, "bias", dt); _h(residual, "residual", dt)
    Cout = w27.shape[0]
    if out is None:
        out = torch.empty((T * H * W, Cout), dtype=dt, device=xp.device)
    ldres = _rowmajor(residual, "residual") if residual is not None else 0
    _L.check(L, L.star_conv3d_causal(_p(xp), _p(w27), _p(bias), _p(residual), ldres, _p(out), _rowmajor(out, "out"),
                                     T, H, W, Cin, Cout, _st()), "star_conv3d_causal")
    return out


@_traced
def groupnorm_mod(x, gamma, beta, ymod, bmod, T, H, W, Tl, Hl, Wl, eps, silu, out=None):
    """SpatialNorm3D: GroupNorm32 over one clip x [T*H*W, C], times ymod[src] plus bmod[src] (latent-resolution
    [Tl*Hl*Wl, C] tables, nearest-neighbour gather with the reference's first-frame split), optional SiLU."""
    L, dt = _bind(x)
    rows, C = x.shape
    assert rows == T * H * W and x.is_contiguous()
    assert tuple(ymod.shape) == (Tl * Hl * Wl, C) and tuple(bmod.shape) == (Tl * Hl * Wl, C)
    ldmod = _rowmajor(ymod, "ymod")                      # column slices of one [rows, 2C] GEMM result are fine
    assert _rowmajor(bmod, "bmod") == ldmod
    _h(gamma, "gamma", dt); _h(beta, "beta", dt); _h(ymod, "ymod", dt); _h(bmod, "bmod", dt)
    ws = torch.empty(L.star_groupnorm_workspace_bytes(1, C), dtype=torch.uint8, device=x.device)
    if out is None:
        out = torch.empty_like(x)
    assert out.is_contiguous() and out.shape == x.shape and out.dtype == x.dtype
    _L.check(L, L.star_groupnorm_mod(_p(x), _p(gamma), _p(beta), _p(ymod), _p(bmod), ldmod, _p(out), T, H, W, Tl, Hl, Wl, C,
                                     float(eps), int(bool(silu)), _p(ws), _st()), "star_groupnorm_mod")
    return out


@_traced
def conv2d_3x3_c4(x, w9, bias=None, residual=None):
    """Stem conv, x [BT, H, W, 4]; w9 [Cout, 3, 3, 4]."""
    L, dt = _bind(x)
    BT, H, W, C = x.shape
    assert C == 4 and x.is_contiguous() and w9.is_contiguous()
    Cout = w9.shape[0]
    out = torch.empty((BT * H * W, Cout), dtype=dt, device=x.device)
    ws = torch.empty(L.star_conv2d_c4_workspace_bytes(BT, H, W, Cout), dtype=torch.uint8, device=x.device)
    _L.check(L, L.star_conv2d_3x3_c4(_p(x), _p(w9), _p(bias), _p(residual), _p(out), _p(ws), BT, H, W, Cout, _st()),
             "star_conv2d_3x3_c4")
    return out


@_traced
def attention(q, k, v, batch, heads, Nq, Nk, kv_batch_div=1, scale=0.125, out=None):
    """q [batch*Nq, >=heads*64] / k, v [kv_batches*Nk, ...] strided 2-D views (head h at columns h*64..)."""
    L, dt = _bind(q)
    ldq, ldk, ldv = _rowmajor(q, "q"), _rowmajor(k, "k"), _rowmajor(v, "v")
    if out is None:
        out = torch.empty((batch * Nq, heads * 64), dtype=dt, device=q.device)
    _L.check(L, L.star_attention(_p(q), ldq, _p(k), ldk, _p(v), ldv, _p(out), _rowmajor(out, "out"), batch, heads,
                                 Nq, Nk, kv_batch_div, float(scale), _st()), "star_attention")
    return out


@_traced
def attention_causal(q, k, v, batch, heads, N, scale=0.125, out=None):
    """causal self-attention (query i sees keys 0..i): q, k, v [batch*N, >=heads*64] strided 2-D views"""
    L, dt = _bind(q)
    ldq, ldk, ldv = _rowmajor(q, "q"), _rowmajor(k, "k"), _rowmajor(v, "v")
    if out is None:
        out = torch.empty((batch * N, heads * 64), dtype=dt, device=q.device)
    _L.check(L, L.star_attention_causal(_p(q), ldq, _p(k), ldk, _p(v), ldv, _p(out), _rowmajor(out, "out"), batch, heads, N,
                                        float(scale), _st()), "star_attention_causal")
    return out


@_traced
def temporal_attention(qkv, B, T, HW, heads, Ci, scale=0.125):
    L, dt = _bind(qkv)
    ld = _rowmajor(qkv, "qkv")
    out = torch.empty((qkv.shape[0], Ci), dtype=dt, device=qkv.device)
    _L.check(L, L.star_temporal_attention(_p(qkv), ld, _p(out), Ci, B, T, HW, heads, Ci, float(scale), _st()),
             "star_temporal_attention")
    return out


@_traced
def groupnorm(x, gamma, beta, nsamples, eps, silu, out=None, bands=None):
    """x [rows, C]; nsamples equal blocks of rows share statistics.  out may alias x (in place).

    With bands=(frame_rows, band) the statistics are taken once and an iterator is returned that yields ((p0, p1), y) for
    consecutive pixel bands of every frame_rows-row frame, y = the normalised rows p0..p1 of every frame, compactly."""
    L, dt = _bind(x)
    rows, C = x.shape
    assert x.is_contiguous() and rows % nsamples == 0
    ws = torch.empty(L.star_groupnorm_workspace_bytes(nsamples, C), dtype=torch.uint8, device=x.device)
    per = rows // nsamples
    if bands is not None:
        _L.check(L, L.star_groupnorm(_p(x), _p(gamma), _p(beta), None, nsamples, per, C, float(eps), 0, per, 0, per, GN_STATS,
                                     _p(ws), _st()), "star_groupnorm")
        return _groupnorm_bands(L, dt, x, ws, nsamples, silu, *bands)
    if out is None:
        out = torch.empty_like(x)
    assert out.is_contiguous() and out.shape == x.shape
    _L.check(L, L.star_groupnorm(_p(x), _p(gamma), _p(beta), _p(out), nsamples, per, C, float(eps), int(bool(silu)), per, 0, per,
                                 GN_STATS | GN_APPLY, _p(ws), _st()), "star_groupnorm")
    return out


def _groupnorm_bands(L, dt, x, ws, nsamples, silu, frame_rows, band):
    rows, C = x.shape
    for p0 in range(0, frame_rows, band):
        p1 = min(frame_rows, p0 + band)
        out = torch.empty((rows // frame_rows * (p1 - p0), C), dtype=dt, device=x.device)
        _L.check(L, L.star_groupnorm(_p(x), None, None, _p(out), nsamples, rows // nsamples, C, 0.0, int(bool(silu)), frame_rows,
                                     p0, p1 - p0, GN_APPLY, _p(ws), _st()), "star_groupnorm")
        yield (p0, p1), out
        del out


@_traced
def layernorm(x, gamma, beta, gate_mode=0, gate=None, w0=0.0, w1=0.0, eps=1e-5):
    L, _ = _bind(x)
    rows, C = x.shape
    assert x.is_contiguous()
    out = torch.empty_like(x)
    _L.check(L, L.star_layernorm(_p(x), _p(gamma), _p(beta), _p(out), rows, C, float(eps), gate_mode, _p(gate),
                                 float(w0), float(w1), _st()), "star_layernorm")
    return out


class LiemPart(NamedTuple):
    """Tokens [r0, r0 + n) of a clip whose channel max / mean map ``liem_spatial_gate(part=)`` reads and writes in mm
    [BT*H*W, 2]: a token-sharded DiT rank's image tokens."""
    mm: torch.Tensor
    r0: int
    n: int


@_traced
def liem_spatial_gate(x, w98, BT, H, W, part=None):
    """gate [BT*H*W] of the clip x [BT*H*W, C].  With part (a LiemPart), the two steps run on the part's tokens only:
    x (or None) holds their rows [n, C], whose max / mean are written to part.mm; w98 (or None: returns part.mm) gates them
    from the whole map part.mm, returning their n gates."""
    if part is not None:
        return _liem_part(x, w98, BT, H, W, part)
    L, dt = _bind(x)
    rows, C = x.shape
    assert rows == BT * H * W and x.is_contiguous()
    mm = torch.empty((rows, 2), dtype=dt, device=x.device)
    gate = torch.empty((rows,), dtype=dt, device=x.device)
    _L.check(L, L.star_liem_spatial_gate(_p(x), _p(w98), _p(mm), _p(gate), BT, H, W, C, 0, rows, _st()),
             "star_liem_spatial_gate")
    return gate


def _liem_part(x, w98, BT, H, W, part):
    L, dt = _bind(part.mm)
    assert part.mm.is_contiguous() and tuple(part.mm.shape) == (BT * H * W, 2)
    C = 8
    if x is not None:
        _h(x, "x", dt)
        assert x.is_contiguous() and x.shape[0] == part.n
        C = x.shape[1]
    gate = torch.empty((part.n,), dtype=dt, device=part.mm.device) if w98 is not None else None
    _L.check(L, L.star_liem_spatial_gate(_p(x), _p(w98), _p(part.mm), _p(gate), BT, H, W, C, int(part.r0), int(part.n),
                                         _st()), "star_liem_spatial_gate")
    return part.mm if gate is None else gate


@_traced
def concat_add(a, b, c=None):
    L, dt = _bind(a)
    rows, Ca = a.shape
    Cb = b.shape[1]
    assert a.is_contiguous() and b.is_contiguous() and (c is None or c.is_contiguous())
    out = torch.empty((rows, Ca + Cb), dtype=dt, device=a.device)
    _L.check(L, L.star_concat_add(_p(a), Ca, _p(b), _p(c), Cb, _p(out), rows, _st()), "star_concat_add")
    return out


@_traced
def add(a, b):
    L, _ = _bind(a)
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    out = torch.empty_like(a)
    _L.check(L, L.star_add(_p(a), _p(b), _p(out), a.numel(), _st()), "star_add")
    return out


@_traced
def time_avgpool2(x, T, HW):
    """frame-pair average of a [(T HW), C] clip (odd T: first frame kept): -> [(ceil(T/2) HW), C]"""
    L, dt = _bind(x)
    C = x.shape[1]
    assert x.is_contiguous() and x.shape[0] == T * HW
    To = (T + 1) // 2 if T % 2 else T // 2
    out = torch.empty((To * HW, C), dtype=dt, device=x.device)
    _L.check(L, L.star_time_avgpool2(_p(x), _p(out), T, HW, C, _st()), "star_time_avgpool2")
    return out


@_traced
def upsample2x_crop(x, BT, H, W):
    L, dt = _bind(x)
    C = x.shape[1]
    out = torch.empty((BT * (2 * H - 2) * (2 * W), C), dtype=dt, device=x.device)
    _L.check(L, L.star_upsample2x_crop(_p(x), _p(out), BT, H, W, C, _st()), "star_upsample2x_crop")
    return out


@_traced
def upsample2x(x, BT, H, W, out=None):
    """plain nearest x2: [BT*H*W, C] -> [BT*2H*2W, C]"""
    L, dt = _bind(x)
    C = x.shape[1]
    assert x.is_contiguous()
    if out is None:
        out = torch.empty((BT * 4 * H * W, C), dtype=dt, device=x.device)
    assert out.is_contiguous() and tuple(out.shape) == (BT * 4 * H * W, C)
    _L.check(L, L.star_upsample2x(_p(x), _p(out), BT, H, W, C, 0, _st()), "star_upsample2x")
    return out


@_traced
def softmax_rows(s, cols, ctas_per_row=1):
    """in-place row softmax of the fp16 matrix s[rows, ld] over its first `cols` columns; each row is split over a cluster
    of ctas_per_row CTAs (1..8) of at most 102 400 columns each"""
    L, _ = _bind(s)
    ld = _rowmajor(s, "s")
    _L.check(L, L.star_softmax_rows(_p(s), ld, s.shape[0], int(cols), int(ctas_per_row), _st()), "star_softmax_rows")
    return s


@_traced
def vae_head(x, w27, bias3, B, T, H, W):
    """x [(b t h w), ld>=3] -> (B*T, 3, H, W) fp16 after the (3,1,1) temporal conv over t"""
    L, dt = _bind(x)
    ld = _rowmajor(x, "x")
    assert w27.is_contiguous() and w27.numel() == 27 and bias3.numel() == 3
    out = torch.empty((B * T, 3, H, W), dtype=dt, device=x.device)
    _L.check(L, L.star_vae_head(_p(x), ld, _p(_h(w27, "w27", dt)), _p(_h(bias3, "bias3", dt)), _p(out), B, T, H * W, _st()),
             "star_vae_head")
    return out


@_traced
def nchw5_to_tokens(x, dtype=torch.float16):
    """(b, c, f, h, w) fp32 -> [(b f h w), c] fp16 (or bf16)"""
    L, dt = _bind(x, dtype)
    x = x.contiguous().float()
    B, C, F, H, W = x.shape
    out = torch.empty((B * F * H * W, C), dtype=dt, device=x.device)
    _L.check(L, L.star_nchw5_to_tokens(_p(x), _p(out), B, C, F, H * W, _st()), "star_nchw5_to_tokens")
    return out


@_traced
def tokens_to_nchw5(x, B, C, F, H, W):
    L, dt = _bind(x)
    out = torch.empty((B, C, F, H, W), dtype=dt, device=x.device)
    _L.check(L, L.star_tokens_to_nchw5(_p(x), _rowmajor(x, "x"), _p(out), B, C, F, H * W, _st()), "star_tokens_to_nchw5")
    return out


@_traced
def sinusoidal(t, dim, dtype=torch.float16):
    L, dt = _bind(t, dtype)
    t = t.to(torch.int64).contiguous()
    out = torch.empty((t.shape[0], dim), dtype=dt, device=t.device)
    _L.check(L, L.star_sinusoidal(_p(t), _p(out), t.shape[0], dim, _st()), "star_sinusoidal")
    return out


@_traced
def silu(x):
    L, _ = _bind(x)
    assert x.is_contiguous()
    out = torch.empty_like(x)
    _L.check(L, L.star_silu(_p(x), _p(out), x.numel(), _st()), "star_silu")
    return out


@_traced
def bilinear_pad(x, H, W, padding=(0, 0, 0, 0), value=1.0):
    """F.interpolate(x, [H, W], mode='bilinear') + F.pad(x, padding=(l, r, t, b), 'constant', value); x fp32 (..., h, w)"""
    L, _ = _bind(x)
    if x.dtype != torch.float32:
        raise _L.StarError("bilinear_pad expects fp32 frames")
    x = x.contiguous()
    *lead, h, w = x.shape
    pl, pr, pt, pb = (int(v) for v in padding)
    out = torch.empty((*lead, H + pt + pb, W + pl + pr), dtype=torch.float32, device=x.device)
    nc = 1
    for d in lead:
        nc *= d
    _L.check(L, L.star_bilinear_pad(_p(x), _p(out), nc, h, w, int(H), int(W), pl, pr, pt, pb, float(value), _st()),
             "star_bilinear_pad")
    return out


@_traced
def adain_color_fix(video, source, uint8=False):
    """tensor2vid + adain_color_fix on the GPU: video (1, C, F, H, W) fp32 in [-1, 1] (test()'s result), source (F, C, h, w) fp32 in
    [-1, 1] (the LR clip) -> (F, H, W, C) in [0, 255], fp32 like the reference or uint8 (rounded; 4x less D2H traffic)."""
    L, _ = _bind(video)
    assert video.dim() == 5 and video.shape[0] == 1 and video.dtype == torch.float32 and source.dtype == torch.float32
    _, C, F, H, W = video.shape
    assert source.shape[0] == F and source.shape[1] == C
    video, source = video.contiguous(), source.to(video.device).contiguous()
    out = torch.empty((F, H, W, C), dtype=torch.uint8 if uint8 else torch.float32, device=video.device)
    ws = torch.empty(L.star_adain_workspace_bytes(C, F), dtype=torch.uint8, device=video.device)
    _L.check(L, L.star_adain_color_fix(_p(video), _p(source), None if uint8 else _p(out), _p(out) if uint8 else None, C, F, H * W,
                                       source.shape[2] * source.shape[3], _p(ws), _st()), "star_adain_color_fix")
    return out


class TileBlend(NamedTuple):
    """Where ``cfg_x0(..., blend=)`` accumulates one (chunk, tile) x0 in tiled sampling: the clip-level fp32 accumulator
    (B, C, F, H, W), the tile's frame / row / column offset in the clip (f0, r0, c0), the kept tile-local frames [lo, hi)
    and the tile's fp32 row / column blend weights wy (th,), wx (tw,) on the device."""
    acc: torch.Tensor
    f0: int
    lo: int
    hi: int
    r0: int
    c0: int
    wy: torch.Tensor
    wx: torch.Tensor


@_traced
def cfg_x0(y_out, u_out, xt, alphas, sigmas, guide_scale, guide_rescale=None, return_guided=False, blend=None):
    """x0 = alphas * xt - sigmas * rescale(u + g (y - u)); y_out / u_out fp16 (B, ...), xt fp32, alphas / sigmas fp32 (B, 1, ...)

    With ``blend`` (a TileBlend), y_out / u_out are the outputs of one tile (B, C, Ft, th, tw), xt is the CLIP-level latent
    (B, C, F, H, W) fp32 contiguous, read in place at the tile's window, and x0 is not returned but accumulated:
    blend.acc[:, :, f0 + lo:f0 + hi, r0:r0 + th, c0:c0 + tw] += wy[:, None] * wx[None, :] * x0[:, :, lo:hi]; returns blend.acc.
    The rescale statistics span the whole tile output."""
    L, dt = _bind(y_out)
    _h(y_out, "y_out", dt); _h(u_out, "u_out", dt)
    if blend is not None:
        return _cfg_x0_blend(L, y_out, u_out, xt, alphas, sigmas, guide_scale, guide_rescale, return_guided, blend)
    assert y_out.is_contiguous() and u_out.is_contiguous() and y_out.shape == u_out.shape == xt.shape
    B = y_out.shape[0]
    per = y_out.numel() // B
    xt = xt.float().contiguous()
    x0 = torch.empty_like(xt)
    guided = torch.empty_like(y_out) if return_guided else None
    al = alphas.reshape(B).float().contiguous()
    sg = sigmas.reshape(B).float().contiguous()
    ws = torch.empty(L.star_cfg_x0_workspace_bytes(B), dtype=torch.uint8, device=y_out.device)
    _L.check(L, L.star_cfg_x0(_p(y_out), _p(u_out), _p(xt), _p(x0), _p(guided), float(guide_scale),
                              -1.0 if guide_rescale is None else float(guide_rescale), _p(al), _p(sg), B, per, _p(ws), _st()),
             "star_cfg_x0")
    return (x0, guided) if return_guided else x0


def _cfg_x0_blend(L, y_out, u_out, xt, alphas, sigmas, guide_scale, guide_rescale, return_guided, blend):
    if return_guided:
        raise ValueError("cfg_x0: return_guided is not available with blend=")
    acc = blend.acc
    if y_out.dim() != 5 or y_out.shape != u_out.shape or not (y_out.is_contiguous() and u_out.is_contiguous()):
        raise ValueError(f"cfg_x0(blend=): y_out / u_out must be contiguous (B, C, Ft, th, tw), got {tuple(y_out.shape)} "
                         f"and {tuple(u_out.shape)}")
    for name, t in (("xt", xt), ("blend.acc", acc), ("blend.wy", blend.wy), ("blend.wx", blend.wx)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != y_out.device:
            raise ValueError(f"cfg_x0(blend=): {name} must be a contiguous fp32 tensor on {y_out.device}")
    B, C, Ft, th, tw = y_out.shape
    if xt.dim() != 5 or acc.shape != xt.shape or xt.shape[:2] != (B, C):
        raise ValueError(f"cfg_x0(blend=): xt {tuple(xt.shape)} and acc {tuple(acc.shape)} must be the same (B, C, F, H, W) clip "
                         f"as the tile's (B, C) = ({B}, {C})")
    if blend.wy.shape != (th,) or blend.wx.shape != (tw,):
        raise ValueError(f"cfg_x0(blend=): weights {tuple(blend.wy.shape)} / {tuple(blend.wx.shape)} do not match the tile {th}x{tw}")
    _, _, F, H, W = xt.shape
    al = alphas.reshape(B).float().contiguous()
    sg = sigmas.reshape(B).float().contiguous()
    ws = torch.empty(L.star_cfg_x0_workspace_bytes(B), dtype=torch.uint8, device=y_out.device)
    _L.check(L, L.star_cfg_x0_blend(_p(y_out), _p(u_out), _p(xt), _p(acc), float(guide_scale),
                                    -1.0 if guide_rescale is None else float(guide_rescale), _p(al), _p(sg), _p(blend.wy),
                                    _p(blend.wx), B, C, Ft, th, tw, F, H, W, int(blend.f0), int(blend.lo), int(blend.hi),
                                    int(blend.r0), int(blend.c0), _p(ws), _st()),
             "star_cfg_x0_blend")
    return acc


FLAG_GELU_TANH = 8


@_traced
def linear_ex(a, w, bias=None, colscale=None, residual=None, flags=0, out=None):
    """out = residual + colscale[n] * act(sum_k a[r,k] w[n,k] + bias[n])   (adaLN-gated residual, tanh-GELU option).
    a is a strided 2-D view [rows, K], or a head-blocked A: a 3-D view [blocks, rows, block_cols] with contiguous columns
    whose row r is its blocks' rows r side by side (K = blocks * block_cols), read in place."""
    L, dt = _bind(a)
    block_cols = pitch = 0
    if a.dim() == 3:
        if a.stride(2) != 1:
            raise _L.StarError("a head-blocked a must have contiguous columns")
        blocks, rows, block_cols = a.shape
        lda, pitch, K = a.stride(1), a.stride(0), blocks * block_cols
    else:
        lda = _rowmajor(a, "a")
        rows, K = a.shape
    N = w.shape[0]
    assert w.is_contiguous() and w.shape[1] == K
    if out is None:
        out = torch.empty((rows, N), dtype=dt, device=a.device)
    ldres = _rowmajor(residual, "residual") if residual is not None else 0
    _L.check(L, L.star_linear_ex(_p(a), lda, _p(w), _p(bias), None, 1, _p(colscale), _p(residual), ldres, _p(out),
                                 _rowmajor(out, "out"), rows, K, N, flags, block_cols, pitch, _st()), "star_linear_ex")
    return out


@_traced
def row_gate(x, mode, gate=None, w0=0.0, w1=0.0, out=None):
    L, _ = _bind(x)
    rows, C = x.shape
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    _L.check(L, L.star_row_gate(_p(x), _p(out), rows, C, mode, _p(gate), float(w0), float(w1), _st()), "star_row_gate")
    return out


@_traced
def qk_ln_rope(qkv, heads, koff, qg, qb, kg, kb, cos, sin, seq, text_len, eps=1e-6):
    """in place on qkv [rows, ld]"""
    L, _ = _bind(qkv)
    ld = _rowmajor(qkv, "qkv")
    assert cos.dtype == torch.float32 and sin.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous()
    _L.check(L, L.star_qk_ln_rope(_p(qkv), ld, qkv.shape[0], heads, koff, _p(qg), _p(qb), _p(kg), _p(kb), _p(cos), _p(sin),
                                  seq, text_len, float(eps), _st()), "star_qk_ln_rope")
    return qkv
