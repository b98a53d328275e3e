"""Per-element error bounds of the flash-attention and long temporal-attention kernels past their ring depths, at the shapes
the UNet, the CogVideoX DiT and the text tower run.

The checker, the error model and attention_core are those of tests/test_kernel_bounds_gpu.py: every output element must
satisfy |got - y| <= u |y| + (1 + u) E + floor against an fp64 reference.  E is relative to P|V| (the softmax weights times
|V|), and with random N(0, 1) inputs P|V| grows like sqrt(Nk) |y| while one missing key moves y by about |y| / Nk:
test_random_inputs_miss_a_dropped_key shows the bound passing a dropped key at Nk = 26 352.  So every case here runs inputs
designed to keep the bound at a few ulps and to turn a tile-level fault into an O(1) error.  In every head:

  needle rows    (query index % 4 in {0, 1}) score one key, their needle, at +12 over the rest: q = 2 h_i, needle key 1.5 h_i
                 on dims 32..63 with h_i a row of the 32 x 32 Hadamard matrix (needles are orthogonal to each other), the
                 other keys N(0, 1/4) there.  Needles sit in every K/V ring slot before the first wrap, after it and after
                 the second, in tiles spread over the rest of the keys, and at the last key (the partial last tile).  Every
                 query tile holds a needle row for every needle, so a stale, skipped or duplicated tile, or a wrong ring
                 phase, moves some row by O(1).  Causal problems also point the row before each needle at it (a key one
                 past the causal limit) and the needle's own row (the diagonal).
  negative rows  (% 4 == 2) score every real key at -12 (dim 0: key 4 s, query -24 s).  s = +-1 alternates between kv batches
                 (flash) or neighbouring pixels and heads (temporal), so a zero-filled padding key (score 0) or a key of the
                 wrong batch / item (score +12) takes most of the weight.
  spread rows    (% 4 == 3) q ~ N(0, 1/4): scores within a few units of each other.
and V is N(0, 1) on dims 0..31 and mean-shifted, 1 + N(0, 1/16), on dims 32..63, where P|V| ~ |y|: a tile missing from the
softmax denominator, or a rescale applied twice, exceeds the bound there.

test_tables_cover_every_ring_path parses the ring depths from the kernel headers and requires the case tables to reach every
ring / phase cell; test_checker_catches_simulated_attention_faults simulates tile-level faults in fp64 and requires the
checker to reject each.  GPU cases print the worst |err| / bound per family and per (row design, V half); the module prints
its runtime and peak device memory (pytest -s).
"""
import os
import re
import time
from collections import namedtuple

import pytest
import torch

from tests.test_kernel_bounds_gpu import (BoundCheck, WORST, NUM_SMS, HALF, BF16, F64, attention_core, attention_ref,
                                          check_bound, temporal_ref, _ceil, _rnd)
from tests.util import assert_close

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_consts(name, *keys):
    src = open(os.path.join(ROOT, "star_b200", "csrc", name)).read()
    return {k: int(re.search(rf"constexpr int {k} = (\d+);", src).group(1)) for k in keys}


_AT = _header_consts("attn.cuh", "AT_BQ", "AT_BKV", "AT_KV_STAGES")
_TL = _header_consts("tattn_long.cuh", "TL_BT", "TL_Q_SLOTS", "TL_KV_STAGES")
BQ, BKV, STAGES = _AT["AT_BQ"], _AT["AT_BKV"], _AT["AT_KV_STAGES"]
TL_BT, TL_Q_SLOTS, TL_KV_STAGES = _TL["TL_BT"], _TL["TL_Q_SLOTS"], _TL["TL_KV_STAGES"]

SCALE = 0.125                  # the designs' scores (+-12) assume the pipelines' 1 / sqrt(64)
MAX_NEEDLES = 32               # orthogonal needle directions: rows of the 32 x 32 Hadamard matrix
CHUNK = 1 << 25                # fp64 score elements per reference chunk (256 MB per intermediate)
GROUPS = ("needle", "negative", "spread")
ROW_GROUP = torch.tensor([0, 0, 1, 2])     # design of query index % 4


def _hadamard32():
    h = torch.ones(1, 1)
    while h.shape[0] < MAX_NEEDLES:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


H32 = _hadamard32()


# ---- input designs -------------------------------------------------------------------------------------------------------
def flash_needles(nk, shift):
    """key positions of the needles of one kv batch: one in each of the first 3 AT_KV_STAGES tiles (every ring slot before
    the first wrap, after it and after the second), one in tiles spread over the rest, and the last key"""
    nt = _ceil(nk, BKV)
    tiles = list(range(min(nt, 3 * STAGES)))
    rest = MAX_NEEDLES - 1 - len(tiles)
    if nt > 3 * STAGES:
        tiles += sorted({3 * STAGES + (nt - 1 - 3 * STAGES) * i // rest for i in range(1, rest + 1)})
    pos = []
    for j in tiles:
        p = BKV * j + (17 * j + 5 + 3 * shift) % min(BKV, nk - BKV * j)
        if p != nk - 1 and p not in pos:
            pos.append(p)
    return pos + [nk - 1]


def flash_inputs(batch, heads, nq, nk, div, causal, dtype, device, seed=1):
    """q [batch nq, heads 64], k / v [kv batches nk, heads 64] of the designs above, and the design of every query row"""
    g = torch.Generator(device=device).manual_seed(seed)
    kvb = _ceil(batch, div)
    needles = [flash_needles(nk, b) for b in range(kvb)]
    n = min(len(p) for p in needles)
    r = torch.arange(nq)
    group = ROW_GROUP[r % 4].repeat(batch, 1)
    target = (((r % BQ) // 4 * 2 + r % 4) % n).repeat(batch, 1)       # needle ordinal within the query tile, mod n
    if causal:
        for b in range(batch):
            for i, p in enumerate(needles[b // div][:n]):
                for row in (p - 1, p):
                    if 0 <= row < nq:
                        group[b, row], target[b, row] = 0, i
    group, target = group.to(device), target.to(device)
    h32 = H32.to(device)
    sig_kv = 1.0 - 2.0 * (torch.arange(kvb, device=device) % 2)
    sig_q = sig_kv[torch.arange(batch, device=device) // div][:, None].expand(batch, nq)

    noise = torch.randn(batch, nq, heads, 64, generator=g, device=device)
    q = torch.zeros(batch, nq, heads, 64, device=device)
    spr, neg, nd = group == 2, group == 1, group == 0
    q[spr] = 0.5 * noise[spr]
    q[neg, :, 0] = -24.0 * sig_q[neg][:, None]
    q[neg, :, 1:32] = 0.25 * noise[neg][:, :, 1:32]
    q[nd, :, 32:] = 2.0 * h32[target[nd]][:, None, :]
    k = 0.5 * torch.randn(kvb, nk, heads, 64, generator=g, device=device)
    k[..., 0] = 4.0 * sig_kv[:, None, None]
    for b in range(kvb):
        k[b, torch.tensor(needles[b], device=device), :, 32:] = 1.5 * h32[:len(needles[b]), None, :]
    v = torch.randn(kvb, nk, heads, 64, generator=g, device=device)
    v[..., 32:] = 1.0 + 0.25 * v[..., 32:]
    flat = lambda t: t.reshape(t.shape[0] * t.shape[1], heads * 64).to(dtype)     # noqa: E731
    return flat(q), flat(k), flat(v), group.reshape(-1), needles


def temporal_needle(j, nblk, T, shift):
    """frame of the needle key in 64-frame key block j; the last block's needle is the last frame"""
    return T - 1 if j == nblk - 1 else TL_BT * j + (13 * j + 5 + 7 * shift) % TL_BT


def temporal_design(T):
    """design and needle target block of every query frame: every query tile has a needle row for every key block"""
    nblk = _ceil(T, TL_BT)
    t = torch.arange(T)
    return ROW_GROUP[t % 4], ((t % TL_BT) // 4 * 2 + t % 4 + t // TL_BT) % nblk


def temporal_inputs(qkv, B, T, HW, heads, Ci, seed=1):
    """fill the q / k / v columns of qkv [B T HW, ld] with the designs (needle positions shift with (b + px) % 3, the sign of
    the negative rows alternates with b + px + head); returns the design of every frame"""
    dev, dt = qkv.device, qkv.dtype
    g = torch.Generator(device=dev).manual_seed(seed)
    nblk = _ceil(T, TL_BT)
    group, target = temporal_design(T)
    group, target = group.to(dev), target.to(dev)
    spr, neg, nd = group == 2, group == 1, group == 0
    h32 = H32.to(dev)
    x = qkv.view(B, T, HW, -1)
    C = heads * 64
    step = max(1, (1 << 24) // (B * T * heads * 64))
    for p0 in range(0, HW, step):
        p1 = min(HW, p0 + step)
        P = p1 - p0
        px = torch.arange(p0, p1, device=dev)
        bb = torch.arange(B, device=dev)[:, None, None]
        sig = 1.0 - 2.0 * ((bb + px[None, :, None] + torch.arange(heads, device=dev)[None, None, :]) % 2)   # [B, P, heads]
        noise = torch.randn(B, T, P, heads, 64, generator=g, device=dev)
        q = torch.zeros(B, T, P, heads, 64, device=dev)
        q[:, spr] = 0.5 * noise[:, spr]
        q[:, neg, :, :, 0] = -24.0 * sig[:, None]
        q[:, neg, :, :, 1:32] = 0.25 * noise[:, neg, :, :, 1:32]
        q[:, nd, :, :, 32:] = 2.0 * h32[target[nd]][None, :, None, None, :]
        k = 0.5 * torch.randn(B, T, P, heads, 64, generator=g, device=dev)
        k[..., 0] = 4.0 * sig[:, None]
        for b in range(B):
            shift = (b + px) % 3
            for s in range(3):
                sel = (shift == s).nonzero().squeeze(1)
                for j in range(nblk):
                    k[b, temporal_needle(j, nblk, T, s), sel, :, 32:] = 1.5 * h32[j]
        v = torch.randn(B, T, P, heads, 64, generator=g, device=dev)
        v[..., 32:] = 1.0 + 0.25 * v[..., 32:]
        for off, t in ((0, q), (Ci, k), (2 * Ci, v)):
            x[:, :, p0:p1, off:off + C] = t.reshape(B, T, P, C).to(dt)
    return group


# ---- chunked fp64 references and the per-design report --------------------------------------------------------------------
DESIGN_WORST = {}


def _design_add(family, got, y, bound, group):
    """worst |err| / bound per (row design, V half) of one chunk; group: the design of every row"""
    ratio = ((got.to(F64) - y).abs() / bound).view(got.shape[0], -1, 2, 32).amax(dim=(1, 3))   # [rows, V half]
    for gi, gname in enumerate(GROUPS):
        sel = group == gi
        if bool(sel.any()):
            for hi, vname in enumerate(("randV", "shiftV")):
                key = (family, gname, vname)
                DESIGN_WORST[key] = max(DESIGN_WORST.get(key, 0.0), ratio[sel, hi].max().item())


def flash_check(chk, family, got, q, k, v, batch, heads, nq, nk, div, dtype, causal, group):
    """compare got [batch nq, heads 64] with attention_core over (batch, head group, query chunk)"""
    rstep = min(nq, max(BQ, CHUNK // nk))
    hstep = max(1, min(heads, CHUNK // (rstep * nk)))
    for b in range(batch):
        kb = b // div
        for h0 in range(0, heads, hstep):
            h1 = min(heads, h0 + hstep)
            cols, hh = slice(h0 * 64, h1 * 64), h1 - h0
            kf = k[kb * nk:(kb + 1) * nk, cols].to(F64).view(nk, hh, 64).transpose(0, 1)
            vf = v[kb * nk:(kb + 1) * nk, cols].to(F64).view(nk, hh, 64).transpose(0, 1)
            for r0 in range(0, nq, rstep):
                r1 = min(nq, r0 + rstep)
                qf = q[b * nq + r0:b * nq + r1, cols].to(F64).view(r1 - r0, hh, 64).transpose(0, 1)
                y, bd = attention_core(qf, kf, vf, SCALE, dtype, causal, q0=r0)
                y, bd = (t.transpose(0, 1).reshape(r1 - r0, hh * 64) for t in (y, bd))
                g = got[b * nq + r0:b * nq + r1, cols]
                chk.add(g, y, bd, row0=b * nq + r0, col0=h0 * 64)
                _design_add(family, g, y, bd, group[b * nq + r0:b * nq + r1])
                del y, bd
    return chk


def temporal_check(chk, family, out, qkv, B, T, HW, heads, Ci, dtype, group):
    """compare the temporal output [B T HW, >= heads 64] with attention_core over pixel chunks"""
    x, o = qkv.view(B, T, HW, -1), out.view(B, T, HW, -1)
    C = heads * 64
    step = max(1, CHUNK // (B * heads * T * T))
    dev = qkv.device
    for p0 in range(0, HW, step):
        p1 = min(HW, p0 + step)
        P = p1 - p0
        xs = x[:, :, p0:p1].to(F64)
        split = lambda off: xs[..., off:off + C].reshape(B, T, P, heads, 64).permute(0, 2, 3, 1, 4)     # noqa: E731
        y, bd = attention_core(split(0), split(Ci), split(2 * Ci), SCALE, dtype)
        y, bd = (t.permute(0, 3, 1, 2, 4).reshape(B * T * P, C) for t in (y, bd))
        del xs
        g = o[:, :, p0:p1, :C].reshape(B * T * P, C)
        rows = ((torch.arange(B, device=dev)[:, None, None] * T + torch.arange(T, device=dev)[None, :, None]) * HW
                + torch.arange(p0, p1, device=dev)[None, None, :]).reshape(-1)
        chk.add(g, y, bd, rows=rows.cpu())
        _design_add(family, g, y, bd, group.to(dev)[None, :, None].expand(B, T, P).reshape(-1))
        del y, bd
    return chk


def flash_locator(nq, group):
    def locate(r, c):
        qr = r % nq
        return (f"[batch {r // nq}, q-tile {qr // BQ}, query {qr}, head {c // 64}, {GROUPS[int(group[r])]} row, "
                f"{'shifted' if c % 64 >= 32 else 'random'} V]")
    return locate


def temporal_locator(T, HW, heads, group):
    def locate(r, c):
        t, px, b = r // HW % T, r % HW, r // (T * HW)
        return (f"[item {(b * HW + px) * heads + c // 64} (b {b}, px {px}, head {c // 64}), frame {t}, q-tile {t // TL_BT}, "
                f"{GROUPS[int(group[t])]} row, {'shifted' if c % 64 >= 32 else 'random'} V]")
    return locate


# ---- case tables ---------------------------------------------------------------------------------------------------------
# layout "qkv": q / k / v are column slices of one [batch N, 3 C] buffer, as the self-attention callers pass them;
# "sep": q [batch Nq, C] and a [kv batches Nk, 2 C] k | v buffer, as the text cross-attention passes them.
A = namedtuple("A", "id dtype batch heads nq nk div causal layout")


def _ring_cases(dtype, tag):
    out = []
    for nt in (4, 5, 8, 9, 13):
        for partial in (False, True):
            nk = nt * BKV - (37 if partial else 0)
            nq = 65 if partial else 300                          # one partial q-tile / a ragged third q-tile
            out.append(A(f"{tag}-nt{nt}-{'partial' if partial else 'full'}", dtype, 3, 2, nq, nk, 2, False, "sep"))
    return out


FLASH_CASES = _ring_cases(HALF, "fp16") + _ring_cases(BF16, "bf16") + [
    A("causal-N513", HALF, 2, 2, 513, 513, 1, True, "qkv"),
    A("causal-N640", HALF, 2, 2, 640, 640, 1, True, "qkv"),
    # UNet self-attention at the bench size (960p latent 122 x 216): levels 0-2 and the middle block, heads = C / 64
    A("unet-self-L0", HALF, 2, 5, 26352, 26352, 1, False, "qkv"),
    A("unet-self-L1", HALF, 2, 10, 6588, 6588, 1, False, "qkv"),
    A("unet-self-L2", HALF, 2, 20, 1674, 1674, 1, False, "qkv"),
    A("unet-self-mid", HALF, 2, 20, 432, 432, 1, False, "qkv"),
    # UNet text cross-attention: batch B T over B text contexts (kv_batch_div = T); T = 32, and T = 5 over 21 frames
    A("unet-cross-T32", HALF, 64, 20, 432, 77, 32, False, "sep"),
    A("unet-cross-T5-ragged", HALF, 21, 5, 300, 77, 5, False, "sep"),
    # CogVideoX DiT full attention over text + video tokens, bf16
    A("dit-S17776", BF16, 2, 48, 17776, 17776, 1, False, "qkv"),
    # OpenCLIP text tower: causal, 77 tokens, 16 heads
    A("text-tower-N77", HALF, 2, 16, 77, 77, 1, True, "qkv"),
]

# B, T, HW, heads, Ci, ld, dtype: 148 items over 132 persistent CTAs (16 CTAs run two items) unless noted
TL = namedtuple("TL", "B T HW heads Ci ld dtype")
TEMPORAL_LONG_CASES = [TL(2, t, 37, 2, 128, 384, HALF) for t in (65, 100, 127, 128, 129, 191, 192, 193, 256, 257, 513, 1024)] + [
    TL(1, 257, 70, 3, 256, 832, HALF),          # heads 64 < Ci, ld > 3 Ci; 210 items
    TL(2, 193, 37, 2, 128, 384, BF16),
    TL(1, 78, 26352, 5, 320, 960, HALF),        # UNet level 0 (960p latent): a 78-frame and a 128-frame chunk
    TL(1, 128, 26352, 5, 320, 960, HALF),
]


def _flash_tiles(c):
    """K/V tiles of the CTA that loads the most (causal: the last query tile)"""
    nt = _ceil(c.nk, BKV)
    return min(nt, _ceil(c.nq, BKV)) if c.causal else nt


def _temporal_plan(c):
    nblk = _ceil(c.T, TL_BT)
    rounds = _ceil(nblk, 2)
    items = c.B * c.HW * c.heads
    per_cta = _ceil(items, min(items, NUM_SMS))
    return nblk, rounds, items, per_cta


# ---- CPU: coverage and simulated faults ----------------------------------------------------------------------------------
def test_tables_cover_every_ring_path():
    cells = set()
    for c in FLASH_CASES:
        nt = _flash_tiles(c)
        wraps = (nt - 1) // STAGES
        cells.add(("flash wraps", min(wraps, 2)))
        if wraps:
            cells.add(("flash last tile after a wrap", "partial" if c.nk % BKV else "full"))
            if c.causal:
                cells.add(("flash causal after a wrap",))
        if c.dtype == BF16:
            cells.add(("flash bf16", min(wraps, 2)))
        if c.div > 2:
            cells.add(("flash kv_batch_div > 2", "ragged" if c.batch % c.div else "even"))
        cells.add(("flash q tiles", "one partial" if c.nq < BQ else "ragged" if c.nq % BQ else "full"))
        # every (ring slot, phase) the case reaches, and its last key, hold a needle in every kv batch
        for b in range(_ceil(c.batch, c.div)):
            pos = flash_needles(c.nk, b)
            assert len(pos) <= MAX_NEEDLES and len(set(pos)) == len(pos) and max(pos) == c.nk - 1, c.id
            reached = {(j % STAGES, min(j // STAGES, 2)) for j in range(nt)}
            held = {(p // BKV % STAGES, min(p // BKV // STAGES, 2)) for p in pos}
            assert reached <= held, f"{c.id}: ring cells without a needle {sorted(reached - held)}"
    want = {("flash wraps", w) for w in (0, 1, 2)}
    want |= {("flash last tile after a wrap", f) for f in ("full", "partial")}
    want |= {("flash causal after a wrap",), ("flash bf16", 2), ("flash kv_batch_div > 2", "ragged"),
             ("flash kv_batch_div > 2", "even")}
    want |= {("flash q tiles", f) for f in ("one partial", "ragged")}

    for c in TEMPORAL_LONG_CASES:
        nblk, rounds, items, per_cta = _temporal_plan(c)
        assert c.T > 64 and nblk <= MAX_NEEDLES
        cells.add(("tl nblk", "odd" if nblk % 2 else "even"))
        if rounds > TL_Q_SLOTS:
            cells.add(("tl rounds > Q slots",))
        if per_cta * rounds > TL_Q_SLOTS:
            cells.add(("tl Q ring wraps within a CTA",))
        if per_cta * rounds * nblk > TL_KV_STAGES:
            cells.add(("tl K/V loads per CTA > stages",))
        if items > NUM_SMS and items % NUM_SMS:
            cells.add(("tl items > SMs",))
        if rounds * nblk % TL_KV_STAGES and per_cta > 1:
            cells.add(("tl second item starts mid-ring",))
        if c.heads * 64 < c.Ci and c.ld > 3 * c.Ci:
            cells.add(("tl strided heads",))
        if c.dtype == BF16:
            cells.add(("tl bf16",))
        group, target = temporal_design(c.T)
        for t0 in range(0, c.T, TL_BT):                      # every full query tile holds a needle row for every key block
            if t0 + TL_BT <= c.T:
                assert set(target[t0:t0 + TL_BT][group[t0:t0 + TL_BT] == 0].tolist()) == set(range(nblk))
    want |= {("tl nblk", "odd"), ("tl nblk", "even"), ("tl rounds > Q slots",), ("tl Q ring wraps within a CTA",),
             ("tl K/V loads per CTA > stages",), ("tl items > SMs",), ("tl second item starts mid-ring",),
             ("tl strided heads",), ("tl bf16",)}
    missing = want - cells
    assert not missing, f"ring / phase cells without a case: {sorted(map(str, missing))}"


def _flash_cpu(nq, nk, k_fn=None):
    """fp64 value and bound of one head of the flash designs on the CPU; k_fn(k, v) -> (k, v) simulates a fault"""
    q, k, v, group, needles = flash_inputs(1, 1, nq, nk, 1, False, HALF, "cpu")
    y, b = attention_ref(q, k, v, 1, 1, nq, nk, 1, SCALE, HALF)
    if k_fn is None:
        return q, k, v, group, needles, y, b
    k2, v2 = k_fn(k.clone(), v.clone())
    return attention_ref(q, k2, v2, 1, 1, nq, k2.shape[0], 1, SCALE, HALF)[0]


def test_checker_catches_simulated_attention_faults():
    """Each tile-level fault, simulated in fp64 on the UNet level-0 key count and rounded to fp16, fails the per-element
    check of the designed inputs; the fault-free result passes it.  Prints which faults assert_close lets through."""
    nq, nk = BQ, 26352                                   # 206 K/V tiles, the last one partial
    q, k, v, group, needles, y, b = _flash_cpu(nq, nk)
    check_bound(y.half(), y, b, "clean designed attention")
    nd = (group == 0).nonzero().squeeze(1)
    faults = {}

    def stale(k, v, j=STAGES):                          # tile j served from the slot of tile j - AT_KV_STAGES
        k[j * BKV:(j + 1) * BKV], v[j * BKV:(j + 1) * BKV] = k[(j - STAGES) * BKV:(j - STAGES + 1) * BKV], \
            v[(j - STAGES) * BKV:(j - STAGES + 1) * BKV]
        return k, v
    faults["stale tile"] = _flash_cpu(nq, nk, stale).half()

    assert (nk - 1) // BKV >= 2 * STAGES                 # the last key sits after two wraps of the ring
    g = y.half()
    g[nd] = _flash_cpu(nq, nk, lambda k, v: (k[:nk - 1], v[:nk - 1]))[nd].half()
    faults["needle in the partial last tile dropped"] = g

    neg_row = int((group == 1).nonzero()[0])
    g = y.half()
    pad = lambda k, v: (torch.cat([k, k.new_zeros(1, 64)]), torch.cat([v, v.new_zeros(1, 64)]))    # noqa: E731
    g[neg_row] = _flash_cpu(nq, nk, pad)[neg_row].half()
    faults["one zero-filled padding key leaked into a negative row"] = g

    spr_row = int((group == 2).nonzero()[0])
    q64, k64, v64 = q.double(), k.double(), v.double()
    e = torch.exp((q64[spr_row] @ k64.t()) * SCALE - ((q64[spr_row] @ k64.t()) * SCALE).max())
    j = nk // BKV - 1                                    # one full tile missing from l only
    l_short = e.sum() - e[j * BKV:(j + 1) * BKV].sum()
    g = y.half()
    g[spr_row, 32:] = ((e @ v64[:, 32:]) / l_short).half()
    faults["a tile missing from l, mean-shifted V"] = g

    # the long temporal kernel: T = 150 has 3 key blocks, so the last round runs one query tile on one warpgroup
    B, T, HW, heads, Ci = 1, 150, 3, 2, 128
    qkv = torch.zeros(B * T * HW, 3 * Ci, dtype=HALF)
    tgroup = temporal_inputs(qkv, B, T, HW, heads, Ci)
    yt, bt = temporal_ref(qkv, B, T, HW, heads, Ci, SCALE, HALF)
    check_bound(yt.half(), yt, bt, "clean designed temporal attention")
    last = (torch.arange(2 * TL_BT, T) * HW + 1)        # frames of the odd last round, pixel 1
    g = yt.half()
    g[last, :64] = 0
    faults["temporal: odd last round left unwritten"] = (g, yt, bt)
    g = yt.half()
    g[last, :64] = yt[last - 1, 64:].half()             # the previous item: pixel 0, head 1
    faults["temporal: odd last round written from the previous item"] = (g, yt, bt)

    missed = []
    for name, f in faults.items():
        got, ref, bound = f if isinstance(f, tuple) else (f, y, b)
        with pytest.raises(AssertionError):
            check_bound(got, ref, bound, name)
        try:
            assert_close(got, ref.half(), what=name)
            missed.append(name)
        except AssertionError:
            pass
    print("[attention bounds] faults assert_close lets pass:", missed)


def test_random_inputs_miss_a_dropped_key():
    """Why the designs exist: with random N(0, 1) q / k / v at the UNet level-0 key count, the bound lets a dropped key pass."""
    nq, nk = 64, 26352
    q, k, v = (_rnd((nq if i == 0 else nk, 64), 1 + i, device="cpu") for i in range(3))
    y, b = attention_ref(q, k, v, 1, 1, nq, nk, 1, SCALE, HALF)
    short, _ = attention_ref(q, k[:nk - 1], v[:nk - 1], 1, 1, nq, nk - 1, 1, SCALE, HALF)
    assert check_bound(short.half(), y, b, "random inputs, last key dropped") <= 1.0


# ---- GPU -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    from star_b200 import ops as O
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield O
    fams = {k: round(w, 3) for k, w in sorted(WORST.items()) if k.startswith(("flash", "temporal-long"))}
    print(f"\n[attention bounds] worst |err|/bound per family: {fams}")
    for (fam, gname, vname), w in sorted(DESIGN_WORST.items()):
        print(f"[attention bounds]   {fam:22s} {gname:9s} {vname}: {w:.3f}")
    print(f"[attention bounds] {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _family(dtype, causal, prefix="flash"):
    return prefix + ("-causal" if causal else "") + ("-bf16" if dtype == BF16 else "-fp16")


@pytest.mark.gpu
@pytest.mark.parametrize("c", FLASH_CASES, ids=[c.id for c in FLASH_CASES])
def test_flash_attention_designed_bound(ops, c):
    C = c.heads * 64
    q, k, v, group, _ = flash_inputs(c.batch, c.heads, c.nq, c.nk, c.div, c.causal, c.dtype, "cuda")
    if c.layout == "qkv":
        buf = torch.cat([q, k, v], 1)
        del q, k, v
        q, k, v = buf[:, :C], buf[:, C:2 * C], buf[:, 2 * C:]
    else:
        kv = torch.cat([k, v], 1)
        del k, v
        k, v = kv[:, :C], kv[:, C:]
    if c.causal:
        got = ops.attention_causal(q, k, v, c.batch, c.heads, c.nq, SCALE)
    else:
        got = ops.attention(q, k, v, c.batch, c.heads, c.nq, c.nk, c.div, SCALE)
    torch.cuda.synchronize()
    fam = _family(c.dtype, c.causal)
    nt = _flash_tiles(c)
    chk = BoundCheck(f"{c.id}: b{c.batch} h{c.heads} {c.nq}x{c.nk} div{c.div} ({nt} K/V tiles, ring wraps "
                     f"{(nt - 1) // STAGES})", fam, flash_locator(c.nq, group.cpu()))
    flash_check(chk, fam, got, q, k, v, c.batch, c.heads, c.nq, c.nk, c.div, c.dtype, c.causal, group).done()


@pytest.mark.gpu
@pytest.mark.parametrize("c", TEMPORAL_LONG_CASES, ids=[f"B{c.B}-T{c.T}-HW{c.HW}-h{c.heads}-Ci{c.Ci}-ld{c.ld}-"
                                                          f"{'bf16' if c.dtype == BF16 else 'fp16'}" for c in TEMPORAL_LONG_CASES])
def test_temporal_long_designed_bound(ops, c):
    g = torch.Generator(device="cuda").manual_seed(2)                # columns outside q / k / v stay random
    qkv = torch.randn(c.B * c.T * c.HW, c.ld, generator=g, device="cuda", dtype=c.dtype)
    group = temporal_inputs(qkv, c.B, c.T, c.HW, c.heads, c.Ci)
    got = ops.temporal_attention(qkv, c.B, c.T, c.HW, c.heads, c.Ci, SCALE)
    torch.cuda.synchronize()
    nblk, rounds, items, per_cta = _temporal_plan(c)
    fam = _family(c.dtype, False, "temporal-long")
    chk = BoundCheck(f"B{c.B} T{c.T} HW{c.HW} heads{c.heads} Ci{c.Ci} ld{c.ld} ({nblk} blocks, {rounds} rounds, {items} items, "
                     f"<= {per_cta} per CTA)", fam, temporal_locator(c.T, c.HW, c.heads, group))
    temporal_check(chk, fam, got, qkv, c.B, c.T, c.HW, c.heads, c.Ci, c.dtype, group).done()
