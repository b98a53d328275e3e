// star_b200 / csrc / rowops.cuh
// HBM-bound kernels of the STAR UNet on the channels-last token matrix X[R, C] (fp16,
// rows ordered (b, t, h, w)): layout conversion, GroupNorm (4-D per-frame and 5-D
// per-clip statistics), LayerNorm with fused LIEM gates, spatial LIEM gate, temporal
// self-attention over T, channel concat, nearest-upsample, stride-2 parity split, and the
// 4-channel stem convolution.  All global accesses are 128-bit along C.
#pragma once
#include "common.cuh"

namespace star {

STAR_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
STAR_DEVINL float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
STAR_DEVINL void unpack8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
STAR_DEVINL uint4 pack8(const float* f) {
    uint4 u;
    u.x = pack_half2(f[0], f[1]);
    u.y = pack_half2(f[2], f[3]);
    u.z = pack_half2(f[4], f[5]);
    u.w = pack_half2(f[6], f[7]);
    return u;
}

// ------------------------------------------------------------------ layout conversion
// (b, c, f, h, w) fp32  ->  tokens [(b f h w), c] fp16      (unet_v2v.py:1772 rearrange + autocast cast)
__global__ void nchw5_to_tokens_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int C, int F,
                                       long long HW) {
    const long long n = (long long)B * F * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long hw = i % HW;
        const long long bf = i / HW;
        const int f = (int)(bf % F), b = (int)(bf / F);
        for (int c = 0; c < C; ++c)
            out[i * C + c] = __float2half_rn(x[(((long long)b * C + c) * F + f) * HW + hw]);
    }
}
// tokens [(b f h w), c] fp16 -> (b, c, f, h, w) fp16         (unet_v2v.py:1808)
__global__ void tokens_to_nchw5_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ out, int B,
                                       int C, int F, long long HW) {
    const long long n = (long long)B * F * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long hw = i % HW;
        const long long bf = i / HW;
        const int f = (int)(bf % F), b = (int)(bf / F);
        for (int c = 0; c < C; ++c) out[(((long long)b * C + c) * F + f) * HW + hw] = x[i * ldx + c];
    }
}

// ------------------------------------------------------------------ stem conv: 3x3, Cin = 4 (unet_v2v.py:1353, :2128)
// stem conv as a tensor-core GEMM: im2col of the 4-channel input to K = 64 (36 taps*channels, zero padded) and the
// matching zero-padded weight matrix [Cout, 64]; the product runs on the tap-GEMM kernel.
__global__ void im2col_c4_kernel(const __half* __restrict__ x, __half* __restrict__ col, int BT, int H, int W) {
    const long long npix = (long long)BT * H * W;
    for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < npix; pix += (long long)gridDim.x * blockDim.x) {
        const int w0 = (int)(pix % W), h0 = (int)((pix / W) % H);
        const long long bt = pix / ((long long)W * H);
        uint2 v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = make_uint2(0, 0);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int hh = h0 + r - 1;
#pragma unroll
            for (int s2 = 0; s2 < 3; ++s2) {
                const int ww = w0 + s2 - 1;
                if (hh >= 0 && hh < H && ww >= 0 && ww < W)
                    v[r * 3 + s2] = __ldg(reinterpret_cast<const uint2*>(x + ((bt * H + hh) * W + ww) * 4));
            }
        }
        uint4* dst = reinterpret_cast<uint4*>(col + pix * 64);
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = make_uint4(v[2 * i].x, v[2 * i].y, v[2 * i + 1].x, v[2 * i + 1].y);
    }
}
__global__ void pad_w36_kernel(const __half* __restrict__ w9, __half* __restrict__ w64, int Cout) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Cout * 64) return;
    const int n = i / 64, k = i % 64;
    w64[i] = k < 36 ? w9[n * 36 + k] : __float2half_rn(0.f);
}

// ------------------------------------------------------------------ GroupNorm (32 groups)
// stats: per (sample, group) sum / sum of squares in double.  A "sample" is rows_per_sample
// consecutive rows: one frame for the 4-D GroupNorms (unet_v2v.py:610, :635, :268) and the whole
// clip (all frames) for the 5-D ones (unet_v2v.py:1002 on b c f h w, :1210-1219).
// Known limitation (gn_stats_kernel and gn_stats2_kernel): each thread sums x and x^2 in fp32 in one pass, and the variance is
// E[x^2] - E[x]^2.  At |mean| / std = r the cancellation multiplies the fp32 error of the x^2 sum by about r^2 (4096 at r = 64),
// so test_groupnorm_offset_bound's r = 64 cases sit on their bound; a shifted (or two-pass) sum is the follow-up.
constexpr int GN_THREADS = 512;
constexpr int GN_SLAB = 256;     // rows per CTA

__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const __half* __restrict__ x, double* __restrict__ stats, long long rows_per_sample, int C) {
    extern __shared__ float red[];            // [lanes][C][2]
    const int O = C / 8;
    const int lanes = max(1, GN_THREADS / O);
    const int sample = blockIdx.y;
    const long long r0 = (long long)blockIdx.x * GN_SLAB;
    const long long r1 = min(rows_per_sample, r0 + GN_SLAB);
    const __half* xs = x + (long long)sample * rows_per_sample * C;
    for (int obase = 0; obase < O; obase += GN_THREADS) {      // only loops when C/8 > 512
        const int tid = threadIdx.x;
        int oc, ln;
        if (O >= GN_THREADS) { oc = obase + tid; ln = 0; }
        else { oc = tid % O; ln = tid / O; }
        float s[8], ss[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = ss[j] = 0.f;
        const bool active = (oc < O) && (ln < lanes);
        if (active) {
            long long r = r0 + ln;
            for (; r + 3ll * lanes < r1; r += 4ll * lanes) {          // 4 independent 16-byte loads in flight
                uint4 u[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xs + (r + (long long)k * lanes) * C + oc * 8));
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float f[8];
                    unpack8(u[k], f);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { s[j] += f[j]; ss[j] = fmaf(f[j], f[j], ss[j]); }
                }
            }
            for (; r < r1; r += lanes) {
                float f[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(xs + r * C + oc * 8)), f);
#pragma unroll
                for (int j = 0; j < 8; ++j) { s[j] += f[j]; ss[j] = fmaf(f[j], f[j], ss[j]); }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                red[((size_t)ln * C + oc * 8 + j) * 2] = s[j];
                red[((size_t)ln * C + oc * 8 + j) * 2 + 1] = ss[j];
            }
        }
    }
    __syncthreads();
    // 32 groups: warp g reduces group g's (lanes x C/32 channels) partials
    const int cg = C / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int g = warp; g < 32; g += GN_THREADS / 32) {
        float s = 0.f, ss = 0.f;
        for (int i = lane; i < lanes * cg; i += 32) {
            const int ln = i / cg, c = g * cg + i % cg;
            s += red[((size_t)ln * C + c) * 2];
            ss += red[((size_t)ln * C + c) * 2 + 1];
        }
        s = warp_sum(s);
        ss = warp_sum(ss);
        if (lane == 0) {
            atomicAdd(&stats[((long long)sample * 32 + g) * 2], (double)s);
            atomicAdd(&stats[((long long)sample * 32 + g) * 2 + 1], (double)ss);
        }
    }
}

// per (sample, channel) affine: y = x * a + b,  a = gamma * rstd, b = beta - mean * a
__global__ void gn_finalize_kernel(const double* __restrict__ stats, const __half* __restrict__ gamma,
                                   const __half* __restrict__ beta, float* __restrict__ ab, long long rows_per_sample,
                                   int C, float eps) {
    const int sample = blockIdx.x;
    const int cg = C / 32;
    const double cnt = (double)rows_per_sample * cg;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cg;
        const double mean = stats[((long long)sample * 32 + g) * 2] / cnt;
        double var = stats[((long long)sample * 32 + g) * 2 + 1] / cnt - mean * mean;
        if (var < 0) var = 0;
        const float rstd = (float)(1.0 / sqrt(var + (double)eps));
        const float a = __half2float(gamma[c]) * rstd;
        ab[((long long)sample * C + c) * 2] = a;
        ab[((long long)sample * C + c) * 2 + 1] = __half2float(beta[c]) - (float)mean * a;
    }
}

__global__ void gn_apply_kernel(const __half* __restrict__ x, const float* __restrict__ ab, __half* __restrict__ out,
                                long long rows_per_sample, long long total_rows, int C, int silu) {
    const int O = C / 8;
    const long long n = total_rows * O;
    const long long stride = (long long)gridDim.x * blockDim.x;
    auto apply = [&](long long i, const uint4& raw) {
        const long long row = i / O;
        const int oc = (int)(i % O);
        const long long sample = row / rows_per_sample;
        float f[8];
        unpack8(raw, f);
        const float4* abp = reinterpret_cast<const float4*>(ab + (sample * C + oc * 8) * 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 q = __ldg(abp + j);
            float y0 = fmaf(f[2 * j], q.x, q.y), y1 = fmaf(f[2 * j + 1], q.z, q.w);
            if (silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
            f[2 * j] = y0;
            f[2 * j + 1] = y1;
        }
        reinterpret_cast<uint4*>(out)[i] = pack8(f);
    };
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n; i += 4 * stride) {                      // 4 independent 16-byte loads in flight
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(x) + i + k * stride);
#pragma unroll
        for (int k = 0; k < 4; ++k) apply(i + k * stride, u[k]);
    }
    for (; i < n; i += stride) apply(i, __ldg(reinterpret_cast<const uint4*>(x) + i));
}

// ---- second generation (default): persistent CTAs over CONTIGUOUS runs of 128-row slabs -------------------------
// gn_stats / gn_apply above ran at 48 % of the copy bandwidth (kbench): a CTA lived for one 160 KB slab (launch +
// block reduction + atomics per slab), and gn_apply re-read its 16 (a, b) pairs (64 B from L1) for every 16 B of
// activations -- 115 B/clk/SM of L1 traffic at the HBM rate, i.e. L1-bound.  Here a CTA walks a contiguous range of
// slabs (slab = GN2_SLAB rows of ONE sample, so a range crosses a sample boundary rarely): statistics stay in
// registers until the sample changes, and the per-channel (a, b) live in registers and are reloaded only then.
constexpr int GN2_SLAB = 128;
constexpr int GN2_THREADS = 256;

struct Gn2Range {
    long long slabs_per_sample, total_slabs;
    __device__ void span(long long& g0, long long& g1) const {      // contiguous, balanced to +-1 slab
        const long long per = total_slabs / gridDim.x, extra = total_slabs % gridDim.x;
        g0 = per * blockIdx.x + (blockIdx.x < extra ? blockIdx.x : extra);
        g1 = g0 + per + (blockIdx.x < extra ? 1 : 0);
    }
};

__global__ void __launch_bounds__(GN2_THREADS)
gn_stats2_kernel(const __half* __restrict__ x, double* __restrict__ stats, long long rows_per_sample, int C, Gn2Range rg) {
    extern __shared__ float red[];            // [lanes][C][2]
    const int O = C / 8;                      // host guarantees O <= GN2_THREADS
    const int lanes = GN2_THREADS / O;
    const int tid = threadIdx.x;
    const int oc = tid % O, ln = tid / O;
    const bool active = ln < lanes;
    const int cg = C / 32;
    const int warp = tid >> 5, lane = tid & 31;
    long long g0, g1;
    rg.span(g0, g1);
    float s[8], ss[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = ss[j] = 0.f;
    long long cur = g0 < g1 ? g0 / rg.slabs_per_sample : -1;
    auto flush = [&](long long sample) {
        if (active) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                red[((size_t)ln * C + oc * 8 + j) * 2] = s[j];
                red[((size_t)ln * C + oc * 8 + j) * 2 + 1] = ss[j];
                s[j] = ss[j] = 0.f;
            }
        }
        __syncthreads();
        for (int g = warp; g < 32; g += GN2_THREADS / 32) {
            float a = 0.f, b = 0.f;
            for (int i = lane; i < lanes * cg; i += 32) {
                const int l2 = i / cg, c = g * cg + i % cg;
                a += red[((size_t)l2 * C + c) * 2];
                b += red[((size_t)l2 * C + c) * 2 + 1];
            }
            a = warp_sum(a);
            b = warp_sum(b);
            if (lane == 0) {
                atomicAdd(&stats[(sample * 32 + g) * 2], (double)a);
                atomicAdd(&stats[(sample * 32 + g) * 2 + 1], (double)b);
            }
        }
        __syncthreads();
    };
    for (long long g = g0; g < g1; ++g) {
        const long long sample = g / rg.slabs_per_sample;
        if (sample != cur) {                  // uniform across the CTA
            flush(cur);
            cur = sample;
        }
        const long long r0 = (g - sample * rg.slabs_per_sample) * GN2_SLAB;
        const long long r1 = min(rows_per_sample, r0 + GN2_SLAB);
        if (active) {
            const __half* xs = x + (sample * rows_per_sample) * C + oc * 8;
            long long r = r0 + ln;
            for (; r + 3ll * lanes < r1; r += 4ll * lanes) {          // 4 independent 16-byte loads in flight
                uint4 u[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xs + (r + (long long)k * lanes) * C));
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float f[8];
                    unpack8(u[k], f);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { s[j] += f[j]; ss[j] = fmaf(f[j], f[j], ss[j]); }
                }
            }
            for (; r < r1; r += lanes) {
                float f[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(xs + r * C)), f);
#pragma unroll
                for (int j = 0; j < 8; ++j) { s[j] += f[j]; ss[j] = fmaf(f[j], f[j], ss[j]); }
            }
        }
    }
    if (cur >= 0) flush(cur);
}

__global__ void __launch_bounds__(GN2_THREADS)
gn_apply2_kernel(const __half* __restrict__ x, const float* __restrict__ ab, __half* __restrict__ out,
                 long long rows_per_sample, int C, int silu, Gn2Range rg) {
    const int O = C / 8;
    const int lanes = GN2_THREADS / O;
    const int tid = threadIdx.x;
    const int oc = tid % O, ln = tid / O;
    if (ln >= lanes) return;
    long long g0, g1;
    rg.span(g0, g1);
    float a[8], b[8];
    long long cur = -1;
    auto apply = [&](const uint4& raw, __half* dst) {
        float f[8];
        unpack8(raw, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float y = fmaf(f[j], a[j], b[j]);
            if (silu) y = silu_f(y);
            f[j] = y;
        }
        *reinterpret_cast<uint4*>(dst) = pack8(f);
    };
    for (long long g = g0; g < g1; ++g) {
        const long long sample = g / rg.slabs_per_sample;
        if (sample != cur) {
            cur = sample;
            const float4* abp = reinterpret_cast<const float4*>(ab + (sample * C + oc * 8) * 2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 q = __ldg(abp + j);
                a[2 * j] = q.x; b[2 * j] = q.y; a[2 * j + 1] = q.z; b[2 * j + 1] = q.w;
            }
        }
        const long long r0 = (g - sample * rg.slabs_per_sample) * GN2_SLAB;
        const long long r1 = min(rows_per_sample, r0 + GN2_SLAB);
        const long long base = (sample * rows_per_sample) * C + oc * 8;
        long long r = r0 + ln;
        for (; r + 3ll * lanes < r1; r += 4ll * lanes) {
            uint4 u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(x + base + (r + (long long)k * lanes) * C));
#pragma unroll
            for (int k = 0; k < 4; ++k) apply(u[k], out + base + (r + (long long)k * lanes) * C);
        }
        for (; r < r1; r += lanes) apply(__ldg(reinterpret_cast<const uint4*>(x + base + r * C)), out + base + r * C);
    }
}

// apply over a pixel band: x holds frames of frame_rows rows (frames_per_sample of them share one sample's (a, b)); rows
// [p0, p0 + band) of every frame go compactly to out [frames * band, C].  Same per-element arithmetic as gn_apply2_kernel.
__global__ void gn_apply_band_kernel(const __half* __restrict__ x, const float* __restrict__ ab, __half* __restrict__ out,
                                     long long frames_per_sample, long long frame_rows, long long p0, long long band,
                                     long long frames, int C, int silu) {
    const int O = C / 8;
    const long long n = frames * band * O;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long orow = i / O;
        const int oc = (int)(i % O);
        const long long f = orow / band;
        const long long sample = f / frames_per_sample;
        float f8[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(x + (f * frame_rows + p0 + orow % band) * C + oc * 8)), f8);
        const float4* abp = reinterpret_cast<const float4*>(ab + (sample * C + oc * 8) * 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 q = __ldg(abp + j);
            float y0 = fmaf(f8[2 * j], q.x, q.y), y1 = fmaf(f8[2 * j + 1], q.z, q.w);
            if (silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
            f8[2 * j] = y0;
            f8[2 * j + 1] = y1;
        }
        reinterpret_cast<uint4*>(out)[i] = pack8(f8);
    }
}

// GroupNorm apply of the CogVideoX 3-D VAE's SpatialNorm3D (cp_enc_dec.py:451-510): y = GN(x) * Y[src] + B[src] (+ SiLU), where
// Y = conv_y(zq), B = conv_b(zq) are 1x1x1 convolutions of the latent and therefore commute with the nearest-neighbour
// interpolation of zq to the feature size: they are evaluated ONCE at latent resolution (Tl, Hl, Wl) and gathered per row.
// Row r = (t, h, w) of the (T, H, W) clip reads latent row (ts, hs, ws), each index F.interpolate(mode="nearest")'s:
// src = min(floor(dst * s), n_in - 1) with the fp32 scale s = n_in / n_out.  For a ratio whose fp32 reciprocal rounds low
// (41, 47, 55, 61, ...) that is one less than dst * n_in / n_out at some multiples of the ratio, so exact integer division
// would read the wrong latent row.  ts follows the reference's split of the first frame when T is odd (> 1): ts = 0 for t = 0,
// else 1 + the nearest index of t - 1 from Tl - 1 to T - 1 frames.  One sample (B = 1).
struct GnModGeom {
    int T, H, W, Tl, Hl, Wl, split_first;
    int hshift, wshift;       // log2(H / Hl), log2(W / Wl) when those ratios are powers of two (the VAE's: 1, 2, 4, 8), else -1
    float tscale, hscale, wscale;   // fp32 source / destination size ratios, computed on the host (T: of the split's rest)
};

// F.interpolate(mode="nearest")'s source index of destination index dst
STAR_DEVINL int nearest_src(int dst, float scale, int n_in) {
    return min((int)floorf(__fmul_rn((float)dst, scale)), n_in - 1);
}

__global__ void __launch_bounds__(GN2_THREADS)
gn_apply_mod_kernel(const __half* __restrict__ x, const float* __restrict__ ab, const __half* __restrict__ ymod,
                    const __half* __restrict__ bmod, long long ldmod, __half* __restrict__ out, long long rows, int C, int silu,
                    Gn2Range rg, GnModGeom gm) {
    const int O = C / 8;
    const int lanes = GN2_THREADS / O;
    const int tid = threadIdx.x;
    const int oc = tid % O, ln = tid / O;
    if (ln >= lanes) return;
    long long g0, g1;
    rg.span(g0, g1);
    float a[8], b[8];
    {
        const float4* abp = reinterpret_cast<const float4*>(ab + (oc * 8) * 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 q = __ldg(abp + j);
            a[2 * j] = q.x; b[2 * j] = q.y; a[2 * j + 1] = q.z; b[2 * j + 1] = q.w;
        }
    }
    const int H = gm.H, W = gm.W, HW = H * W;
    auto t_src = [&](int t) {
        if (gm.split_first) return t == 0 ? 0 : 1 + nearest_src(t - 1, gm.tscale, gm.Tl - 1);
        return nearest_src(t, gm.tscale, gm.Tl);
    };
    // one division set per slab, then (t, h, w) advance incrementally: the row index arithmetic must not outweigh 48 bytes of traffic
    for (long long g = g0; g < g1; ++g) {
        const int r0 = (int)(g * GN2_SLAB);
        const int r1 = (int)min(rows, (long long)r0 + GN2_SLAB);
        int r = r0 + ln;
        if (r >= r1) continue;
        int t = r / HW;
        int h = (r - t * HW) / W;
        int w = r - t * HW - h * W;
        int ts = t_src(t);
        while (r < r1) {
            uint4 ux[4], uy[4], ub[4];
            int rr[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                rr[k] = r < r1 ? r : -1;
                if (rr[k] >= 0) {
                    const int hs = gm.hshift >= 0 ? (h >> gm.hshift) : nearest_src(h, gm.hscale, gm.Hl);
                    const int ws = gm.wshift >= 0 ? (w >> gm.wshift) : nearest_src(w, gm.wscale, gm.Wl);
                    const long long src = ((long long)(ts * gm.Hl + hs) * gm.Wl + ws) * ldmod + oc * 8;
                    ux[k] = __ldg(reinterpret_cast<const uint4*>(x + (long long)r * C + oc * 8));
                    uy[k] = __ldg(reinterpret_cast<const uint4*>(ymod + src));
                    ub[k] = __ldg(reinterpret_cast<const uint4*>(bmod + src));
                    r += lanes;
                    w += lanes;
                    while (w >= W) {
                        w -= W;
                        if (++h == H) {
                            h = 0;
                            ts = t_src(++t);
                        }
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (rr[k] < 0) continue;
                float f[8], fy[8], fb[8];
                unpack8(ux[k], f);
                unpack8(uy[k], fy);
                unpack8(ub[k], fb);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float y = fmaf(fmaf(f[j], a[j], b[j]), fy[j], fb[j]);
                    if (silu) y = silu_f(y);
                    f[j] = y;
                }
                *reinterpret_cast<uint4*>(out + (long long)rr[k] * C + oc * 8) = pack8(f);
            }
        }
    }
}

// ------------------------------------------------------------------ LayerNorm over C with fused LIEM gate
// gate_mode 0: y = LN(x)
// gate_mode 1: y = LN(x * gate[row])            spatial LIEM, gate from liem_spatial_gate (unet_v2v.py:468-473)
// gate_mode 2: y = LN(x * sigmoid(w0*max_c(x) + w1*mean_c(x)))   temporal LIEM (unet_v2v.py:402-411, :481-487)
// One warp per row; the row lives in registers (C <= 1280 -> <= 5 x 8 values per lane).
constexpr int LN_MAX_OCT = 5;
// Persistent warps (grid-stride over rows) with the NEXT row of the warp prefetched as packed 16-byte registers;
// register use is kept low (launch bounds) so that ~50 warps/SM x 2 rows are in flight (HBM latency hiding).
template <int LN_OCT>          // 16-byte column groups per lane: 2 (C <= 512), 3 (C <= 768), 5 (C <= 1280)
__global__ void __launch_bounds__(256, LN_OCT <= 2 ? 5 : (LN_OCT == 3 ? 4 : (LN_OCT <= 5 ? 2 : 1)))
layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ gamma, const __half* __restrict__ beta,
                 __half* __restrict__ out, long long rows, int C, float eps, int gate_mode,
                 const __half* __restrict__ gate, float w0, float w1) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int O = C / 8;
    const float inv_c = 1.0f / (float)C;
    uint4 nxt[LN_OCT];
#pragma unroll
    for (int i = 0; i < LN_OCT; ++i) {
        const int oc = lane + 32 * i;
        if (oc < O) nxt[i] = __ldg(reinterpret_cast<const uint4*>(x + row * C + oc * 8));
    }
    for (; row < rows; row += nwarps) {
        float v[LN_OCT][8];
        float s = 0.f, mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < LN_OCT; ++i) {
            const int oc = lane + 32 * i;
            if (oc < O) {
                unpack8(nxt[i], v[i]);
#pragma unroll
                for (int j = 0; j < 8; ++j) { s += v[i][j]; mx = fmaxf(mx, v[i][j]); }
            }
        }
        const long long nrow = row + nwarps;
        if (nrow < rows) {                              // prefetch the next row of this warp
#pragma unroll
            for (int i = 0; i < LN_OCT; ++i) {
                const int oc = lane + 32 * i;
                if (oc < O) nxt[i] = __ldg(reinterpret_cast<const uint4*>(x + nrow * C + oc * 8));
            }
        }
        if (gate_mode != 0) {
            float g;
            if (gate_mode == 1) {
                g = __half2float(gate[row]);
            } else {
                s = warp_sum(s);
                mx = warp_max(mx);
                // reference computes max / mean / Linear(2->1) / sigmoid in fp16 (autocast keeps input dtype)
                const float mean_h = __half2float(__float2half_rn(s * inv_c));
                const float lin = __half2float(__float2half_rn(w0 * mx + w1 * mean_h));
                g = __half2float(__float2half_rn(sigmoid_f(lin)));
            }
            s = 0.f;
#pragma unroll
            for (int i = 0; i < LN_OCT; ++i) {
                const int oc = lane + 32 * i;
                if (oc < O) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        v[i][j] = __half2float(__float2half_rn(v[i][j] * g));     // fp16 product, as the reference
                        s += v[i][j];
                    }
                }
            }
        }
        const float mean = warp_sum(s) * inv_c;
        float var = 0.f;
#pragma unroll
        for (int i = 0; i < LN_OCT; ++i) {
            const int oc = lane + 32 * i;
            if (oc < O) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; var = fmaf(d, d, var); }
            }
        }
        const float rstd = rsqrtf(warp_sum(var) * inv_c + eps);
#pragma unroll
        for (int i = 0; i < LN_OCT; ++i) {
            const int oc = lane + 32 * i;
            if (oc < O) {
                float gm[8], bt[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + oc * 8)), gm);
                unpack8(__ldg(reinterpret_cast<const uint4*>(beta + oc * 8)), bt);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[i][j] = (v[i][j] - mean) * rstd * gm[j] + bt[j];
                *reinterpret_cast<uint4*>(out + row * C + oc * 8) = pack8(v[i]);
            }
        }
    }
}

// Narrow rows: C = 40 * LPR channels (320 -> LPR 8, 640 -> LPR 16).  A warp normalises 32 / LPR rows at once, LPR lanes
// x 5 sixteen-byte groups per row, every lane busy (layernorm_kernel<2> keeps only 20 of 32 lanes busy at C = 320 and
// spends a full 5-step shuffle tree per row: ~150 instructions per row against ~80 here).  Same arithmetic and gate modes as layernorm_kernel.
template <int LPR>
__global__ void __launch_bounds__(256, 2)
layernorm_sub_kernel(const __half* __restrict__ x, const __half* __restrict__ gamma, const __half* __restrict__ beta,
                     __half* __restrict__ out, long long rows, float eps, int gate_mode, const __half* __restrict__ gate,
                     float w0, float w1) {
    constexpr int RPW = 32 / LPR;             // rows per warp and iteration
    constexpr int C = 40 * LPR;
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPR, sl = lane % LPR;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long ngroups = (rows + RPW - 1) / RPW;
    long long grp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (grp >= ngroups) return;
    const float inv_c = 1.0f / (float)C;
    auto sub_sum = [](float v) {
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    auto sub_max = [](float v) {
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        return v;
    };
    uint4 nxt[5];
    {
        const long long row = grp * RPW + sub;
#pragma unroll
        for (int i = 0; i < 5; ++i)
            nxt[i] = row < rows ? __ldg(reinterpret_cast<const uint4*>(x + row * C + (sl + LPR * i) * 8)) : make_uint4(0, 0, 0, 0);
    }
    for (; grp < ngroups; grp += nwarps) {
        const long long row = grp * RPW + sub;
        const bool valid = row < rows;
        float v[5][8];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            unpack8(nxt[i], v[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) s += v[i][j];
        }
        const long long nrow = (grp + nwarps) * RPW + sub;
        if (grp + nwarps < ngroups) {                   // prefetch this lane's share of the warp's next row group
#pragma unroll
            for (int i = 0; i < 5; ++i)
                nxt[i] = nrow < rows ? __ldg(reinterpret_cast<const uint4*>(x + nrow * C + (sl + LPR * i) * 8)) : make_uint4(0, 0, 0, 0);
        }
        if (gate_mode != 0) {
            float g;
            if (gate_mode == 1) {
                g = valid ? __half2float(gate[row]) : 0.f;
            } else {
                float mx = -INFINITY;
#pragma unroll
                for (int i = 0; i < 5; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[i][j]);
                s = sub_sum(s);
                mx = sub_max(mx);
                const float mean_h = __half2float(__float2half_rn(s * inv_c));
                const float lin = __half2float(__float2half_rn(w0 * mx + w1 * mean_h));
                g = __half2float(__float2half_rn(sigmoid_f(lin)));
            }
            s = 0.f;
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    v[i][j] = __half2float(__float2half_rn(v[i][j] * g));     // fp16 product, as the reference
                    s += v[i][j];
                }
        }
        const float mean = sub_sum(s) * inv_c;
        float var = 0.f;
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; var = fmaf(d, d, var); }
        const float rstd = rsqrtf(sub_sum(var) * inv_c + eps);
        if (valid) {
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                const int oc = sl + LPR * i;
                float gm[8], bt[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + oc * 8)), gm);
                unpack8(__ldg(reinterpret_cast<const uint4*>(beta + oc * 8)), bt);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[i][j] = (v[i][j] - mean) * rstd * gm[j] + bt[j];
                *reinterpret_cast<uint4*>(out + row * C + oc * 8) = pack8(v[i]);
            }
        }
    }
}

// ------------------------------------------------------------------ spatial LIEM gate (unet_v2v.py:380-394)
// step 1: per token channel-max and channel-mean -> mm[R][2] fp16
__global__ void __launch_bounds__(256)
liem_reduce_kernel(const __half* __restrict__ x, __half* __restrict__ mm, long long rows, int C) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const int O = C / 8;
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nwarps) {
        float s = 0.f, mx = -INFINITY;
        for (int oc = lane; oc < O; oc += 32) {
            float f[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + oc * 8)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) { s += f[j]; mx = fmaxf(mx, f[j]); }
        }
        s = warp_sum(s);
        mx = warp_max(mx);
        if (lane == 0) {
            __half2 h = __floats2half2_rn(mx, s / (float)C);
            *reinterpret_cast<__half2*>(mm + row * 2) = h;
        }
    }
}
// step 2: 7x7 conv (2 -> 1, pad 3, no bias) + sigmoid -> gate[R] fp16.  wt = conv1.weight[0] as [2][7][7]
// The gate of token i of the mm map [BT, H, W][2]; w_s = wt in fp32.
__device__ __forceinline__ __half liem_conv7_gate(const __half* __restrict__ mm, const float* w_s, long long i, int H, int W) {
    const int w0 = (int)(i % W), h0 = (int)((i / W) % H);
    const long long bt = i / ((long long)W * H);
    float acc = 0.f;
    for (int r = 0; r < 7; ++r) {
        const int hh = h0 + r - 3;
        if (hh < 0 || hh >= H) continue;
        for (int s = 0; s < 7; ++s) {
            const int ww = w0 + s - 3;
            if (ww < 0 || ww >= W) continue;
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(mm + ((bt * H + hh) * W + ww) * 2));
            acc = fmaf(v.x, w_s[r * 7 + s], acc);
            acc = fmaf(v.y, w_s[49 + r * 7 + s], acc);
        }
    }
    const float a = __half2float(__float2half_rn(acc));      // fp16 conv output in the reference
    return __float2half_rn(sigmoid_f(a));
}

__global__ void liem_conv7_kernel(const __half* __restrict__ mm, const __half* __restrict__ wt, __half* __restrict__ gate,
                                  int BT, int H, int W) {
    __shared__ float w_s[98];
    if (threadIdx.x < 98) w_s[threadIdx.x] = __half2float(wt[threadIdx.x]);
    __syncthreads();
    const long long n = (long long)BT * H * W;
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    gate[i] = liem_conv7_gate(mm, w_s, i, H, W);
}

// The same gates for tokens [r0, r0 + n) of the map only (gate[0..n)): a rank of a token-sharded DiT holds the whole
// map but gates only its own tokens.
__global__ void liem_conv7_rows_kernel(const __half* __restrict__ mm, const __half* __restrict__ wt, __half* __restrict__ gate,
                                       int H, int W, long long r0, long long n) {
    __shared__ float w_s[98];
    if (threadIdx.x < 98) w_s[threadIdx.x] = __half2float(wt[threadIdx.x]);
    __syncthreads();
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    gate[i] = liem_conv7_gate(mm, w_s, r0 + i, H, W);
}

// ------------------------------------------------------------------ CogVideoX DiT helpers (cogvideox-based/sat/dit_video_concat.py)
// out = x * g(row): mode 1 external per-row gate (spatial LIEM, :523-527); mode 2 temporal LIEM gate
// sigmoid(w0*max_c + w1*mean_c) computed in-kernel (:529-531).  Any C that is a multiple of 8.
__global__ void __launch_bounds__(256)
row_gate_kernel(const __half* __restrict__ x, __half* __restrict__ out, long long rows, int C, int mode,
                const __half* __restrict__ gate, float w0, float w1) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const int O = C / 8;
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nwarps) {
        float g;
        if (mode == 1) {
            g = __half2float(gate[row]);
        } else {
            float s = 0.f, mx = -INFINITY;
            for (int oc = lane; oc < O; oc += 32) {
                float f[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + oc * 8)), f);
#pragma unroll
                for (int j = 0; j < 8; ++j) { s += f[j]; mx = fmaxf(mx, f[j]); }
            }
            s = warp_sum(s);
            mx = warp_max(mx);
            const float mean_h = __half2float(__float2half_rn(s / (float)C));
            const float lin = __half2float(__float2half_rn(w0 * mx + w1 * mean_h));
            g = __half2float(__float2half_rn(sigmoid_f(lin)));
        }
        for (int oc = lane; oc < O; oc += 32) {
            float f[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + oc * 8)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] *= g;
            *reinterpret_cast<uint4*>(out + row * C + oc * 8) = pack8(f);
        }
    }
}

// In-place per-head LayerNorm(64) of q and k (:583-587) followed by the 3-D rotary embedding of the image tokens
// (:306-333; interleaved pairs (x1, x2) -> (x1 cos - x2 sin, x2 cos + x1 sin)).  qkv [rows, ld]; q at column 0,
// k at column `koff`; 8 lanes per (row, head, q|k), 8 elements per lane.  cos/sin: fp32 [n_img, 64].
__global__ void __launch_bounds__(256)
qk_ln_rope_kernel(__half* __restrict__ qkv, long long ld, long long rows, int heads, int koff,
                  const __half* __restrict__ qg, const __half* __restrict__ qb, const __half* __restrict__ kg,
                  const __half* __restrict__ kb, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                  int seq, int text_len, float eps) {
    const long long ngroups = rows * heads * 2;
    const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int sub = threadIdx.x & 7;
    if (gid >= ngroups) return;
    const int which = (int)(gid & 1);                     // 0 = q, 1 = k
    const int head = (int)((gid >> 1) % heads);
    const long long row = (gid >> 1) / heads;
    __half* ptr = qkv + row * ld + (which ? koff : 0) + head * 64 + sub * 8;
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(ptr), f);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    const float mean = s * (1.f / 64.f);
    float var = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; var = fmaf(d, d, var); }
    var += __shfl_xor_sync(0xffffffffu, var, 1);
    var += __shfl_xor_sync(0xffffffffu, var, 2);
    var += __shfl_xor_sync(0xffffffffu, var, 4);
    const float rstd = rsqrtf(var * (1.f / 64.f) + eps);
    float gm[8], bt[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>((which ? kg : qg) + sub * 8)), gm);
    unpack8(__ldg(reinterpret_cast<const uint4*>((which ? kb : qb) + sub * 8)), bt);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __half2float(__float2half_rn((f[j] - mean) * rstd * gm[j] + bt[j]));   // LN output is fp16/bf16 in the reference
    const int tok = (int)(row % seq);
    if (tok >= text_len) {
        const float* c = cos_t + (long long)(tok - text_len) * 64 + sub * 8;
        const float* sn = sin_t + (long long)(tok - text_len) * 64 + sub * 8;
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            const float x1 = f[j], x2 = f[j + 1];
            f[j] = x1 * c[j] - x2 * sn[j];
            f[j + 1] = x2 * c[j + 1] + x1 * sn[j + 1];
        }
    }
    *reinterpret_cast<uint4*>(ptr) = pack8(f);
}

// ------------------------------------------------------------------ elementwise / copies
// out[R, Ca+Cb] = [ a | b (+ c) ]        decoder skip concat with the control residual (unet_v2v.py:1792)
__global__ void concat_add_kernel(const __half* __restrict__ a, int Ca, const __half* __restrict__ b,
                                  const __half* __restrict__ c, int Cb, __half* __restrict__ out, long long rows) {
    const int Oa = Ca / 8, Ob = Cb / 8, O = Oa + Ob;
    const long long n = rows * O;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / O;
        const int oc = (int)(i % O);
        uint4 v;
        if (oc < Oa) {
            v = __ldg(reinterpret_cast<const uint4*>(a + row * Ca + oc * 8));
        } else {
            v = __ldg(reinterpret_cast<const uint4*>(b + row * Cb + (oc - Oa) * 8));
            if (c) {
                float f[8], g[8];
                unpack8(v, f);
                unpack8(__ldg(reinterpret_cast<const uint4*>(c + row * Cb + (oc - Oa) * 8)), g);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] += g[j];
                v = pack8(f);
            }
        }
        *reinterpret_cast<uint4*>(out + row * (long long)(Ca + Cb) + oc * 8) = v;
    }
}
// out = a + b (fp16), n8 = number of 8-element groups
__global__ void add_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ out,
                           long long n8) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        float f[8], g[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(a) + i), f);
        unpack8(__ldg(reinterpret_cast<const uint4*>(b) + i), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += g[j];
        reinterpret_cast<uint4*>(out)[i] = pack8(f);
    }
}
// temporal half of DownSample3D of the CogVideoX 3-D VAE encoder (cp_enc_dec.py:581-596): avg_pool1d(k = 2, s = 2) over the frames
// of a [(T HW), C] clip; for odd T the first frame is kept and the remaining T - 1 are pooled.  per8 = HW * C / 8.
__global__ void time_avgpool2_kernel(const __half* __restrict__ x, __half* __restrict__ out, int T, long long per8) {
    const int odd = T & 1;
    const int To = odd ? (T + 1) / 2 : T / 2;
    const long long n = (long long)To * per8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int to = (int)(i / per8);
        const long long off = i - (long long)to * per8;
        if (odd && to == 0) {
            reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(x) + off);
            continue;
        }
        const long long t0 = odd ? 2 * to - 1 : 2 * to;
        float f[8], g[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(x) + t0 * per8 + off), f);
        unpack8(__ldg(reinterpret_cast<const uint4*>(x) + (t0 + 1) * per8 + off), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = 0.5f * (f[j] + g[j]);
        reinterpret_cast<uint4*>(out)[i] = pack8(f);
    }
}
// nearest x2 upsample then drop the first and last row (unet_v2v.py:563-564): out H' = 2H-2, W' = 2W
// crop = 0: plain nearest x2 (the VAE decoder's Upsample2D), out H' = 2H
__global__ void upsample2x_crop_kernel(const __half* __restrict__ x, __half* __restrict__ out, int BT, int H, int W,
                                       int C, int crop) {
    const int O = C / 8, Ho = 2 * H - 2 * crop, Wo = 2 * W;
    const long long n = (long long)BT * Ho * Wo * O;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int oc = (int)(i % O);
        long long t = i / O;
        const int ow = (int)(t % Wo); t /= Wo;
        const int oh = (int)(t % Ho);
        const long long bt = t / Ho;
        const int ih = (oh + crop) >> 1, iw = ow >> 1;
        reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(x + ((bt * H + ih) * W + iw) * C + oc * 8));
    }
}
// stride-2 conv input split (unet_v2v.py:709: stride 2, padding (2,1)):
// planes[bt][pq][i][j][:] = Xpad[2i + p][2j + q],  Xpad = X zero-padded by 2 rows / 1 column on each side,
// pq = 2p + q, plane extent (Ho+1, Wo+1) with Ho = (H+1)/2 + 1... computed by the host.
// pad_t / pad_l: zero rows / columns in front (2, 1 for the UNet; 0, 0 for the VAE encoder's pad (0,1,0,1)).
__global__ void s2_split_kernel(const __half* __restrict__ x, __half* __restrict__ planes, int BT, int H, int W, int C,
                                int H2, int W2, int pad_t, int pad_l) {
    const int O = C / 8;
    const long long n = (long long)BT * 4 * H2 * W2 * O;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int oc = (int)(idx % O);
        long long t = idx / O;
        const int j = (int)(t % W2); t /= W2;
        const int i = (int)(t % H2); t /= H2;
        const int pq = (int)(t % 4);
        const long long bt = t / 4;
        const int ih = 2 * i + (pq >> 1) - pad_t, iw = 2 * j + (pq & 1) - pad_l;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (ih >= 0 && ih < H && iw >= 0 && iw < W)
            v = __ldg(reinterpret_cast<const uint4*>(x + ((bt * H + ih) * W + iw) * C + oc * 8));
        reinterpret_cast<uint4*>(planes)[idx] = v;
    }
}
// ------------------------------------------------------------------ single-head attention pieces (VAE mid block)
// In-place softmax over the first `cols` entries of each row of S[rows, ld] (fp16 logits, already scaled), statistics in
// fp32.  Columns cols..ld-1 are zeroed.  Each row is handled by one cluster of n CTAs (grid rows * n): CTA r stages columns
// [r seg, (r + 1) seg) of the row (seg a multiple of 8; a segment may be short or empty) in its shared memory, so every
// logit is read once and written once.  The CTAs' maxima and then their exp-sums are exchanged through distributed shared
// memory and combined in rank order; with n = 1 both combines are exact and the kernel computes what a one-CTA-per-row
// kernel does.
constexpr int SOFTMAX_SEG_MAX = 102400;     // columns one CTA stages: 200 KiB of fp16
__global__ void __launch_bounds__(256)
softmax_rows_kernel(__half* __restrict__ S, long long ld, int cols, int seg) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    __half* row_s = reinterpret_cast<__half*>(sm_raw);
    __shared__ float red[8];
    __shared__ float stat[2];                  // this CTA's max and exp-sum, read by the whole cluster
    const uint32_t rank = cluster_ctarank(), n = cluster_nctarank();
    const int c0 = (int)rank * seg;
    const int len = max(0, min(cols - c0, seg));
    __half* row = S + (long long)(blockIdx.x / n) * ld;
    __half* sg = row + min(c0, cols);          // this CTA's segment
    const int tid = threadIdx.x, nv = len / 8;
    float mx = -INFINITY;
    for (int i = tid; i < nv; i += 256) {
        const uint4 u = reinterpret_cast<const uint4*>(sg)[i];
        reinterpret_cast<uint4*>(row_s)[i] = u;
        float f[8];
        unpack8(u, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) mx = fmaxf(mx, f[j]);
    }
    for (int i = nv * 8 + tid; i < len; i += 256) {
        const __half h = sg[i];
        row_s[i] = h;
        mx = fmaxf(mx, __half2float(h));
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    if (tid == 0) stat[0] = mx;
    cluster_arrive();                          // also orders this CTA's reads of red before its rewrite below
    cluster_wait();
    mx = -INFINITY;
    for (uint32_t r = 0; r < n; ++r) mx = fmaxf(mx, ld_dsmem_f32(&stat[0], r));
    float sum = 0.f;
    for (int i = tid; i < len; i += 256) sum += __expf(__half2float(row_s[i]) - mx);
    sum = warp_sum(sum);
    if ((tid & 31) == 0) red[tid >> 5] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += red[w];
    if (tid == 0) stat[1] = sum;
    cluster_arrive();
    cluster_wait();
    sum = 0.f;
    for (uint32_t r = 0; r < n; ++r) sum += ld_dsmem_f32(&stat[1], r);
    cluster_arrive();                          // this CTA reads no peer's shared memory from here on
    const float inv = 1.f / sum;
    for (int i = tid; i < nv; i += 256) {
        float f[8];
        unpack8(reinterpret_cast<const uint4*>(row_s)[i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = __expf(f[j] - mx) * inv;
        reinterpret_cast<uint4*>(sg)[i] = pack8(f);
    }
    for (int i = nv * 8 + tid; i < len; i += 256) sg[i] = __float2half_rn(__expf(__half2float(row_s[i]) - mx) * inv);
    if (rank + 1 == n)
        for (long long i = cols + tid; i < ld; i += 256) row[i] = __float2half_rn(0.f);
    cluster_wait();                            // no CTA exits while a peer may still read its stat
}

// ------------------------------------------------------------------ VAE decoder head
// time_conv_out: Conv3d(3 -> 3, kernel (3,1,1), padding (1,0,0)) over the frames of x[(b t hw), ldx] (3 valid
// channels) fused with the tokens -> (b t) c h w conversion; w[co][ci][dt], fp16 output.
__global__ void vae_head_kernel(const __half* __restrict__ x, long long ldx, const __half* __restrict__ w16,
                                const __half* __restrict__ bias16, __half* __restrict__ out, int B, int T, long long HW) {
    float w[27], bias[3];
#pragma unroll
    for (int k = 0; k < 27; ++k) w[k] = __half2float(w16[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) bias[k] = bias16 ? __half2float(bias16[k]) : 0.f;
    const long long n = (long long)B * T * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long hw = i % HW;
        const long long bt = i / HW;
        const int t = (int)(bt % T);
        float acc[3] = {bias[0], bias[1], bias[2]};
#pragma unroll
        for (int dt = 0; dt < 3; ++dt) {
            const int tt = t + dt - 1;
            if (tt < 0 || tt >= T) continue;
            const __half* xr = x + (i + (long long)(dt - 1) * HW) * ldx;
            const float x0 = __half2float(xr[0]), x1 = __half2float(xr[1]), x2 = __half2float(xr[2]);
#pragma unroll
            for (int co = 0; co < 3; ++co)
                acc[co] += w[(co * 3 + 0) * 3 + dt] * x0 + w[(co * 3 + 1) * 3 + dt] * x1 + w[(co * 3 + 2) * 3 + dt] * x2;
        }
#pragma unroll
        for (int co = 0; co < 3; ++co) out[(bt * 3 + co) * HW + hw] = __float2half_rn(acc[co]);
    }
}

// sinusoidal timestep embedding cos || sin (unet_v2v.py:96-108) -> fp16 [B, dim]
__global__ void sinusoidal_kernel(const long long* __restrict__ t, __half* __restrict__ out, int B, int dim) {
    const int half_d = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half_d) return;
    const int b = i / half_d, k = i % half_d;
    const float freq = powf(10000.f, -(float)k / (float)half_d);
    const float a = (float)t[b] * freq;
    out[b * dim + k] = __float2half_rn(cosf(a));
    out[b * dim + half_d + k] = __float2half_rn(sinf(a));
}
__global__ void silu_kernel(const __half* __restrict__ x, __half* __restrict__ out, long long n) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i < n) out[i] = __float2half_rn(silu_f(__half2float(x[i])));
}


// ------------------------------------------------------------------ pre-processing (video_to_video_model.py:81-87)
// F.interpolate(x, [H, W], mode='bilinear') (align_corners = False) followed by F.pad(..., (pl, pr, pt, pb), value):
// x (NC, h, w) fp32 -> out (NC, H + pt + pb, W + pl + pr) fp32.  One thread per output pixel, x fastest.
__global__ void __launch_bounds__(256)
bilinear_pad_kernel(const float* __restrict__ x, float* __restrict__ out, long long NC, int h, int w, int H, int W, int pl,
                    int pt, int Hp, int Wp, float sh, float sw, float padv) {
    const long long total = NC * Hp * Wp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wp);
        const int oy = (int)((i / Wp) % Hp);
        const long long nc = i / ((long long)Wp * Hp);
        const int dx = ox - pl, dy = oy - pt;
        float v = padv;
        if (dx >= 0 && dx < W && dy >= 0 && dy < H) {
            const float fy = fmaxf(__fmaf_rn((float)dy + 0.5f, sh, -0.5f), 0.f);
            const float fx = fmaxf(__fmaf_rn((float)dx + 0.5f, sw, -0.5f), 0.f);
            const int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
            const int y1 = y0 + (y0 < h - 1), x1 = x0 + (x0 < w - 1);
            const float ly = fy - (float)y0, lx = fx - (float)x0;
            const float hy = 1.f - ly, hx = 1.f - lx;
            const float* p = x + nc * (long long)h * w;
            v = hy * (hx * __ldg(p + (long long)y0 * w + x0) + lx * __ldg(p + (long long)y0 * w + x1)) +
                ly * (hx * __ldg(p + (long long)y1 * w + x0) + lx * __ldg(p + (long long)y1 * w + x1));
        }
        out[i] = v;
    }
}

// ------------------------------------------------------------------ post-processing (inference_utils.py:16-23, color_fix.py:15-74)
// tensor2vid + adain_color_fix on the GPU: per (frame, channel) the SR frame t = clamp((x + 1) / 2, 0, 1) is re-normalised to the
// mean / std of the LR frame s = (src + 1) / 2 (unbiased variance + 1e-5, like calc_mean_std) and written as (T, H, W, C) * 255.
// Stage 1: sum / sum of squares of one tensor's planes into stats[plane][2] (double atomics); `clamp01` applies tensor2vid's clamp.
__global__ void __launch_bounds__(256)
plane_stats_kernel(const float* __restrict__ x, long long plane_elems, int clamp01, double* __restrict__ stats) {
    const float* p = x + (long long)blockIdx.y * plane_elems;
    float s = 0.f, ss = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < plane_elems; i += (long long)gridDim.x * blockDim.x) {
        float v = __fmaf_rn(p[i], 0.5f, 0.5f);
        if (clamp01) v = fminf(fmaxf(v, 0.f), 1.f);
        s += v;
        ss = fmaf(v, v, ss);
    }
    s = warp_sum(s);
    ss = warp_sum(ss);
    __shared__ float red[2][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][warp] = s; red[1][warp] = ss; }
    __syncthreads();
    if (threadIdx.x < 2) {
        double acc = 0.0;
        for (int k = 0; k < 8; ++k) acc += (double)red[threadIdx.x][k];
        atomicAdd(&stats[blockIdx.y * 2 + threadIdx.x], acc);
    }
}

// Stage 2: video (C, F, H*W) fp32 in [-1, 1] -> out (F, H*W, C) fp32 in [0, 255] (or uint8 when out_u8 != nullptr).
// tgt_stats planes are ordered (c, f) like the video, src_stats planes (f, c) like the LR clip (F, C, h, w).
__global__ void __launch_bounds__(256)
adain_apply_kernel(const float* __restrict__ video, float* __restrict__ out_f32, unsigned char* __restrict__ out_u8, int C, int F,
                   long long HW, long long src_hw, const double* __restrict__ tgt_stats, const double* __restrict__ src_stats) {
    const int f = blockIdx.y;
    float scale[4], shift[4];
    for (int c = 0; c < C && c < 4; ++c) {
        const double nt = (double)HW, ns = (double)src_hw;
        const double tm = tgt_stats[(c * F + f) * 2] / nt, sm = src_stats[(f * C + c) * 2] / ns;
        const double tv = (tgt_stats[(c * F + f) * 2 + 1] - nt * tm * tm) / (nt - 1.0) + 1e-5;
        const double sv = (src_stats[(f * C + c) * 2 + 1] - ns * sm * sm) / (ns - 1.0) + 1e-5;
        const double k = sqrt(sv > 0 ? sv : 0.0) / sqrt(tv);
        scale[c] = (float)k;
        shift[c] = (float)(sm - tm * k);
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
        for (int c = 0; c < C && c < 4; ++c) {
            float v = __fmaf_rn(video[((long long)c * F + f) * HW + i], 0.5f, 0.5f);
            v = fminf(fmaxf(v, 0.f), 1.f);
            v = fminf(fmaxf(fmaf(v, scale[c], shift[c]), 0.f), 1.f) * 255.f;
            const long long o = ((long long)f * HW + i) * C + c;
            if (out_u8) out_u8[o] = (unsigned char)__float2int_rn(v);
            else out_f32[o] = v;
        }
    }
}

// ------------------------------------------------------------------ guided x0 (diffusion_sdedit.py:89-99)
// out = u + g (y - u) in fp16 (each op rounded like the reference's fp16 tensor ops), std-ratio rescale
// out *= r * std(y) / (std(out) + 1e-12) + (1 - r) with per-sample (unbiased) std over the whole chunk, then
// x0 = alpha * xt - sigma * out in fp32.  Two launches: statistics (double atomics into stats[sample][4]), apply.
STAR_DEVINL float cfg_combine_h(__half y, __half u, float g) {
    const float d = __half2float(__float2half_rn(__half2float(y) - __half2float(u)));
    const float gd = __half2float(__float2half_rn(g * d));
    return __half2float(__float2half_rn(__half2float(u) + gd));
}

__global__ void __launch_bounds__(256)
cfg_stats_kernel(const __half* __restrict__ y, const __half* __restrict__ u, float g, long long per_sample,
                 double* __restrict__ stats) {
    const int sample = blockIdx.y;
    const __half* ys = y + sample * per_sample;
    const __half* us = u + sample * per_sample;
    float sy = 0.f, syy = 0.f, so = 0.f, soo = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per_sample; i += (long long)gridDim.x * blockDim.x) {
        const float yv = __half2float(ys[i]);
        const float ov = cfg_combine_h(ys[i], us[i], g);
        sy += yv; syy += yv * yv; so += ov; soo += ov * ov;
    }
    __shared__ float red[4][8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        syy += __shfl_xor_sync(0xffffffffu, syy, o);
        so += __shfl_xor_sync(0xffffffffu, so, o);
        soo += __shfl_xor_sync(0xffffffffu, soo, o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][warp] = sy; red[1][warp] = syy; red[2][warp] = so; red[3][warp] = soo; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double acc = 0.0;
        for (int k = 0; k < 8; ++k) acc += (double)red[threadIdx.x][k];
        atomicAdd(&stats[sample * 4 + threadIdx.x], acc);
    }
}

__global__ void __launch_bounds__(256)
cfg_x0_kernel(const __half* __restrict__ y, const __half* __restrict__ u, const float* __restrict__ xt,
              float* __restrict__ x0, __half* __restrict__ out_g, float g, float r, int has_rescale,
              const float* __restrict__ alpha, const float* __restrict__ sigma, long long per_sample,
              const double* __restrict__ stats) {
    const int sample = blockIdx.y;
    float scale = 1.f;
    if (has_rescale) {
        const double n = (double)per_sample;
        const double vy = (stats[sample * 4 + 1] - stats[sample * 4 + 0] * stats[sample * 4 + 0] / n) / (n - 1.0);
        const double vo = (stats[sample * 4 + 3] - stats[sample * 4 + 2] * stats[sample * 4 + 2] / n) / (n - 1.0);
        const float sdy = __half2float(__float2half_rn((float)sqrt(vy > 0.0 ? vy : 0.0)));       // tensor.std() in fp16
        const float sdo = __half2float(__float2half_rn((float)sqrt(vo > 0.0 ? vo : 0.0)));
        const float ratio = __half2float(__float2half_rn(__fdiv_rn(sdy, __half2float(__float2half_rn(sdo + 1e-12f)))));
        const float a = __half2float(__float2half_rn(r * ratio));
        scale = __half2float(__float2half_rn(a + (1.f - r)));
    }
    const float al = alpha[sample], sg = sigma[sample];
    const long long base = sample * per_sample;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per_sample; i += (long long)gridDim.x * blockDim.x) {
        float o = cfg_combine_h(y[base + i], u[base + i], g);
        if (has_rescale) o = __half2float(__float2half_rn(o * scale));
        if (out_g) out_g[base + i] = __float2half_rn(o);
        x0[base + i] = __fsub_rn(__fmul_rn(al, xt[base + i]), __fmul_rn(sg, o));
    }
}

// Spatially tiled sampling: the same guided x0 for one (chunk, tile) model call, accumulated into the clip-level x0 with the
// tile's separable blend weights: acc[b, c, f0 + f, r0 + i, c0 + j] += wy[i] * wx[j] * x0 for the kept frames lo <= f < hi.
// y / u: [samples][C][Ft][th][tw] (the tile), xt / acc: [samples][C][F][H][W] (the clip), read and written in place.
// Element order and rounding of x0 are cfg_x0_kernel's, so a unit weight into a zeroed acc reproduces it bit for bit.
struct CfgBlendGeom {
    int C, Ft, th, tw, lo, hi;                  // tile extents and kept frame range (tile-local)
    long long F, H, W, f0, r0, c0;              // clip extents and the tile's window offset
};

__global__ void __launch_bounds__(256)
cfg_x0_blend_kernel(const __half* __restrict__ y, const __half* __restrict__ u, const float* __restrict__ xt,
                    float* __restrict__ acc, float g, float r, int has_rescale, const float* __restrict__ alpha,
                    const float* __restrict__ sigma, const float* __restrict__ wy, const float* __restrict__ wx,
                    CfgBlendGeom q, const double* __restrict__ stats) {
    const int sample = blockIdx.y;
    const unsigned per_sample = (unsigned)q.C * q.Ft * q.th * q.tw;
    float scale = 1.f;
    if (has_rescale) {
        const double n = (double)per_sample;
        const double vy = (stats[sample * 4 + 1] - stats[sample * 4 + 0] * stats[sample * 4 + 0] / n) / (n - 1.0);
        const double vo = (stats[sample * 4 + 3] - stats[sample * 4 + 2] * stats[sample * 4 + 2] / n) / (n - 1.0);
        const float sdy = __half2float(__float2half_rn((float)sqrt(vy > 0.0 ? vy : 0.0)));
        const float sdo = __half2float(__float2half_rn((float)sqrt(vo > 0.0 ? vo : 0.0)));
        const float ratio = __half2float(__float2half_rn(__fdiv_rn(sdy, __half2float(__float2half_rn(sdo + 1e-12f)))));
        const float a = __half2float(__float2half_rn(r * ratio));
        scale = __half2float(__float2half_rn(a + (1.f - r)));
    }
    const float al = alpha[sample], sg = sigma[sample];
    const unsigned nf = (unsigned)(q.hi - q.lo), plane = (unsigned)q.th * q.tw;
    const unsigned kept = (unsigned)q.C * nf * plane;
    const long long tile_base = (long long)sample * per_sample;
    for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < kept; k += gridDim.x * blockDim.x) {
        const unsigned j = k % q.tw, ij = k / q.tw;
        const unsigned i = ij % q.th, cf = ij / q.th;
        const unsigned f = q.lo + cf % nf, c = cf / nf;
        const long long src = tile_base + ((long long)(c * q.Ft + f) * plane + i * q.tw + j);
        const long long dst = (((long long)sample * q.C + c) * q.F + q.f0 + f) * q.H * q.W + (q.r0 + i) * q.W + q.c0 + j;
        float o = cfg_combine_h(y[src], u[src], g);
        if (has_rescale) o = __half2float(__float2half_rn(o * scale));
        const float x0 = __fsub_rn(__fmul_rn(al, xt[dst]), __fmul_rn(sg, o));
        acc[dst] = __fmaf_rn(__fmul_rn(wy[i], wx[j]), x0, acc[dst]);
    }
}

}  // namespace star
