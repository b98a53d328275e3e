// star_b200 / csrc / tapgemm.cuh
// "tap-GEMM": one wgmma implicit-GEMM kernel for every dense contraction of the
// STAR UNet on channels-last fp16 activations:
//     Out[row, n] = epi( sum_{tap} sum_{k} A[row + tap_offset, k] * W[n, tap*K + k] )
//   * Linear / 1x1 conv / Conv1d(k=1)   : 1 tap                 (unet_v2v.py:151-155, :274, :1005)
//   * Conv2d 3x3 (stride 1, pad 1)      : 9 taps over (h, w)    (unet_v2v.py:612, :639)
//   * Conv2d 3x3 stride 2 pad (2,1)     : 9 taps over 4 parity planes (unet_v2v.py:709-722)
//   * Conv3d (3,1,1) temporal conv      : 3 taps over t         (unet_v2v.py:1209-1220)
//   * causal Conv3d 3x3x3               : 27 taps over (t, h, w) of a clip stored with two leading frames
//                                         (cogvideox-based/sat/vae_modules/cp_enc_dec.py:360-430)
// The A operand is addressed through a rank-5 TMA tensor map (C, n1, n2, n3, n4); an
// M-tile is a box of <=128 "pixels"; each tap is a coordinate shift and out-of-bounds
// coordinates are zero-filled by TMA, which implements the conv zero padding and the
// ragged tile edges with no im2col buffer and no extra HBM traffic.
//
// Persistent kernel, one CTA per SM looping over 128 x BN output tiles (n fastest, so concurrently running CTAs
// share the A tile in L2).  Warpgroup 0: one TMA producer thread filling a ring of (A, W) stages; warpgroups 1 and 2:
// consumers, each computing 64 tile rows x BN columns with wgmma (fp32 accumulators in registers) and applying the
// fused epilogue.  The producer runs ahead into the next tile while the consumers finish the epilogue of the current one.
// The staged epilogue (calls whose output and residual TMA can address) writes each tile through two shared-memory slabs
// stored with TMA, without waiting for the writes; a second producer thread TMA-loads the residual into the slabs, the
// first two slabs of a tile under its main loop.  The direct epilogue (other calls) stores from registers.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace star {

constexpr int TG_BM = 128;      // rows (pixels) per tile
constexpr int TG_BK = 64;       // fp16 K elements per stage == 128 B swizzle span
constexpr int TG_MAX_TAPS = 27;   // 3x3x3 causal Conv3d of the CogVideoX VAE (cp_enc_dec.py:360-430)
constexpr int TG_THREADS = 384;
constexpr int TG_CONSUMER_WARPS = 8;

enum TapGemmFlags : int {
    TG_GEGLU = 1,        // W has 2N rows (value | gate); out = value * gelu_erf(gate)
    TG_SILU_OUT = 2,     // out = silu(acc)
    TG_GELU_ERF = 4,     // out = gelu_erf(acc)   (nn.GELU of the OpenCLIP text tower's MLP, embedder.py:27)
    TG_GELU_TANH = 8,    // out = gelu_tanh(acc)  (CogVideoX MLP, sat default gelu)
};

struct TapGemmParams {
    int on[4];            // output extents n1..n4 (n1 fastest); rows_out = prod
    int row_ext[4];       // extents of the output's row space (>= on; launch_tapgemm defaults them to on): a sub-box of a
                          // larger row space, e.g. a pixel band of every frame, is written in place (out and residual;
                          // launch_tapgemm refuses rowvec with extended extents)
    int box[4];           // tile box b1..b4, prod <= 128
    int tiles[4];         // ceil(on / box)
    int box_rows;         // prod(box)
    int ntaps;
    int tap[TG_MAX_TAPS][4];
    int K;                // per-tap reduction length
    int k_chunks;         // ceil(K / 64)
    int N;                // output columns
    int flags;
    int num_tiles;        // m_tiles * n_tiles
    int n_tiles;
    const __half* bias;   // [N] ([2N] with GEGLU) or null
    const __half* rowvec; // [rows_out / rowvec_div, N] or null  (time-embedding add, unet_v2v.py:684)
    int rowvec_div;
    long long rowvec_ld;  // row pitch of rowvec in elements (>= N)
    const __half* colscale;   // [N] or null: acc = colscale[n] * (acc + bias[n]) before the residual add (adaLN gate)
    const __half* residual;   // [rows_out, res_ld] or null
    long long res_ld;
    __half* out;
    long long out_ld;
};

// Shared memory: the stage ring, then (staged epilogue) two output slabs of 128 rows x 64 columns, then the barriers.
template <int BN, bool STAGED>
struct TapGemmSmem {
    static constexpr int A_BYTES = TG_BM * TG_BK * 2;          // 16 KB
    static constexpr int B_BYTES = BN * TG_BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int SLAB_BYTES = TG_BM * 64 * 2;          // 16 KB, 1024-B aligned (STAGE_BYTES is a multiple of 1024)
    static constexpr int SLABS = STAGED ? 2 : 0;
    static constexpr int MAX_STAGES = 8;
    static constexpr int STAGES_FIT = (232448 - 1024 - 256 - SLABS * SLAB_BYTES) / STAGE_BYTES;  // 227 KB minus slabs, slack, barriers
    static constexpr int STAGES = STAGES_FIT < MAX_STAGES ? STAGES_FIT : MAX_STAGES;
    static constexpr int SLAB_OFF = STAGES * STAGE_BYTES;
    static constexpr int BAR_OFF = SLAB_OFF + SLABS * SLAB_BYTES;
    static constexpr int TOTAL = BAR_OFF + 1024 + 256;
};

template <int BN>
STAR_DEVINL void tg_mma_k16(float* acc, uint64_t da, uint64_t db) {
    if constexpr (BN == 128) wgmma_m64n128_ss(acc, da, db);
    else if constexpr (BN == 160) wgmma_m64n160_ss(acc, da, db);
    else wgmma_m64n256_ss(acc, da, db);
}

STAR_DEVINL float tg_ld(const __half* p) { return __half2float(__ldg(p)); }

// Epilogue kinds.  An instance of the kernel is compiled for one set of epilogue operations, so its unrolled
// per-element code carries only the operations the call applies (the fully unrolled generic epilogue is 100-200 KB of
// SASS per kernel).  TG_EPI_GENERIC reads every option from the parameters at run time: it serves any combination that
// has no instance of its own.  The fp32 order per element is the same in every instance: bias, GEGLU / activation,
// colscale, rowvec, residual, SiLU.
enum TapGemmEpi : int {
    TG_EPI_BIAS = 1,
    TG_EPI_GEGLU = 2,
    TG_EPI_ROWVEC = 4,
    TG_EPI_COLSCALE = 8,
    TG_EPI_RES = 16,
    TG_EPI_ERF = 32,
    TG_EPI_TANH = 64,
    TG_EPI_SILU = 128,
    TG_EPI_GENERIC = 256,
};

// The combinations the library's callers pass (UNet, OpenCLIP text tower, CogVideoX DiT, both VAEs), and the generic
// instance.  Kinds with TG_EPI_GEGLU are compiled only at the tile widths GEGLU runs with (128 / 256): see tg_instance.
#define TG_EPI_KINDS(X)                                   \
    X(0)                                                  \
    X(TG_EPI_BIAS)                                        \
    X(TG_EPI_BIAS | TG_EPI_RES)                           \
    X(TG_EPI_BIAS | TG_EPI_ROWVEC)                        \
    X(TG_EPI_BIAS | TG_EPI_GEGLU)                         \
    X(TG_EPI_BIAS | TG_EPI_SILU)                          \
    X(TG_EPI_BIAS | TG_EPI_ERF)                           \
    X(TG_EPI_BIAS | TG_EPI_TANH)                          \
    X(TG_EPI_BIAS | TG_EPI_COLSCALE | TG_EPI_RES)         \
    X(TG_EPI_GENERIC)

// Whether instance <BN, EPI> of a kind in TG_EPI_KINDS is compiled: every one except the GEGLU kinds at BN = 160.
constexpr bool tg_instance(int bn, int epi) { return !(bn == 160 && (epi & TG_EPI_GEGLU)); }

// The kind of a call: its flags and which epilogue inputs it passes.
inline int tg_epi_kind(int flags, bool bias, bool rowvec, bool colscale, bool residual) {
    return (bias ? TG_EPI_BIAS : 0) | ((flags & TG_GEGLU) ? TG_EPI_GEGLU : 0) | (rowvec ? TG_EPI_ROWVEC : 0) |
           (colscale ? TG_EPI_COLSCALE : 0) | (residual ? TG_EPI_RES : 0) | ((flags & TG_GELU_ERF) ? TG_EPI_ERF : 0) |
           ((flags & TG_GELU_TANH) ? TG_EPI_TANH : 0) | ((flags & TG_SILU_OUT) ? TG_EPI_SILU : 0);
}

// The epilogue options of instance EPI: compile-time constants, or read from the parameters for TG_EPI_GENERIC.
template <int EPI>
struct TapGemmEpiOpts {
    static constexpr bool GEN = (EPI & TG_EPI_GENERIC) != 0;
    bool geglu, bias, rowvec, colscale, res, erf, tanh, silu;
    STAR_DEVINL explicit TapGemmEpiOpts(const TapGemmParams& p)
        : geglu(GEN ? (p.flags & TG_GEGLU) != 0 : (EPI & TG_EPI_GEGLU) != 0),
          bias(GEN ? p.bias != nullptr : (EPI & TG_EPI_BIAS) != 0),
          rowvec(GEN ? p.rowvec != nullptr : (EPI & TG_EPI_ROWVEC) != 0),
          colscale(GEN ? p.colscale != nullptr : (EPI & TG_EPI_COLSCALE) != 0),
          res(GEN ? p.residual != nullptr : (EPI & TG_EPI_RES) != 0),
          erf(GEN ? (p.flags & TG_GELU_ERF) != 0 : (EPI & TG_EPI_ERF) != 0),
          tanh(GEN ? (p.flags & TG_GELU_TANH) != 0 : (EPI & TG_EPI_TANH) != 0),
          silu(GEN ? (p.flags & TG_SILU_OUT) != 0 : (EPI & TG_EPI_SILU) != 0) {}
};

// Epilogue of one consumer warpgroup: rows row_in_wg and row_in_wg + 8 of warpgroup cw's 64 tile rows, from the
// accumulators straight to global memory.  Per column pair the bias / colscale values are loaded once for both rows, and
// the residual loads of JG column pairs are issued ahead of the arithmetic that consumes them (a thread only ever stores
// to elements whose residual it has already read, so an output that aliases the residual stays correct).
template <int BN, int EPI>
STAR_DEVINL void tg_epilogue(const float (&acc)[BN / 2], const TapGemmParams& p, const int (&org)[4], int n_tile, int cw,
                             int row_in_wg, int q4) {
    const TapGemmEpiOpts<EPI> o(p);
    const int n_per_tile = o.geglu ? BN / 2 : BN;
    const bool out_pair = ((p.out_ld & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 3) == 0);
    const bool res_pair = !o.res || (((p.res_ld & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0));
    const int n_base = n_tile * n_per_tile;
    bool valid[2];
    __half* out_row[2];
    const __half *res_row[2], *rv_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = cw * 64 + row_in_wg + 8 * h;
        int rr = r;
        long long orow = 0, mul = 1;
        bool ok = r < p.box_rows;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int l = rr % p.box[i];
            rr /= p.box[i];
            const int g = org[i] + l;
            ok = ok && (g < p.on[i]);
            orow += (long long)g * mul;
            mul *= p.row_ext[i];
        }
        valid[h] = ok;
        out_row[h] = p.out + orow * p.out_ld;
        res_row[h] = o.res ? p.residual + orow * p.res_ld : nullptr;
        rv_row[h] = o.rowvec ? p.rowvec + (orow / p.rowvec_div) * p.rowvec_ld : nullptr;
    }
    if (!valid[0] && !valid[1]) return;
    constexpr int JG = 4;
    constexpr int JH = BN / 16;                      // GEGLU: value column groups [0, JH), gate column groups [JH, 2 JH)
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += JG) {
        if (o.geglu && j0 >= JH) break;
        uint32_t res2[JG][2];
#pragma unroll
        for (int jj = 0; jj < JG; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * (j0 + jj) + 2 * q4, n = n_base + c;
                res2[jj][h] = 0u;
                if (o.res && res_pair && valid[h] && c < n_per_tile && n + 1 < p.N)
                    res2[jj][h] = *reinterpret_cast<const uint32_t*>(res_row[h] + n);
            }
#pragma unroll
        for (int jj = 0; jj < JG; ++jj) {
            const int j = j0 + jj;
            const int jg = j < JH ? j + JH : j;
            if (o.geglu && j >= JH) break;
            const int c = 8 * j + 2 * q4;                    // tile column of this thread's pair
            const int n = n_base + c;
            if (c >= n_per_tile || n >= p.N) continue;
            const bool two = n + 1 < p.N;
            const int n1 = two ? n + 1 : n;                  // clamped index for the loads of a lone last column
            float bv[2] = {0.f, 0.f}, bg[2] = {0.f, 0.f}, cs[2] = {1.f, 1.f};
            if (o.bias) {
                bv[0] = tg_ld(p.bias + n);
                bv[1] = tg_ld(p.bias + n1);
                if (o.geglu) { bg[0] = tg_ld(p.bias + p.N + n); bg[1] = tg_ld(p.bias + p.N + n1); }
            }
            if (o.colscale) { cs[0] = tg_ld(p.colscale + n); cs[1] = tg_ld(p.colscale + n1); }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!valid[h]) continue;
                float f[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float x = acc[4 * j + 2 * h + e];
                    if (o.geglu) {
                        float g = acc[4 * jg + 2 * h + e];
                        if (o.bias) { x += bv[e]; g += bg[e]; }
                        x *= gelu_erf_f(g);
                    } else if (o.bias) {
                        x += bv[e];
                    }
                    if (o.tanh) x = gelu_tanh_f(x);
                    if (o.erf) x = gelu_erf_f(x);
                    if (o.colscale) x *= cs[e];
                    if (o.rowvec) x += tg_ld(rv_row[h] + (e ? n1 : n));
                    f[e] = x;
                }
                if (o.res) {
                    if (two && res_pair) {
                        const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(&res2[jj][h]));
                        f[0] += rv.x;
                        f[1] += rv.y;
                    } else {
                        f[0] += __half2float(res_row[h][n]);
                        if (two) f[1] += __half2float(res_row[h][n + 1]);
                    }
                }
                if (o.silu) { f[0] = silu_f(f[0]); f[1] = silu_f(f[1]); }
                if (two && out_pair) {
                    *reinterpret_cast<uint32_t*>(out_row[h] + n) = pack_half2(f[0], f[1]);
                } else {
                    out_row[h][n] = __float2half_rn(f[0]);
                    if (two) out_row[h][n + 1] = __float2half_rn(f[1]);
                }
            }
        }
    }
}

// Staged epilogue.  A tile's output columns are walked in slabs of 64 (the 128-wide tile: 2, 160: 64 + 64 + 32, 256: 4;
// GEGLU at 256: 2, at 128: 1), alternating between two shared-memory slab buffers laid out as the output tensor maps'
// boxes: box_rows rows of 128 B (the 32-column tail: 64 B) in the tile's row order, 128-byte (tail: 64-byte) swizzled.
// Buffer b has a full barrier (the residual slab's TMA bytes) and an empty barrier (arrived by the thread that stored the
// buffer's previous slab, once the store has read it).  The slabs of all tiles of a CTA are numbered in order; slab i
// uses buffer i & 1 for the (i >> 1)-th time.
STAR_DEVINL int tg_slab_count(const TapGemmParams& p, int n_per_tile, int n_base) {
    return (min(n_per_tile, p.N - n_base) + 63) >> 6;
}
// Byte offset of (row r, slab column cc) in a slab buffer: SWIZZLE_128B on 128-byte rows, SWIZZLE_64B on the 64-byte rows
// of the 32-column tail.  A warp's 8 rows of a column pair land in 8 different 16-B chunks: no bank conflicts.
STAR_DEVINL uint32_t tg_slab_off(int r, int cc, bool tail) {
    return tail ? (uint32_t)(r * 64 + cc * 2) ^ ((uint32_t)((r >> 1) & 3) << 4)
                : (uint32_t)(r * 128 + cc * 2) ^ ((uint32_t)(r & 7) << 4);
}
STAR_DEVINL void tg_consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Epilogue of one consumer warpgroup through the slab buffers.  Per slab: wait for the residual slab (or, without a
// residual, for the buffer to be free), read each element's residual from the slab, apply the same fp32 sequence as
// tg_epilogue, write the fp16 result over it in place, then one thread stores the slab with TMA (clipped at N and at the
// output extents, so ragged tiles and sub-box writes need no masking) and moves on without waiting for the write.
template <int BN, int EPI>
STAR_DEVINL void tg_epilogue_staged(const float (&acc)[BN / 2], const TapGemmParams& p, const CUtensorMap* tm_out,
                                    const CUtensorMap* tm_out_tail, uint8_t* slabs, uint64_t* slab_full,
                                    uint64_t* slab_empty, uint32_t& slab_i, const int (&org)[4], int n_tile, int cw,
                                    int row_in_wg, int q4) {
    const TapGemmEpiOpts<EPI> o(p);
    const int n_per_tile = o.geglu ? BN / 2 : BN;
    const int n_base = n_tile * n_per_tile;
    const int ns = tg_slab_count(p, n_per_tile, n_base);
    int row[2];
    bool valid[2];
    const __half* rv_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = cw * 64 + row_in_wg + 8 * h;
        int rr = r;
        long long orow = 0, mul = 1;
        bool ok = r < p.box_rows;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int l = rr % p.box[i];
            rr /= p.box[i];
            const int g = org[i] + l;
            ok = ok && (g < p.on[i]);
            orow += (long long)g * mul;
            mul *= p.row_ext[i];
        }
        row[h] = r;
        valid[h] = ok;
        rv_row[h] = o.rowvec ? p.rowvec + (orow / p.rowvec_div) * p.rowvec_ld : nullptr;
    }
    constexpr int JH = BN / 16;                      // GEGLU: value column groups [0, JH), gate column groups [JH, 2 JH)
#pragma unroll
    for (int s = 0; s < (BN + 63) / 64; ++s) {
        if (s >= ns) break;
        const bool tail = BN == 160 && s == 2;       // the 32-column tail slab of the 160-wide tile
        const int b = slab_i & 1;
        const uint32_t use_parity = (slab_i >> 1) & 1;
        uint8_t* slab = slabs + b * TapGemmSmem<BN, true>::SLAB_BYTES;
        if (o.res) mbar_wait(&slab_full[b], use_parity);
        else mbar_wait(&slab_empty[b], use_parity ^ 1);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * s + jj;
            if (j >= BN / 8) break;
            if (o.geglu && j >= JH) break;
            const int jg = j < JH ? j + JH : j;
            const int cc = 8 * jj + 2 * q4;                  // slab column of this thread's pair
            const int c = 64 * s + cc;                       // tile column
            const int n = n_base + c;
            if (c >= n_per_tile || n >= p.N) continue;
            const int n1 = n + 1 < p.N ? n + 1 : n;          // clamped index for the loads of a lone last column
            float bv[2] = {0.f, 0.f}, bg[2] = {0.f, 0.f}, cs[2] = {1.f, 1.f};
            if (o.bias) {
                bv[0] = tg_ld(p.bias + n);
                bv[1] = tg_ld(p.bias + n1);
                if (o.geglu) { bg[0] = tg_ld(p.bias + p.N + n); bg[1] = tg_ld(p.bias + p.N + n1); }
            }
            if (o.colscale) { cs[0] = tg_ld(p.colscale + n); cs[1] = tg_ld(p.colscale + n1); }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!valid[h]) continue;
                uint32_t* sp = reinterpret_cast<uint32_t*>(slab + tg_slab_off(row[h], cc, tail));
                float f[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float x = acc[4 * j + 2 * h + e];
                    if (o.geglu) {
                        float g = acc[4 * jg + 2 * h + e];
                        if (o.bias) { x += bv[e]; g += bg[e]; }
                        x *= gelu_erf_f(g);
                    } else if (o.bias) {
                        x += bv[e];
                    }
                    if (o.tanh) x = gelu_tanh_f(x);
                    if (o.erf) x = gelu_erf_f(x);
                    if (o.colscale) x *= cs[e];
                    if (o.rowvec) x += tg_ld(rv_row[h] + (e ? n1 : n));
                    f[e] = x;
                }
                if (o.res) {           // not contracted with a product before it: tg_epilogue adds it in a block of its own
                    const uint32_t r2 = *sp;
                    const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(&r2));
                    f[0] = __fadd_rn(f[0], rv.x);
                    f[1] = __fadd_rn(f[1], rv.y);
                }
                if (o.silu) { f[0] = silu_f(f[0]); f[1] = silu_f(f[1]); }
                *sp = pack_half2(f[0], f[1]);
            }
        }
        fence_proxy_async_smem();                    // the slab's generic writes, before the async proxy reads them
        tg_consumer_sync();
        if (threadIdx.x == TG_THREADS / 3) {         // first consumer thread: issues every store of the CTA
            tma_store_5d(tail ? tm_out_tail : tm_out, slab, n_base + 64 * s, org[0], org[1], org[2], org[3]);
            bulk_commit_group();
            bulk_wait_group_read<0>();
            mbar_arrive(&slab_empty[b]);
        }
        ++slab_i;
    }
}

template <int BN, int EPI, bool STAGED>
__global__ void __launch_bounds__(TG_THREADS, 1)
tapgemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_res,
               const __grid_constant__ CUtensorMap tmap_out_tail, const __grid_constant__ CUtensorMap tmap_res_tail,
               const __grid_constant__ TapGemmParams p) {
    using SM = TapGemmSmem<BN, STAGED>;
    uint8_t* smem = dyn_smem_1024();
    StageRing<SM::STAGES> ring(reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF));
    uint8_t* slabs = smem + SM::SLAB_OFF;
    uint64_t* slab_full = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF) + 2 * SM::STAGES;
    uint64_t* slab_empty = slab_full + 2;

    const int wg = threadIdx.x >> 7;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const TapGemmEpiOpts<EPI> opts(p);
    const bool geglu = opts.geglu;
    const int total_iters = p.ntaps * p.k_chunks;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_w);
        ring.init(TG_CONSUMER_WARPS);
        if constexpr (STAGED) {
            tma_prefetch_desc(&tmap_out);
            for (int b = 0; b < 2; ++b) {
                mbar_init(&slab_full[b], 1);
                mbar_init(&slab_empty[b], 1);
            }
        }
        fence_barrier_init();
    }
    __syncthreads();

    auto tile_origin = [&](int tile, int* org, int& n_tile) {
        n_tile = tile % p.n_tiles;
        int m_tile = tile / p.n_tiles;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            org[i] = (m_tile % p.tiles[i]) * p.box[i];
            m_tile /= p.tiles[i];
        }
    };

    if (wg == 0) {
        // ------------------------------------------------ TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            const uint32_t tx = (uint32_t)p.box_rows * 128u + (uint32_t)SM::B_BYTES;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                int org[4], n_tile;
                tile_origin(tile, org, n_tile);
                for (int t = 0; t < p.ntaps; ++t) {
                    const int c1 = org[0] + p.tap[t][0], c2 = org[1] + p.tap[t][1];
                    const int c3 = org[2] + p.tap[t][2], c4 = org[3] + p.tap[t][3];
                    for (int kc = 0; kc < p.k_chunks; ++kc) {
                        ring.wait_empty();
                        uint64_t* full = &ring.full[ring.s];
                        uint8_t* sa = smem + ring.s * SM::STAGE_BYTES;
                        uint8_t* sb = sa + SM::A_BYTES;
                        mbar_expect_tx(full, tx);
                        tma_load_5d(sa, &tmap_a, full, kc * TG_BK, c1, c2, c3, c4);
                        const int kw = t * p.K + kc * TG_BK;
                        if (!geglu) {
                            tma_load_2d(sb, &tmap_w, full, kw, n_tile * BN);
                        } else {
                            tma_load_2d(sb, &tmap_w, full, kw, n_tile * (BN / 2));
                            tma_load_2d(sb + (BN / 2) * 128, &tmap_w, full, kw, p.N + n_tile * (BN / 2));
                        }
                        ring.advance();
                    }
                }
            }
        } else if (STAGED && opts.res && threadIdx.x == 32) {
            // ------------------------------------------------ residual producer: each tile's residual slabs, in the
            // consumers' slab order, as soon as their buffer is free (the first two of a tile arrive under its main loop)
            const int n_per_tile = geglu ? BN / 2 : BN;
            uint32_t slab_i = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                int org[4], n_tile;
                tile_origin(tile, org, n_tile);
                const int n_base = n_tile * n_per_tile;
                const int ns = tg_slab_count(p, n_per_tile, n_base);
                for (int s = 0; s < ns; ++s, ++slab_i) {
                    const int b = slab_i & 1;
                    const bool tail = BN == 160 && s == 2;
                    mbar_wait(&slab_empty[b], ((slab_i >> 1) & 1) ^ 1);
                    mbar_expect_tx(&slab_full[b], (uint32_t)p.box_rows * (tail ? 64u : 128u));
                    tma_load_5d(slabs + b * SM::SLAB_BYTES, tail ? &tmap_res_tail : &tmap_res, &slab_full[b], n_base + 64 * s,
                                org[0], org[1], org[2], org[3]);
                }
            }
        }
        return;
    }

    // ---------------------------------------------------- consumers: warpgroup cw owns tile rows [64 cw, 64 cw + 64)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int q4 = lane & 3;
    const int row_in_wg = (warp & 3) * 16 + (lane >> 2);
    const uint64_t desc_a0 = wgmma_desc_sw128(smem_u32(smem) + cw * 64 * 128, 16, 1024);
    const uint64_t desc_b0 = wgmma_desc_sw128(smem_u32(smem) + SM::A_BYTES, 16, 1024);
    constexpr uint64_t STAGE_INC = (uint64_t)(SM::STAGE_BYTES >> 4);
    uint32_t slab_i = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        int org[4], n_tile;
        tile_origin(tile, org, n_tile);
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev_s = -1;
#pragma unroll 1
        for (int it = 0; it < total_iters; ++it) {
            ring.wait_full();
            const uint64_t da = desc_a0 + STAGE_INC * (uint64_t)ring.s;
            const uint64_t db = desc_b0 + STAGE_INC * (uint64_t)ring.s;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TG_BK / 16; ++k) tg_mma_k16<BN>(acc, da + 2 * k, db + 2 * k);
            wgmma_commit();
            wgmma_wait<1>();                         // the MMAs of the previous stage have retired: release it
            if (prev_s >= 0) ring.release(prev_s);
            prev_s = ring.s;
            ring.advance();
        }
        wgmma_wait<0>();
        if (prev_s >= 0) ring.release(prev_s);

        if constexpr (STAGED)
            tg_epilogue_staged<BN, EPI>(acc, p, &tmap_out, &tmap_out_tail, slabs, slab_full, slab_empty, slab_i, org, n_tile,
                                        cw, row_in_wg, q4);
        else
            tg_epilogue<BN, EPI>(acc, p, org, n_tile, cw, row_in_wg, q4);
    }
    if (STAGED && threadIdx.x == TG_THREADS / 3) bulk_wait_group<0>();      // the stores have written global memory
}

}  // namespace star
