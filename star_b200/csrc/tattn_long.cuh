// star_b200 / csrc / tattn_long.cuh
// Temporal self-attention over T > 64 frames per (pixel, head) (unet_v2v.py:483-489 with a long chunk).  T <= 64 is
// temporal_attn2_kernel (tattn2.cuh, mma.sync: a 32-frame problem cannot fill a 64-row wgmma tile); from 65 frames on
// every 64-frame query tile is full enough for wgmma.
//
// Persistent CTAs loop over items (clip, pixel, head), heads fastest.  Warp roles (384 threads):
//   warpgroup 0      one TMA producer thread.  One 4-D tensor map over QKV, dims {columns, t, pixel, clip}, box
//                    {64, 64, 1, 1}: one copy lands a 64-frame x 64-channel tile of one (pixel, head), 128-byte
//                    swizzled.  Frames >= T are zero-filled by TMA and masked.  Per round of two query tiles it loads
//                    the Q tiles into a ring of Q slots, then every 64-frame K/V block into a ring of K/V stages, so
//                    the next items' loads overlap the current item's math.
//   warpgroups 1, 2  query tiles 2r and 2r + 1 of round r (T <= 128 is one round):
//                      S_j = Q K_j^T            wgmma m64n64k16, both operands K-major in shared memory
//                      online softmax over 64-key blocks in registers (two rows per thread, quad shuffles)
//                      O  += P_j V_j            wgmma m64n64k16, P as the register A operand, V MN-major
//                    A warpgroup without a tile in the last round of an odd tile count still waits and releases
//                    every slot, so both warpgroups walk the same barrier sequence.
// Output rows (strided by HW * ldo) are written from registers, only for t < T.
// Bounds: B * HW * heads < 2^31 items (int32 item index and TMA coordinates) and T * HW * ld * 2 bytes < 2^40 (the
// tensor-map stride limit); T itself has no other bound.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace star {

constexpr int TL_BT = 64;                  // frames per query tile and per key block
constexpr int TL_D = 64;
constexpr int TL_Q_SLOTS = 4;              // Q slots of two tiles each (one round)
constexpr int TL_KV_STAGES = 8;
constexpr int TL_THREADS = 384;
constexpr int TL_CONSUMER_WARPS = 8;

struct TattnLongParams {
    int T, heads, HW;
    int nitems;                // items = B * HW * heads
    int Ci;                    // K at column Ci + 64 head, V at 2 Ci + 64 head
    float scale_log2;          // softmax scale * log2(e)
    __half* out;
    long long ldo;
};

struct TattnLongSmem {
    static constexpr int TILE = TL_BT * TL_D * 2;                   // 8 KB
    static constexpr int OFF_Q = 0;                                 // TL_Q_SLOTS x 2 tiles
    static constexpr int OFF_K = OFF_Q + TL_Q_SLOTS * 2 * TILE;
    static constexpr int OFF_V = OFF_K + TL_KV_STAGES * TILE;
    static constexpr int OFF_BAR = OFF_V + TL_KV_STAGES * TILE;
    static constexpr int TOTAL = OFF_BAR + 256 + 1024;              // barriers + 1 KB for the alignment of the tiles
};

__global__ void __launch_bounds__(TL_THREADS, 1)
temporal_attn_long_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ TattnLongParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TattnLongSmem::OFF_BAR);
    uint64_t* q_full = bars;                            // TL_Q_SLOTS
    uint64_t* q_empty = q_full + TL_Q_SLOTS;            // TL_Q_SLOTS
    uint64_t* kv_full = q_empty + TL_Q_SLOTS;           // TL_KV_STAGES
    uint64_t* kv_empty = kv_full + TL_KV_STAGES;        // TL_KV_STAGES

    const int wg = threadIdx.x >> 7;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int T = p.T;
    const int nblk = (T + TL_BT - 1) / TL_BT;           // query tiles = key blocks
    const int rounds = (nblk + 1) / 2;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        for (int s = 0; s < TL_Q_SLOTS; ++s) {
            mbar_init(&q_full[s], 1);
            mbar_init(&q_empty[s], TL_CONSUMER_WARPS);
        }
        for (int s = 0; s < TL_KV_STAGES; ++s) {
            mbar_init(&kv_full[s], 1);
            mbar_init(&kv_empty[s], TL_CONSUMER_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");       // the item / round / block loop spills at 24
        if (threadIdx.x == 0) {
            int qs = 0, s = 0;
            uint32_t qph = 0, ph = 0;
            for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
                const int head = item % p.heads;
                const int px = (item / p.heads) % p.HW;
                const int b = item / (p.heads * p.HW);
                for (int r = 0; r < rounds; ++r) {
                    const int ntiles = min(2, nblk - 2 * r);
                    mbar_wait(&q_empty[qs], qph ^ 1);
                    mbar_expect_tx(&q_full[qs], ntiles * TattnLongSmem::TILE);
                    for (int c = 0; c < ntiles; ++c)
                        tma_load_4d(smem + TattnLongSmem::OFF_Q + (qs * 2 + c) * TattnLongSmem::TILE, &tmap, &q_full[qs],
                                    head * TL_D, (2 * r + c) * TL_BT, px, b);
                    if (++qs == TL_Q_SLOTS) { qs = 0; qph ^= 1; }
                    for (int j = 0; j < nblk; ++j) {
                        mbar_wait(&kv_empty[s], ph ^ 1);
                        mbar_expect_tx(&kv_full[s], 2 * TattnLongSmem::TILE);
                        tma_load_4d(smem + TattnLongSmem::OFF_K + s * TattnLongSmem::TILE, &tmap, &kv_full[s],
                                    p.Ci + head * TL_D, j * TL_BT, px, b);
                        tma_load_4d(smem + TattnLongSmem::OFF_V + s * TattnLongSmem::TILE, &tmap, &kv_full[s],
                                    2 * p.Ci + head * TL_D, j * TL_BT, px, b);
                        if (++s == TL_KV_STAGES) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int q4 = lane & 3;
    const int row_in_wg = (warp & 3) * 16 + (lane >> 2);
    const uint64_t dq0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_Q + cw * TattnLongSmem::TILE), 16, 1024);
    const uint64_t dk0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_K), 16, 1024);
    const uint64_t dv0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_V), TattnLongSmem::TILE, 1024);
    constexpr uint64_t TILE_INC = (uint64_t)(TattnLongSmem::TILE >> 4);
    const float sl2 = p.scale_log2;

    int qs = 0, s = 0;
    uint32_t qph = 0, ph = 0;
#pragma unroll 1
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
        const int head = item % p.heads;
        const int px = (item / p.heads) % p.HW;
        const int b = item / (p.heads * p.HW);
#pragma unroll 1
        for (int r = 0; r < rounds; ++r) {
            const int t0 = (2 * r + cw) * TL_BT;
            const bool active = t0 < T;
            const uint64_t dq = dq0 + 2 * TILE_INC * (uint64_t)qs;
            mbar_wait(&q_full[qs], qph);

            float o[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = 0.f;
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
            for (int j = 0; j < nblk; ++j) {
                mbar_wait(&kv_full[s], ph);
                if (active) {
                    float sacc[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
                    const uint64_t dk = dk0 + TILE_INC * (uint64_t)s;
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < TL_D / 16; ++k) wgmma_m64n64_ss(sacc, dq + 2 * k, dk + 2 * k);
                    wgmma_commit();
                    wgmma_wait<0>();

                    const int kbase = j * TL_BT;
                    float alpha[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (kbase + TL_BT > T) {
#pragma unroll
                            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                                for (int e = 0; e < 2; ++e)
                                    if (kbase + 8 * jj + 2 * q4 + e >= T) sacc[4 * jj + 2 * h + e] = -INFINITY;
                        }
                        float mx = -INFINITY;
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sacc[4 * jj + 2 * h], sacc[4 * jj + 2 * h + 1]));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                        const float m_new = fmaxf(m_run[h], mx * sl2);
                        alpha[h] = ex2_approx(m_run[h] - m_new);
                        m_run[h] = m_new;
                        float l = 0.f;
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const float pv = ex2_approx(fmaf(sacc[4 * jj + 2 * h + e], sl2, -m_new));
                                sacc[4 * jj + 2 * h + e] = pv;
                                l += pv;
                            }
                        l_run[h] = l_run[h] * alpha[h] + l;
                    }
                    // P as the A operand of P V: k-step kk covers keys [16 kk, 16 kk + 16) = accumulator pairs 2kk, 2kk+1
                    uint32_t pa[TL_BT / 16][4];
#pragma unroll
                    for (int kk = 0; kk < TL_BT / 16; ++kk) {
                        pa[kk][0] = pack_half2(sacc[8 * kk + 0], sacc[8 * kk + 1]);
                        pa[kk][1] = pack_half2(sacc[8 * kk + 2], sacc[8 * kk + 3]);
                        pa[kk][2] = pack_half2(sacc[8 * kk + 4], sacc[8 * kk + 5]);
                        pa[kk][3] = pack_half2(sacc[8 * kk + 6], sacc[8 * kk + 7]);
                    }
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        o[4 * jj + 0] *= alpha[0];
                        o[4 * jj + 1] *= alpha[0];
                        o[4 * jj + 2] *= alpha[1];
                        o[4 * jj + 3] *= alpha[1];
                    }
                    const uint64_t dv = dv0 + TILE_INC * (uint64_t)s;
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < TL_BT / 16; ++kk) wgmma_m64n64_rs_tb(o, pa[kk], dv + (uint64_t)(kk * (2048 >> 4)));
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                if (lane == 0) mbar_arrive(&kv_empty[s]);
                if (++s == TL_KV_STAGES) { s = 0; ph ^= 1; }
            }
            if (lane == 0) mbar_arrive(&q_empty[qs]);           // Q is only read by the S wgmmas, all complete
            if (++qs == TL_Q_SLOTS) { qs = 0; qph ^= 1; }

            if (active) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float l = l_run[h];
                    l += __shfl_xor_sync(0xffffffffu, l, 1);
                    l += __shfl_xor_sync(0xffffffffu, l, 2);
                    const float inv = 1.0f / l;
                    const int t = t0 + row_in_wg + 8 * h;
                    if (t < T) {
                        __half* op = p.out + (((long long)b * T + t) * p.HW + px) * p.ldo + head * TL_D + 2 * q4;
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj)
                            *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_half2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
                    }
                }
            }
        }
    }
}

}  // namespace star
