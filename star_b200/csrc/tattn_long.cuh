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
//   warpgroups 1, 2  query tiles 2r and 2r + 1 of round r (T <= 128 is one round), each key block through
//                    attn_block_step<64> of attn.cuh.  A warpgroup without a tile in the last round of an odd tile
//                    count still waits and releases every slot, so both warpgroups walk the same barrier sequence.
// Output rows (strided by HW * ldo) are written from registers, only for t < T.
// Bounds: B * HW * heads < 2^31 items (int32 item index and TMA coordinates) and T * HW * ld * 2 bytes < 2^40 (the
// tensor-map stride limit); T itself has no other bound.
#pragma once
#include "attn.cuh"

namespace star {

constexpr int TL_BT = 64;                  // frames per query tile and per key block
constexpr int TL_D = 64;
static_assert(TL_D == AT_D, "attn_block_step is for head_dim AT_D");
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
    uint8_t* smem = dyn_smem_1024();
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TattnLongSmem::OFF_BAR);
    StageRing<TL_Q_SLOTS> qr(bars);
    StageRing<TL_KV_STAGES> kv(bars + 2 * TL_Q_SLOTS);

    const int wg = threadIdx.x >> 7;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int T = p.T;
    const int nblk = (T + TL_BT - 1) / TL_BT;           // query tiles = key blocks
    const int rounds = (nblk + 1) / 2;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        qr.init(TL_CONSUMER_WARPS);
        kv.init(TL_CONSUMER_WARPS);
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");       // the item / round / block loop spills at 24
        if (threadIdx.x == 0) {
            for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
                const int head = item % p.heads;
                const int px = (item / p.heads) % p.HW;
                const int b = item / (p.heads * p.HW);
                for (int r = 0; r < rounds; ++r) {
                    const int ntiles = min(2, nblk - 2 * r);
                    qr.wait_empty();
                    uint64_t* q_full = &qr.full[qr.s];
                    mbar_expect_tx(q_full, ntiles * TattnLongSmem::TILE);
                    for (int c = 0; c < ntiles; ++c)
                        tma_load_4d(smem + TattnLongSmem::OFF_Q + (qr.s * 2 + c) * TattnLongSmem::TILE, &tmap, q_full,
                                    head * TL_D, (2 * r + c) * TL_BT, px, b);
                    qr.advance();
                    for (int j = 0; j < nblk; ++j) {
                        kv.wait_empty();
                        uint64_t* kv_full = &kv.full[kv.s];
                        mbar_expect_tx(kv_full, 2 * TattnLongSmem::TILE);
                        tma_load_4d(smem + TattnLongSmem::OFF_K + kv.s * TattnLongSmem::TILE, &tmap, kv_full,
                                    p.Ci + head * TL_D, j * TL_BT, px, b);
                        tma_load_4d(smem + TattnLongSmem::OFF_V + kv.s * TattnLongSmem::TILE, &tmap, kv_full,
                                    2 * p.Ci + head * TL_D, j * TL_BT, px, b);
                        kv.advance();
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
    const int klim[2] = {T, T};                          // every frame attends frames [0, T)
    const uint64_t dq0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_Q + cw * TattnLongSmem::TILE), 16, 1024);
    const uint64_t dk0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_K), 16, 1024);
    const uint64_t dv0 = wgmma_desc_sw128(smem_u32(smem + TattnLongSmem::OFF_V), TattnLongSmem::TILE, 1024);
    constexpr uint64_t TILE_INC = (uint64_t)(TattnLongSmem::TILE >> 4);

#pragma unroll 1
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
        const int head = item % p.heads;
        const int px = (item / p.heads) % p.HW;
        const int b = item / (p.heads * p.HW);
#pragma unroll 1
        for (int r = 0; r < rounds; ++r) {
            const int t0 = (2 * r + cw) * TL_BT;
            const bool active = t0 < T;
            const uint64_t dq = dq0 + 2 * TILE_INC * (uint64_t)qr.s;
            qr.wait_full();

            float o[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = 0.f;
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
            for (int j = 0; j < nblk; ++j) {
                kv.wait_full();
                if (active)
                    attn_block_step<TL_BT>(o, m_run, l_run, dq, dk0 + TILE_INC * (uint64_t)kv.s,
                                           dv0 + TILE_INC * (uint64_t)kv.s, j * TL_BT, klim, p.scale_log2);
                kv.release(kv.s);
                kv.advance();
            }
            qr.release(qr.s);                   // Q is only read by the S wgmmas, all complete
            qr.advance();

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
