// star_b200 / csrc / attn.cuh
// Flash-style attention forward for head_dim 64, fp16 in / fp32 softmax + accumulate:
//     O = softmax(Q K^T * scale) V          (no bias; optional causal mask for the text tower)
// replaces xformers.ops.memory_efficient_attention at unet_v2v.py:179/:184 for the
// spatial self-attention (N = H*W up to 26 352) and the text cross-attention (Nk = 77).
//
// One CTA = 192 query rows of one (batch, head).  Warp roles (512 threads):
//   warpgroup 0        one TMA producer thread: Q once, then K/V tiles (128 keys) through a ring of stages
//   warpgroups 1 - 3   64 query rows each, one attn_block_step<128> per K/V tile: a third consumer gives the scheduler
//                      a third independent chain of MMA, MUFU and FMA work to interleave
// Keys beyond Nk are zero-filled by TMA and masked; with `causal` the key tiles past the last query row are skipped.
// attn_block_step is also the consumer step of temporal_attn_long_kernel (tattn_long.cuh).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace star {

constexpr int AT_BQ = 192;
constexpr int AT_BKV = 128;
constexpr int AT_D = 64;
constexpr int AT_KV_STAGES = 4;
constexpr int AT_THREADS = 512;
constexpr int AT_CONSUMER_WARPS = 12;

struct AttnParams {
    int Nq, Nk;
    int causal;             // 1: query row q attends keys 0..q only (text tower)
    int kv_batch_div;       // kv batch index = q batch index / kv_batch_div (text context shared by the frames of a clip)
    float scale_log2;       // softmax scale * log2(e)
    __half* out;
    long long ldo;          // elements between consecutive rows of O
};

struct AttnSmem {
    static constexpr int Q_TILE = AT_BQ * AT_D * 2;           // 24 KB
    static constexpr int TILE = AT_BKV * AT_D * 2;            // 16 KB: one K or V tile
    static constexpr int OFF_Q = 0;
    static constexpr int OFF_K = OFF_Q + Q_TILE;
    static constexpr int OFF_V = OFF_K + AT_KV_STAGES * TILE;
    static constexpr int OFF_BAR = OFF_V + AT_KV_STAGES * TILE;
    static constexpr int TOTAL = OFF_BAR + 256 + 1024;
};

// One key block of a consumer warpgroup's online softmax over 64 query rows, for the thread's two rows h of the
// accumulator fragment (wgmma.cuh):
//     S = Q K^T     over the BKV keys from kbase, wgmma m64nBKVk16, both operands K-major in shared memory
//     softmax       keys at or past klim[h] masked; running max m_run (scaled, log2 domain) and sum l_run updated with
//                   quad shuffles, O rescaled
//     O += P V      wgmma m64n64k16 with P as the register A operand (the S fragment packed to pairs), V MN-major
template <int BKV>
STAR_DEVINL void attn_block_step(float (&o)[32], float (&m_run)[2], float (&l_run)[2], uint64_t dq, uint64_t dk,
                                 uint64_t dv, int kbase, const int (&klim)[2], float sl2) {
    static_assert(BKV == 64 || BKV == 128, "key blocks of 64 or 128");
    const int q4 = threadIdx.x & 3;
    float sacc[BKV / 2];
#pragma unroll
    for (int i = 0; i < BKV / 2; ++i) sacc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) {
        if constexpr (BKV == 128) wgmma_m64n128_ss(sacc, dq + 2 * k, dk + 2 * k);
        else wgmma_m64n64_ss(sacc, dq + 2 * k, dk + 2 * k);
    }
    wgmma_commit();
    wgmma_wait<0>();

    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (kbase + BKV > klim[h]) {
#pragma unroll
            for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (kbase + 8 * jj + 2 * q4 + e >= klim[h]) sacc[4 * jj + 2 * h + e] = -INFINITY;
        }
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) mx = fmaxf(mx, fmaxf(sacc[4 * jj + 2 * h], sacc[4 * jj + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[h], mx * sl2);
        alpha[h] = ex2_approx(m_run[h] - m_new);
        m_run[h] = m_new;
        float l = 0.f;
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float pv = ex2_approx(fmaf(sacc[4 * jj + 2 * h + e], sl2, -m_new));
                sacc[4 * jj + 2 * h + e] = pv;
                l += pv;
            }
        l_run[h] = l_run[h] * alpha[h] + l;
    }
    // P as the A operand of P V: k-step kk covers keys [16 kk, 16 kk + 16) = accumulator columns of pairs 2kk, 2kk+1
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
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
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) wgmma_m64n64_rs_tb(o, pa[kk], dv + (uint64_t)(kk * (2048 >> 4)));
    wgmma_commit();
    wgmma_wait<0>();
}

__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ AttnParams p) {
    uint8_t* smem = dyn_smem_1024();
    uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + AttnSmem::OFF_BAR);
    StageRing<AT_KV_STAGES> kv(q_full + 1);

    // warp-uniform through the shuffle, so the Q descriptor of the warpgroup lives in uniform registers: held in vector
    // registers, dq + 2k spills at the 512-thread register budget
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * AT_BQ;
    const int head = blockIdx.y;
    const int batch = blockIdx.z;
    const int kv_batch = batch / p.kv_batch_div;
    int nt = (p.Nk + AT_BKV - 1) / AT_BKV;
    if (p.causal) nt = min(nt, (min(p.Nq, q0 + AT_BQ) + AT_BKV - 1) / AT_BKV);   // keys past the tile's last query

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_k);
        tma_prefetch_desc(&tmap_v);
        mbar_init(q_full, 1);
        kv.init(AT_CONSUMER_WARPS);
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
        if (threadIdx.x == 0) {
            mbar_expect_tx(q_full, AttnSmem::Q_TILE);
            tma_load_3d(smem + AttnSmem::OFF_Q, &tmap_q, q_full, head * AT_D, q0, batch);
            for (int j = 0; j < nt; ++j) {
                kv.wait_empty();
                uint64_t* full = &kv.full[kv.s];
                mbar_expect_tx(full, 2 * AttnSmem::TILE);
                tma_load_3d(smem + AttnSmem::OFF_K + kv.s * AttnSmem::TILE, &tmap_k, full, head * AT_D, j * AT_BKV, kv_batch);
                tma_load_3d(smem + AttnSmem::OFF_V + kv.s * AttnSmem::TILE, &tmap_v, full, head * AT_D, j * AT_BKV, kv_batch);
                kv.advance();
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");         // 128 x 24 + 384 x 160 <= 64K registers
    const int cw = wg - 1;
    const int q4 = lane & 3;
    const int row_in_wg = (warp & 3) * 16 + (lane >> 2);
    const int qrow[2] = {q0 + cw * 64 + row_in_wg, q0 + cw * 64 + row_in_wg + 8};
    const int klim[2] = {p.causal ? min(p.Nk, qrow[0] + 1) : p.Nk,           // keys [0, klim) are visible to the row
                         p.causal ? min(p.Nk, qrow[1] + 1) : p.Nk};
    const uint64_t dq = wgmma_desc_sw128(smem_u32(smem + AttnSmem::OFF_Q) + cw * 64 * 128, 16, 1024);
    const uint64_t dk0 = wgmma_desc_sw128(smem_u32(smem + AttnSmem::OFF_K), 16, 1024);
    const uint64_t dv0 = wgmma_desc_sw128(smem_u32(smem + AttnSmem::OFF_V), 8192, 1024);
    constexpr uint64_t TILE_INC = (uint64_t)(AttnSmem::TILE >> 4);

    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    mbar_wait(q_full, 0);
#pragma unroll 1
    for (int j = 0; j < nt; ++j) {
        kv.wait_full();
        attn_block_step<AT_BKV>(o, m_run, l_run, dq, dk0 + TILE_INC * (uint64_t)kv.s, dv0 + TILE_INC * (uint64_t)kv.s,
                                j * AT_BKV, klim, p.scale_log2);
        kv.release(kv.s);
        kv.advance();
    }

#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        // the row again from threadIdx, not qrow[h]: held across the key loop, qrow spills at 512 threads
        const int row = q0 + ((int)(threadIdx.x >> 7) - 1) * 64 + row_in_wg + 8 * h;
        if (row < p.Nq) {
            __half* op = p.out + ((long long)batch * p.Nq + row) * p.ldo + head * AT_D + 2 * q4;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
                *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_half2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        }
    }
}

}  // namespace star
