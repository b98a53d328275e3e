// star_b200 / csrc / tattn2.cuh
// Temporal self-attention over T <= 64 frames per (pixel, head) (unet_v2v.py:483-489), second version.  Chunks of
// T > 64 frames (max_chunk_len >= 52) run temporal_attn_long_kernel (tattn_long.cuh, wgmma); star_temporal_attention
// picks the kernel by T.
// The problem is a 32x32x64 attention per item, 131 760 items per call at level 0: HBM-bound (the q|k|v
// rows of a pixel are 128-byte segments strided by H*W rows).  v1 did the two small matmuls on the FMA
// pipes with per-element fp16->fp32 converts and was instruction-bound (988 GB/s).  Here one warp handles
// one item with warp-level tensor-core MMAs (mma.sync m16n8k16, fp16 in / fp32 accumulate): a 64-row
// wgmma tile cannot be filled by a 32-row problem, and the kernel stays memory-bound either way.
//   * Q, K, V rows are copied global -> smem with 16-byte cp.async (4 rows per warp instruction), padded row
//     pitch 144 B so ldmatrix is conflict-free; rows >= T are zero-filled and masked
//   * per 16-query block: S = Q K^T in registers, row softmax with quad shuffles, P re-used as the A
//     fragments of P V, O staged through smem and written with 16-byte stores
#pragma once
#include "common.cuh"

namespace star {

constexpr int TA2_WARPS = 8;
constexpr int TA2_MAXT = 64;             // frames per chunk (the reference uses 32, stretched last chunk up to 40)
constexpr int TA2_PITCH = 144;           // bytes per smem row (128 B of data + 16 B pad)

STAR_DEVINL void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
STAR_DEVINL void cp_async_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }
STAR_DEVINL void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
STAR_DEVINL void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
STAR_DEVINL void mma_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32." STAR_MMA_SYNC_T "." STAR_MMA_SYNC_T ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int TP>                    // frames padded to a multiple of 16: 16, 32, 48, 64
__global__ void __launch_bounds__(TA2_WARPS * 32)
temporal_attn2_kernel(const __half* __restrict__ qkv, long long ld, __half* __restrict__ out, long long ldo, int B, int T,
                      long long HW, int heads, int Ci, float scale) {
    extern __shared__ __align__(16) uint8_t ta2_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int MAT = TP * TA2_PITCH;                      // one matrix (Q, K or V) of one warp
    uint8_t* base = ta2_smem + (size_t)warp * 3 * MAT;
    const uint32_t sq = smem_u32(base), sk = sq + MAT, sv = sk + MAT;
    const long long nitems = (long long)B * HW * heads;
    const long long stride = (long long)gridDim.x * TA2_WARPS;
    const float sl2 = scale * 1.4426950408889634f;
    const int g = lane >> 2, tq = lane & 3;

    // zero the padding rows once (rows T..TP-1 of all three matrices)
    for (int i = lane; i < (TP - T) * 9; i += 32) {
        const int row = T + i / 9, ch = i % 9;
#pragma unroll
        for (int m = 0; m < 3; ++m) *reinterpret_cast<uint4*>(base + m * MAT + row * TA2_PITCH + ch * 16) = make_uint4(0, 0, 0, 0);
    }

    for (long long item = (long long)blockIdx.x * TA2_WARPS + warp; item < nitems; item += stride) {
        const int head = (int)(item % heads);
        const long long px = (item / heads) % HW;
        const int b = (int)(item / (heads * HW));
        const long long row0 = (long long)b * T * HW + px;
        __syncwarp();
        // ---- global -> smem: 3 matrices x T rows x 8 chunks of 16 B
        for (int i = lane; i < T * 8; i += 32) {
            const int t = i >> 3, ch = i & 7;
            const __half* src = qkv + (row0 + (long long)t * HW) * ld + head * 64 + ch * 8;
            const uint32_t off = (uint32_t)(t * TA2_PITCH + ch * 16);
            cp_async16(sq + off, src);
            cp_async16(sk + off, src + Ci);
            cp_async16(sv + off, src + 2 * Ci);
        }
        cp_async_wait_all();
        __syncwarp();

#pragma unroll 1
        for (int mi = 0; mi < TP / 16; ++mi) {
            if (mi * 16 >= T) break;
            // ---- S = Q K^T for 16 query rows
            float s[TP / 8][4];
#pragma unroll
            for (int ni = 0; ni < TP / 8; ++ni) s[ni][0] = s[ni][1] = s[ni][2] = s[ni][3] = 0.f;
            uint32_t qa[4][4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const int row = mi * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
                const int col = kk * 16 + 8 * (lane >> 4);
                ldsm_x4(sq + row * TA2_PITCH + col * 2, qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3]);
            }
#pragma unroll
            for (int ni = 0; ni < TP / 8; ++ni) {
                uint32_t kb[8];
                const int row = ni * 8 + (lane & 7);
                ldsm_x4(sk + row * TA2_PITCH + (lane >> 3) * 16, kb[0], kb[1], kb[2], kb[3]);            // d  0..31
                ldsm_x4(sk + row * TA2_PITCH + 64 + (lane >> 3) * 16, kb[4], kb[5], kb[6], kb[7]);       // d 32..63
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) mma_16816(s[ni], qa[kk], kb[kk * 2], kb[kk * 2 + 1]);
            }
            // ---- softmax over keys for rows g and g+8 of this block
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int ni = 0; ni < TP / 8; ++ni) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const bool ok = (ni * 8 + tq * 2 + e) < T;
                    s[ni][e] = ok ? s[ni][e] * sl2 : -INFINITY;
                    s[ni][2 + e] = ok ? s[ni][2 + e] * sl2 : -INFINITY;
                    m0 = fmaxf(m0, s[ni][e]);
                    m1 = fmaxf(m1, s[ni][2 + e]);
                }
            }
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            float l0 = 0.f, l1 = 0.f;
            uint32_t pa[TP / 16][4];
#pragma unroll
            for (int ni = 0; ni < TP / 8; ++ni) {
                const float p0 = ex2_approx(s[ni][0] - m0), p1 = ex2_approx(s[ni][1] - m0);
                const float p2 = ex2_approx(s[ni][2] - m1), p3 = ex2_approx(s[ni][3] - m1);
                l0 += p0 + p1;
                l1 += p2 + p3;
                pa[ni >> 1][(ni & 1) * 2] = pack_half2(p0, p1);
                pa[ni >> 1][(ni & 1) * 2 + 1] = pack_half2(p2, p3);
            }
            l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
            l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
            // ---- O = P V
            float o[8][4];
#pragma unroll
            for (int nd = 0; nd < 8; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
#pragma unroll
            for (int kj = 0; kj < TP / 16; ++kj) {
#pragma unroll
                for (int np = 0; np < 4; ++np) {                 // two 8-wide d tiles per ldmatrix.x4.trans
                    uint32_t vb[4];
                    const int row = kj * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
                    const int col = np * 16 + 8 * (lane >> 4);
                    ldsm_x4_trans(sv + row * TA2_PITCH + col * 2, vb[0], vb[1], vb[2], vb[3]);
                    mma_16816(o[np * 2], pa[kj], vb[0], vb[1]);
                    mma_16816(o[np * 2 + 1], pa[kj], vb[2], vb[3]);
                }
            }
            // ---- stage O rows (reuse this block's Q rows, already consumed) and write 16-byte chunks
            const float i0 = 1.f / l0, i1 = 1.f / l1;
            __syncwarp();
#pragma unroll
            for (int nd = 0; nd < 8; ++nd) {
                *reinterpret_cast<uint32_t*>(base + (mi * 16 + g) * TA2_PITCH + (nd * 8 + tq * 2) * 2) = pack_half2(o[nd][0] * i0, o[nd][1] * i0);
                *reinterpret_cast<uint32_t*>(base + (mi * 16 + g + 8) * TA2_PITCH + (nd * 8 + tq * 2) * 2) = pack_half2(o[nd][2] * i1, o[nd][3] * i1);
            }
            __syncwarp();
            for (int i = lane; i < 16 * 8; i += 32) {
                const int t = mi * 16 + (i >> 3), ch = i & 7;
                if (t < T)
                    *reinterpret_cast<uint4*>(out + (row0 + (long long)t * HW) * ldo + head * 64 + ch * 8) =
                        *reinterpret_cast<const uint4*>(base + t * TA2_PITCH + ch * 16);
            }
        }
    }
}

}  // namespace star
