// star_b200 / csrc / common.cuh
// sm_90a device helpers: mbarrier, TMA (cp.async.bulk.tensor), math.  Raw PTX; the
// warpgroup MMA wrappers are in wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// One source, two builds: libstar_sm100.so computes on fp16 tokens, libstar_sm100_bf16.so (-DSTAR_BF16) on bf16 tokens
// (the CogVideoX DiT runs bf16: cogvideox_5b_infer_sr.yaml:11).  Every storage-type conversion in the kernels goes through
// the intrinsics re-pointed below; accumulation, statistics and softmax stay fp32 in both builds.
#ifdef STAR_BF16
#include <cuda_bf16.h>
#define __half __nv_bfloat16
#define __half2 __nv_bfloat162
#define __float2half_rn __float2bfloat16_rn
#define __half2float __bfloat162float
#define __floats2half2_rn __floats2bfloat162_rn
#define __half22float2 __bfloat1622float2
#define STAR_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
#define STAR_MMA_SYNC_T "bf16"
#else
#define STAR_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_FLOAT16
#define STAR_MMA_SYNC_T "f16"
#endif

namespace star {

#define STAR_DEVINL __device__ __forceinline__

STAR_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
STAR_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
STAR_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
STAR_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
STAR_DEVINL void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
STAR_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug (lost arrive / wrong parity) traps after ~2 s of SM clocks instead of hanging
// the GPU (try_wait itself may block for a system-dependent time, so the bound is on clock64, not on spins).
// No printf here: a function call between wgmma issue and wait makes ptxas serialise the wgmma pipeline.
#ifndef STAR_WAIT_CYCLES
#define STAR_WAIT_CYCLES 4000000000ll
#endif
STAR_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    long long t0 = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 255u) == 0) {
            const long long now = clock64();
            if (t0 == 0) {
                t0 = now;
            } else if (now - t0 > STAR_WAIT_CYCLES) {
                __trap();
            }
        }
    }
}

// A ring of NS shared-memory stages between one TMA producer thread and the consumer warps.  Stage s has a full
// barrier (the producer's expect_tx, completed by the TMA bytes) and an empty barrier (one arrive per consumer warp),
// full[0..NS) followed by empty[0..NS).  The producer and every consumer thread each keep their own position and walk
// the stages in the same order.  A stage's n-th use completes phase n of its full barrier and, once released, phase n of
// its empty barrier.  So for use n a consumer waits for full at parity n & 1, and the producer waits for phase n - 1 of
// empty, at the opposite parity, which a freshly initialised barrier passes: the first lap needs no release.
template <int NS>
struct StageRing {
    uint64_t* full;
    uint64_t* empty;
    int s = 0;           // current stage
    uint32_t ph = 0;     // parity of the current lap

    STAR_DEVINL explicit StageRing(uint64_t* bars) : full(bars), empty(bars + NS) {}
    STAR_DEVINL void init(uint32_t consumer_warps) const {       // thread 0, before the CTA-wide barrier-init fence
        for (int i = 0; i < NS; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], consumer_warps);
        }
    }
    STAR_DEVINL void wait_empty() const { mbar_wait(&empty[s], ph ^ 1); }
    STAR_DEVINL void wait_full() const { mbar_wait(&full[s], ph); }
    // Called by every thread of a consumer warp once its reads of the stage are complete.
    STAR_DEVINL void release(int stage) const {
        if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage]);
    }
    STAR_DEVINL void advance() {
        if (++s == NS) { s = 0; ph ^= 1; }
    }
};

// Dynamic shared memory rounded up to 1024 B, the alignment of 128-byte-swizzled TMA tiles and wgmma operands: kernels
// that use it request 1 KB more than their layout needs.
STAR_DEVINL uint8_t* dyn_smem_1024() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

// ---------------------------------------------------------------- fences
STAR_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- thread-block clusters
STAR_DEVINL uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
STAR_DEVINL uint32_t cluster_nctarank() {
    uint32_t n;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
    return n;
}
// Every thread of every CTA of the cluster arrives (release: its earlier shared-memory writes become visible to the
// cluster) and waits (acquire) for all of them; both must be reached by whole warps.
STAR_DEVINL void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
STAR_DEVINL void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// The float at the same shared-memory offset as p in the CTA of cluster rank `rank` (distributed shared memory).
STAR_DEVINL float ld_dsmem_f32(const float* p, uint32_t rank) {
    uint32_t a;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(p)), "r"(rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

// ---------------------------------------------------------------- TMA
STAR_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
STAR_DEVINL void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
STAR_DEVINL void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
STAR_DEVINL void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
STAR_DEVINL void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3), "r"(c4)
        : "memory");
}
// Store of a shared-memory box to global memory (clipped at the tensor map's extents), tracked in the issuing thread's
// bulk async-groups: commit closes a group; bulk_wait_group_read<N> returns once at most N groups still read shared memory
// (their source may then be overwritten), bulk_wait_group<N> once at most N groups are still writing global memory.
STAR_DEVINL void tma_store_5d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
        ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
STAR_DEVINL void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
STAR_DEVINL void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
STAR_DEVINL void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- misc math
STAR_DEVINL float ex2_approx(float x);
STAR_DEVINL float silu_f(float x) { return x / (1.0f + __expf(-x)); }
// exact (erf) GELU, nn.GELU() default (unet_v2v.py:504).  erf by Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7, far
// below the fp16 rounding of the result): 2 MUFU + ~12 FMA-pipe ops instead of libdevice erff's ~30.
STAR_DEVINL float erf_as(float x) {
    const float ax = fabsf(x);
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float e = ex2_approx(-1.4426950408889634f * ax * ax);
    const float r = fmaf(-poly * t, e, 1.0f);
    return copysignf(r, x);
}
STAR_DEVINL float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f)); }
STAR_DEVINL float gelu_tanh_f(float x) {
    const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
    return 0.5f * x * (1.0f + t);
}
STAR_DEVINL float sigmoid_f(float x) { return 1.0f / (1.0f + __expf(-x)); }

STAR_DEVINL uint32_t pack_half2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace star

namespace star {
STAR_DEVINL void unpack8h(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

STAR_DEVINL float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
}  // namespace star
