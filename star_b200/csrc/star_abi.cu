// star_b200 / csrc / star_abi.cu -- host side of libstar_sm100.so, the sm_90a kernel library (C ABI in include/star_sm100.h)
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../include/star_sm100.h"
#include "attn.cuh"
#include "rowops.cuh"
#include "tattn2.cuh"
#include "tattn_long.cuh"
#include "tapgemm.cuh"

using namespace star;

namespace {

thread_local std::string g_err;
PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
constexpr int STAR_MAX_DEVICES = 64;
int g_sms[STAR_MAX_DEVICES] = {0};            // SM count per initialised device (0 = star_init not called for it)
std::atomic<long long> g_launches{0};

// SM count of the CURRENT device (kernels are launched on the caller's current device / stream)
inline int num_sms() {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < STAR_MAX_DEVICES && g_sms[dev] > 0) return g_sms[dev];
    return 132;
}

int fail(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return 1;
}

#define STAR_CHECK_INIT()                                                                                        \
    do {                                                                                                         \
        int dev_ = -1;                                                                                           \
        if (!g_encode || cudaGetDevice(&dev_) != cudaSuccess || dev_ < 0 || dev_ >= STAR_MAX_DEVICES || !g_sms[dev_]) \
            return fail("star_init(%d) has not been called for the current device (or failed)", dev_);           \
    } while (0)
#define STAR_CUDA(x)                                                                        \
    do {                                                                                    \
        cudaError_t e_ = (x);                                                               \
        if (e_ != cudaSuccess) return fail("%s failed: %s", #x, cudaGetErrorString(e_));    \
    } while (0)
#define STAR_LAUNCH_CHECK(name)                                                             \
    do {                                                                                    \
        g_launches.fetch_add(1, std::memory_order_relaxed);                                 \
        cudaError_t e_ = cudaGetLastError();                                                \
        if (e_ != cudaSuccess) return fail("launch %s failed: %s", name, cudaGetErrorString(e_)); \
    } while (0)

// rank-`rank` fp16 tensor map, dims[0] innermost (contiguous), strides in ELEMENTS for dims 1..rank-1
int make_tmap(CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
              const unsigned long long* strides_elems, const unsigned* box,
              CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
        if (i > 0) {
            gstr[i - 1] = strides_elems[i] * 2ull;
            if (gstr[i - 1] % 16) return fail("tensor map stride %llu B of dim %d is not a multiple of 16", (unsigned long long)gstr[i - 1], i);
        }
        if (box[i] == 0 || box[i] > 256) return fail("tensor map box[%d]=%u out of range", i, box[i]);
    }
    if (reinterpret_cast<uintptr_t>(base) % 16) return fail("tensor map base not 16-byte aligned");
    CUresult r = g_encode(m, STAR_TMAP_DTYPE, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return 0;
}

inline int grid_for(long long n, int block, int cap_mult = 32) {
    long long g = (n + block - 1) / block;
    return (int)std::max(1ll, std::min(g, (long long)num_sms() * cap_mult));
}

// ------------------------------------------------------------------ tap-GEMM launcher
// Tile width: the one of 128 / 160 / 256 output columns (GEGLU: 64 / 128 value columns) that pads N least, the wider on
// a tie (fewer tiles, more reuse of each A tile).
int tile_width(int N, bool geglu) {
    auto padded = [&](int w) { return ((long long)N + w - 1) / w * w; };
    if (geglu) return padded(128) <= padded(64) ? 256 : 128;
    const long long p128 = padded(128), p160 = padded(160), p256 = padded(256);
    if (p256 <= p128 && p256 <= p160) return 256;
    return p160 <= p128 ? 160 : 128;
}

// The tensor maps of one tap-GEMM launch: the A and W operands and, for the staged epilogue, the output and residual
// slabs (64 columns, and the 32-column tail of the 160-wide tile).  All of them together with TapGemmParams must fit the
// 4 KB of kernel parameters.
struct TapGemmMaps {
    CUtensorMap a, w, out{}, res{}, out_tail{}, res_tail{};
};
static_assert(sizeof(TapGemmMaps) + sizeof(TapGemmParams) <= 4096, "tap-GEMM kernel parameters exceed 4 KB");

// The epilogue instance compiled for exactly this call's epilogue kind, else the generic one.
template <int BN, bool STAGED>
void launch_tapgemm_epi(const TapGemmMaps& m, const TapGemmParams& p, int grid, cudaStream_t st) {
    const int kind = tg_epi_kind(p.flags, p.bias, p.rowvec, p.colscale, p.residual);
    auto kernel = tapgemm_kernel<BN, TG_EPI_GENERIC, STAGED>;
#define TG_EPI_CASE(K)                                                     \
    if constexpr ((K) != TG_EPI_GENERIC && tg_instance(BN, (K)))          \
        if (kind == (K)) kernel = tapgemm_kernel<BN, (K), STAGED>;
    TG_EPI_KINDS(TG_EPI_CASE)
#undef TG_EPI_CASE
    kernel<<<grid, TG_THREADS, TapGemmSmem<BN, STAGED>::TOTAL, st>>>(m.a, m.w, m.out, m.res, m.out_tail, m.res_tail, p);
}

// Raises the dynamic shared-memory limit of instance <BN, EPI> (both epilogue paths), if it is compiled.
template <int BN, int EPI>
int tapgemm_smem_attr() {
    if constexpr (tg_instance(BN, EPI)) {
        STAR_CUDA(cudaFuncSetAttribute(tapgemm_kernel<BN, EPI, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       TapGemmSmem<BN, true>::TOTAL));
        STAR_CUDA(cudaFuncSetAttribute(tapgemm_kernel<BN, EPI, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       TapGemmSmem<BN, false>::TOTAL));
    }
    return 0;
}

// Whether TMA can address the slabs of an [rows, N] view with row pitch ld: a 16-byte-aligned base, and a row pitch and
// a row length of whole 16-byte units (on an H100 a TMA store was seen to clip the inner extent only to 16 bytes: with
// N % 8 != 0 it wrote past column N).  The staged epilogue needs it of the output and of the
// residual; other calls take the direct one.
bool tma_addressable(const void* base, long long ld, int N) {
    return reinterpret_cast<uintptr_t>(base) % 16 == 0 && ld % 8 == 0 && N % 8 == 0;
}

// Tensor map of the output (or residual) slabs of a tile: (column, n1..n4) over the output extents, rows laid out over the
// row extents, box = `cols` columns x the tile box.  TMA clips the box at the output extents and at N.
int make_slab_tmap(CUtensorMap* m, const void* base, long long ld, const TapGemmParams& p, unsigned cols) {
    unsigned long long dim[5] = {(unsigned long long)p.N}, str[5] = {1, (unsigned long long)ld};
    unsigned box[5] = {cols};
    for (int i = 0; i < 4; ++i) {
        dim[i + 1] = (unsigned long long)p.on[i];
        box[i + 1] = (unsigned)p.box[i];
        if (i > 0) str[i + 1] = str[i] * (unsigned long long)p.row_ext[i - 1];
    }
    return make_tmap(m, base, 5, dim, str, box, cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}

// Launches a tap-GEMM whose caller has filled p's output extents, box, taps, K, N, flags and epilogue inputs.  A holds
// p.K channels per row, rows lda elements apart, viewed as extents n1..n4 (n1 fastest); W is [N (2N with GEGLU), ntaps * K].
// Every other field of p, and the tensor maps, follow from those here.
// a_stride2 (elements, 0 = n1 rows of lda) is the distance between A's n2 slices when they are not packed back to back.
int launch_tapgemm(TapGemmParams& p, const void* A, unsigned long long lda, unsigned long long n1, unsigned long long n2,
                   unsigned long long n3, unsigned long long n4, const void* W, cudaStream_t st,
                   unsigned long long a_stride2 = 0) {
    long long m_tiles = 1;
    p.box_rows = 1;
    for (int i = 0; i < 4; ++i) {
        if (p.row_ext[i] == 0) p.row_ext[i] = p.on[i];
        p.tiles[i] = (p.on[i] + p.box[i] - 1) / p.box[i];
        m_tiles *= p.tiles[i];
        p.box_rows *= p.box[i];
    }
    if (p.box_rows > TG_BM) return fail("tapgemm: box has %d rows (> %d)", p.box_rows, TG_BM);
    for (int i = 0; i < 4; ++i)
        if (p.rowvec && p.row_ext[i] != p.on[i]) return fail("tapgemm: rowvec rows are not defined over extended row extents");
    p.k_chunks = (p.K + TG_BK - 1) / TG_BK;
    p.rowvec_div = std::max(1, p.rowvec_div);
    if (p.rowvec_ld <= 0) p.rowvec_ld = p.N;
    const bool geglu = p.flags & TG_GEGLU;
    const int bn = tile_width(p.N, geglu);
    const int n_per_tile = geglu ? bn / 2 : bn;
    p.n_tiles = (p.N + n_per_tile - 1) / n_per_tile;
    const long long total = m_tiles * p.n_tiles;
    if (total > 0x7fffffffll) return fail("tapgemm: too many tiles");
    p.num_tiles = (int)total;

    TapGemmMaps m;
    unsigned long long adim[5] = {(unsigned long long)p.K, n1, n2, n3, n4}, astr[5] = {1, lda};
    for (int i = 2; i < 5; ++i) astr[i] = (i == 2 && a_stride2) ? a_stride2 : astr[i - 1] * adim[i - 1];
    unsigned abox[5] = {TG_BK, (unsigned)p.box[0], (unsigned)p.box[1], (unsigned)p.box[2], (unsigned)p.box[3]};
    if (make_tmap(&m.a, A, 5, adim, astr, abox)) return 1;
    const unsigned long long wrows = geglu ? 2ull * p.N : (unsigned long long)p.N;
    unsigned long long wdim[2] = {(unsigned long long)p.ntaps * p.K, wrows};
    unsigned long long wstr[2] = {1, (unsigned long long)p.ntaps * p.K};
    unsigned wbox[2] = {TG_BK, (unsigned)n_per_tile};
    if (make_tmap(&m.w, W, 2, wdim, wstr, wbox)) return 1;

    // The staged epilogue stores through TMA and loads the residual with it; the direct one serves the calls TMA cannot address.
    const bool staged = tma_addressable(p.out, p.out_ld, p.N) && (!p.residual || tma_addressable(p.residual, p.res_ld, p.N));
    if (staged) {
        if (make_slab_tmap(&m.out, p.out, p.out_ld, p, 64)) return 1;
        if (p.residual && make_slab_tmap(&m.res, p.residual, p.res_ld, p, 64)) return 1;
        if (bn == 160) {
            if (make_slab_tmap(&m.out_tail, p.out, p.out_ld, p, 32)) return 1;
            if (p.residual && make_slab_tmap(&m.res_tail, p.residual, p.res_ld, p, 32)) return 1;
        }
    }
    const int grid = (int)std::min<long long>(total, num_sms());
    if (bn == 256) staged ? launch_tapgemm_epi<256, true>(m, p, grid, st) : launch_tapgemm_epi<256, false>(m, p, grid, st);
    else if (bn == 160) staged ? launch_tapgemm_epi<160, true>(m, p, grid, st) : launch_tapgemm_epi<160, false>(m, p, grid, st);
    else staged ? launch_tapgemm_epi<128, true>(m, p, grid, st) : launch_tapgemm_epi<128, false>(m, p, grid, st);
    STAR_LAUNCH_CHECK("tapgemm");
    return 0;
}

// Box of a conv tile over (w, h, frames): the 2-D box of at most 128 pixels that covers H x W in the fewest tiles (the
// wider on a tie), then as many of `frames` frames as fill 128 rows.
void conv_box(int H, int W, int frames, int* box) {
    long long best = -1;
    int th = 1, tw = 1;
    for (int w = 1; w <= std::min(W, 128); ++w) {
        int h = std::min(H, 128 / w);
        if (h < 1) continue;
        long long tiles = (long long)((W + w - 1) / w) * ((H + h - 1) / h);
        if (best < 0 || tiles < best || (tiles == best && w > tw)) {
            best = tiles;
            th = h;
            tw = w;
        }
    }
    box[0] = tw; box[1] = th; box[2] = std::max(1, std::min(frames, TG_BM / (tw * th))); box[3] = 1;
}

}  // namespace

extern "C" {

#ifdef STAR_BF16
int star_version(void) { return 101; }     /* odd: bf16 build */
#else
int star_version(void) { return 100; }
#endif
const char* star_last_error(void) { return g_err.c_str(); }
long long star_launch_count(void) { return g_launches.load(); }

// Per-device initialisation: checks the architecture, records the SM count and raises the dynamic shared-memory limit of
// every kernel ON THAT DEVICE (function attributes are per device).  The caller's current device is restored.
static int star_init_on_current(int device) {
    cudaDeviceProp prop;
    STAR_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail("libstar_sm100 is built for sm_90a and needs an sm_90 device, found sm_%d%d", prop.major, prop.minor);
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        STAR_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr));
        if (!fn || qr != cudaDriverEntryPointSuccess) return fail("cuTensorMapEncodeTiled not available from the driver");
        g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    }
#define STAR_SMEM_ATTR(kernel, bytes) STAR_CUDA((cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))))
#define TG_SMEM_ATTR(K) \
    if (tapgemm_smem_attr<128, (K)>() || tapgemm_smem_attr<160, (K)>() || tapgemm_smem_attr<256, (K)>()) return 1;
    TG_EPI_KINDS(TG_SMEM_ATTR)
#undef TG_SMEM_ATTR
    STAR_SMEM_ATTR(attn_fwd_kernel, AttnSmem::TOTAL);
    STAR_SMEM_ATTR(temporal_attn2_kernel<16>, TA2_WARPS * 3 * 16 * TA2_PITCH);
    STAR_SMEM_ATTR(temporal_attn2_kernel<32>, TA2_WARPS * 3 * 32 * TA2_PITCH);
    STAR_SMEM_ATTR(temporal_attn2_kernel<48>, TA2_WARPS * 3 * 48 * TA2_PITCH);
    STAR_SMEM_ATTR(temporal_attn2_kernel<64>, TA2_WARPS * 3 * 64 * TA2_PITCH);
    STAR_SMEM_ATTR(temporal_attn_long_kernel, TattnLongSmem::TOTAL);
    STAR_SMEM_ATTR(softmax_rows_kernel, SOFTMAX_SEG_MAX * 2);
#undef STAR_SMEM_ATTR
    g_sms[device] = prop.multiProcessorCount;
    return 0;
}

int star_init(int device) {
    if (device < 0 || device >= STAR_MAX_DEVICES) return fail("star_init: device index %d out of range", device);
    int prev = -1;
    STAR_CUDA(cudaGetDevice(&prev));
    if (prev != device) STAR_CUDA(cudaSetDevice(device));
    const int rc = star_init_on_current(device);
    if (prev != device && prev >= 0) cudaSetDevice(prev);          // never change the caller's current device
    return rc;
}

int star_linear(const void* A, long long lda, const void* W, const void* bias, const void* rowvec,
                long long rowvec_div, const void* residual, long long ldres, void* out, long long ldo,
                long long rows, int K, int N, int flags, void* stream) {
    return star_linear_ex(A, lda, W, bias, rowvec, rowvec_div, nullptr, residual, ldres, out, ldo, rows, K, N, flags, 0, 0,
                          stream);
}

// A head-blocked A (a_block_cols > 0) is a tap-GEMM with one tap per block: A viewed as (a_block_cols, rows, blocks) with
// the blocks a_block_pitch apart, tap t shifts to block t, and W's [N, K] columns are the taps' K ranges side by side.  The
// K loop (taps outer, 64-column chunks inner) thus visits W's columns in the order of the unblocked call, 64 at a time.
int star_linear_ex(const void* A, long long lda, const void* W, const void* bias, const void* rowvec,
                   long long rowvec_div, const void* colscale, const void* residual, long long ldres, void* out,
                   long long ldo, long long rows, int K, int N, int flags, int a_block_cols, long long a_block_pitch,
                   void* stream) {
    STAR_CHECK_INIT();
    if (rows <= 0) return 0;
    if (K % 8 || lda % 8) return fail("star_linear: K and lda must be multiples of 8 (K=%d lda=%lld)", K, lda);
    if (rows > 0x7fffffffll) return fail("star_linear: too many rows");
    const int blocks = a_block_cols > 0 ? K / a_block_cols : 1;
    if (a_block_cols > 0) {
        if (a_block_cols % TG_BK || K % a_block_cols)
            return fail("star_linear_ex: a_block_cols (%d) must be a multiple of %d dividing K (%d)", a_block_cols, TG_BK, K);
        if (blocks > TG_MAX_TAPS) return fail("star_linear_ex: %d A blocks (at most %d)", blocks, TG_MAX_TAPS);
        if (a_block_pitch % 8 || a_block_pitch < rows * lda)
            return fail("star_linear_ex: a_block_pitch %lld must be a multiple of 8 and hold %lld rows", a_block_pitch, rows);
        if (flags & TG_GEGLU) return fail("star_linear_ex: GEGLU does not take a head-blocked A");
    }
    TapGemmParams p{};
    p.on[0] = (int)rows; p.on[1] = p.on[2] = p.on[3] = 1;
    p.box[0] = TG_BM; p.box[1] = p.box[2] = p.box[3] = 1;
    p.ntaps = blocks;
    for (int t = 0; t < blocks; ++t) p.tap[t][1] = t;
    p.K = a_block_cols > 0 ? a_block_cols : K; p.N = N; p.flags = flags;
    p.bias = (const __half*)bias; p.rowvec = (const __half*)rowvec; p.rowvec_div = (int)rowvec_div;
    p.colscale = (const __half*)colscale; p.residual = (const __half*)residual; p.res_ld = ldres;
    p.out = (__half*)out; p.out_ld = ldo;
    return launch_tapgemm(p, A, lda, rows, blocks, 1, 1, W, (cudaStream_t)stream,
                          a_block_cols > 0 ? (unsigned long long)a_block_pitch : 0ull);
}

int star_conv2d_3x3(const void* X, const void* W9, const void* bias, const void* rowvec, long long rowvec_div, long long ldrowvec,
                    const void* residual, long long ldres, void* out, long long ldo, int BT, int H, int W, int Cin,
                    int Cout, int row0, int H_out, void* stream) {
    STAR_CHECK_INIT();
    if (Cin % 8) return fail("star_conv2d_3x3: Cin must be a multiple of 8");
    if (rowvec && ldrowvec % 8) return fail("star_conv2d_3x3: ldrowvec must be a multiple of 8");
    if (row0 < 0 || H_out < 1 || row0 + H_out > H) return fail("star_conv2d_3x3: output rows [%d, %d) outside [0, %d)", row0, row0 + H_out, H);
    TapGemmParams p{};
    p.on[0] = W; p.on[1] = H_out; p.on[2] = BT; p.on[3] = 1;
    conv_box(H_out, W, BT, p.box);
    p.ntaps = 9;
    for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
            p.tap[r * 3 + s][0] = s - 1;
            p.tap[r * 3 + s][1] = row0 + r - 1;
        }
    p.K = Cin; p.N = Cout;
    p.bias = (const __half*)bias; p.rowvec = (const __half*)rowvec; p.rowvec_div = (int)rowvec_div; p.rowvec_ld = ldrowvec;
    p.residual = (const __half*)residual; p.res_ld = ldres;
    p.out = (__half*)out; p.out_ld = ldo;
    return launch_tapgemm(p, X, Cin, W, H, BT, 1, W9, (cudaStream_t)stream);
}

long long star_conv2d_s2p_workspace_bytes(int BT, int H, int W, int Cin, int pad_t, int pad_b, int pad_l, int pad_r) {
    const long long Ho = (H + pad_t + pad_b - 3) / 2 + 1, Wo = (W + pad_l + pad_r - 3) / 2 + 1;
    return (long long)BT * 4 * (Ho + 1) * (Wo + 1) * Cin * 2;
}

long long star_conv2d_s2_workspace_bytes(int BT, int H, int W, int Cin) {
    return star_conv2d_s2p_workspace_bytes(BT, H, W, Cin, 2, 2, 1, 1);
}

int star_conv2d_3x3_s2(const void* X, const void* W9, const void* bias, void* out, long long ldo, void* planes_ws,
                       int BT, int H, int W, int Cin, int Cout, void* stream) {
    return star_conv2d_3x3_s2p(X, W9, bias, out, ldo, planes_ws, BT, H, W, Cin, Cout, 2, 2, 1, 1, stream);
}

int star_conv2d_3x3_s2p(const void* X, const void* W9, const void* bias, void* out, long long ldo, void* planes_ws,
                        int BT, int H, int W, int Cin, int Cout, int pad_t, int pad_b, int pad_l, int pad_r,
                        void* stream) {
    STAR_CHECK_INIT();
    if (Cin % 8) return fail("star_conv2d_3x3_s2p: Cin must be a multiple of 8");
    if (pad_t < 0 || pad_b < 0 || pad_l < 0 || pad_r < 0 || H + pad_t + pad_b < 3 || W + pad_l + pad_r < 3)
        return fail("star_conv2d_3x3_s2p: bad padding");
    const int Ho = (H + pad_t + pad_b - 3) / 2 + 1, Wo = (W + pad_l + pad_r - 3) / 2 + 1, H2 = Ho + 1, W2 = Wo + 1;
    cudaStream_t st = (cudaStream_t)stream;
    const long long n = (long long)BT * 4 * H2 * W2 * (Cin / 8);
    s2_split_kernel<<<grid_for(n, 256), 256, 0, st>>>((const __half*)X, (__half*)planes_ws, BT, H, W, Cin, H2, W2, pad_t, pad_l);
    STAR_LAUNCH_CHECK("s2_split");
    TapGemmParams p{};
    p.on[0] = Wo; p.on[1] = Ho; p.on[2] = 1; p.on[3] = BT;
    conv_box(Ho, Wo, 1, p.box);
    p.ntaps = 9;
    for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
            p.tap[r * 3 + s][0] = s >> 1;
            p.tap[r * 3 + s][1] = r >> 1;
            p.tap[r * 3 + s][2] = (r & 1) * 2 + (s & 1);
        }
    p.K = Cin; p.N = Cout;
    p.bias = (const __half*)bias;
    p.out = (__half*)out; p.out_ld = ldo;
    return launch_tapgemm(p, planes_ws, Cin, W2, H2, 4, BT, W9, st);
}

// X holds pixels [p0, p0 + band) of every frame compactly ([B, T, band, Cin]); residual / out rows are those pixels of the
// full [B, T, HW] row space (the tap-GEMM's row extents), so a pixel band of a clip-sized output is written in place.
int star_conv_t3(const void* X, const void* W3, const void* bias, const void* residual, long long ldres, void* out,
                      long long ldo, int B, int T, long long HW, long long p0, long long band, int Cin, int Cout, void* stream) {
    STAR_CHECK_INIT();
    if (Cin % 8) return fail("star_conv_t3: Cin must be a multiple of 8");
    if (HW > 0x7fffffffll) return fail("star_conv_t3: HW too large");
    if (p0 < 0 || band < 1 || p0 + band > HW) return fail("star_conv_t3: band [%lld, %lld) outside [0, %lld)", p0, p0 + band, HW);
    TapGemmParams p{};
    p.on[0] = (int)band; p.on[1] = T; p.on[2] = B; p.on[3] = 1;
    p.row_ext[0] = (int)HW;
    p.box[0] = (int)std::min<long long>(TG_BM, band); p.box[1] = 1; p.box[2] = 1; p.box[3] = 1;
    if (band < TG_BM) p.box[1] = (int)std::min<long long>(T, TG_BM / band);     // small latents: several frames per tile
    p.ntaps = 3;
    for (int k = 0; k < 3; ++k) p.tap[k][1] = k - 1;
    p.K = Cin; p.N = Cout;
    p.bias = (const __half*)bias;
    p.residual = residual ? (const __half*)residual + p0 * ldres : nullptr; p.res_ld = ldres;
    p.out = (__half*)out + p0 * ldo; p.out_ld = ldo;
    return launch_tapgemm(p, X, Cin, band, T, B, 1, W3, (cudaStream_t)stream);
}

// Causal Conv3d 3x3x3 of the CogVideoX 3-D VAE (cogvideox-based/sat/vae_modules/cp_enc_dec.py:360-430): X holds T + 2 frames --
// the two frames the reference concatenates in front of the clip (copies of frame 0, or the cache of the previous latent
// chunk, :265-268) followed by the T frames of the clip -- so output frame t reads input frames t, t+1, t+2; the spatial
// zero padding is the TMA out-of-bounds fill.  W27 is [Cout, 3(t), 3(h), 3(w), Cin].
int star_conv3d_causal(const void* X, const void* W27, const void* bias, const void* residual, long long ldres, void* out,
                       long long ldo, int T, int H, int W, int Cin, int Cout, void* stream) {
    STAR_CHECK_INIT();
    if (Cin % 8) return fail("star_conv3d_causal: Cin must be a multiple of 8");
    TapGemmParams p{};
    p.on[0] = W; p.on[1] = H; p.on[2] = T; p.on[3] = 1;
    conv_box(H, W, T, p.box);
    p.ntaps = 27;
    for (int q = 0; q < 3; ++q)
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 3; ++s) {
                int* tp = p.tap[(q * 3 + r) * 3 + s];
                tp[0] = s - 1; tp[1] = r - 1; tp[2] = q;
            }
    p.K = Cin; p.N = Cout;
    p.bias = (const __half*)bias; p.residual = (const __half*)residual; p.res_ld = ldres;
    p.out = (__half*)out; p.out_ld = ldo;
    return launch_tapgemm(p, X, Cin, W, H, T + 2, 1, W27, (cudaStream_t)stream);
}

long long star_conv2d_c4_workspace_bytes(int BT, int H, int W, int Cout) {
    return ((long long)BT * H * W * 64 + (long long)Cout * 64) * 2;
}

int star_conv2d_3x3_c4(const void* X, const void* W9, const void* bias, const void* residual, void* out, void* ws,
                       int BT, int H, int W, int Cout, void* stream) {
    STAR_CHECK_INIT();
    if (Cout % 8) return fail("star_conv2d_3x3_c4: Cout must be a multiple of 8");
    cudaStream_t st = (cudaStream_t)stream;
    const long long rows = (long long)BT * H * W;
    __half* col = (__half*)ws;
    __half* w64 = col + rows * 64;
    pad_w36_kernel<<<(Cout * 64 + 255) / 256, 256, 0, st>>>((const __half*)W9, w64, Cout);
    STAR_LAUNCH_CHECK("pad_w36");
    im2col_c4_kernel<<<grid_for(rows, 256), 256, 0, st>>>((const __half*)X, col, BT, H, W);
    STAR_LAUNCH_CHECK("im2col_c4");
    return star_linear(col, 64, w64, bias, nullptr, 1, residual, Cout, out, Cout, rows, 64, Cout, 0, stream);
}

static int attention_impl(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                          long long ldo, int batch, int heads, int Nq, int Nk, int kv_batch_div, float scale, int causal,
                          void* stream) {
    STAR_CHECK_INIT();
    if (ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) return fail("star_attention: leading dims must be multiples of 8");
    if (Nq <= 0 || Nk <= 0 || batch <= 0) return fail("star_attention: empty problem");
    if (kv_batch_div < 1) kv_batch_div = 1;
    const int kv_batches = (batch + kv_batch_div - 1) / kv_batch_div;
    CUtensorMap tq, tk, tv;
    {
        unsigned long long dims[3] = {(unsigned long long)heads * AT_D, (unsigned long long)Nq, (unsigned long long)batch};
        unsigned long long str[3] = {1, (unsigned long long)ldq, (unsigned long long)ldq * Nq};
        unsigned box[3] = {AT_D, AT_BQ, 1};
        if (make_tmap(&tq, Q, 3, dims, str, box)) return 1;
    }
    {
        unsigned long long dims[3] = {(unsigned long long)heads * AT_D, (unsigned long long)Nk, (unsigned long long)kv_batches};
        unsigned long long strk[3] = {1, (unsigned long long)ldk, (unsigned long long)ldk * Nk};
        unsigned long long strv[3] = {1, (unsigned long long)ldv, (unsigned long long)ldv * Nk};
        unsigned box[3] = {AT_D, AT_BKV, 1};
        if (make_tmap(&tk, K, 3, dims, strk, box)) return 1;
        if (make_tmap(&tv, V, 3, dims, strv, box)) return 1;
    }
    AttnParams p;
    p.Nq = Nq; p.Nk = Nk; p.kv_batch_div = kv_batch_div; p.causal = causal;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.out = (__half*)O; p.ldo = ldo;
    if (heads > 65535 || batch > 65535) return fail("star_attention: grid too large");
    dim3 grid((Nq + AT_BQ - 1) / AT_BQ, heads, batch);
    attn_fwd_kernel<<<grid, AT_THREADS, AttnSmem::TOTAL, (cudaStream_t)stream>>>(tq, tk, tv, p);
    STAR_LAUNCH_CHECK("attn_fwd");
    return 0;
}

int star_attention(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                   long long ldo, int batch, int heads, int Nq, int Nk, int kv_batch_div, float scale, void* stream) {
    return attention_impl(Q, ldq, K, ldk, V, ldv, O, ldo, batch, heads, Nq, Nk, kv_batch_div, scale, 0, stream);
}

// causal self-attention (query i attends keys 0..i): the text tower's attn_mask (embedder.py:57, open_clip build_attention_mask)
int star_attention_causal(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                          long long ldo, int batch, int heads, int N, float scale, void* stream) {
    return attention_impl(Q, ldq, K, ldk, V, ldv, O, ldo, batch, heads, N, N, 1, scale, 1, stream);
}

// T > 64: the wgmma kernel of tattn_long.cuh, one persistent CTA per SM
static int temporal_attention_long(const void* QKV, long long ld, void* O, long long ldo, int B, int T, long long HW,
                                   int heads, int Ci, float scale, long long items, cudaStream_t st) {
    if (B < 1 || HW < 1 || heads < 1) return fail("star_temporal_attention: empty problem");
    if (heads * TL_D > Ci || 3ll * Ci > ld) return fail("star_temporal_attention: need heads*64 <= Ci and 3*Ci <= ld");
    if (items > 0x7fffffffll) return fail("star_temporal_attention: B*HW*heads must be below 2^31");
    if ((unsigned long long)T * HW * ld * 2 >= (1ull << 40))
        return fail("star_temporal_attention: T*HW*ld*2 bytes must be below 2^40 (tensor-map stride limit)");
    CUtensorMap tm;
    unsigned long long dims[4] = {3ull * Ci, (unsigned long long)T, (unsigned long long)HW, (unsigned long long)B};
    unsigned long long str[4] = {1, (unsigned long long)(HW * ld), (unsigned long long)ld, (unsigned long long)T * HW * ld};
    unsigned box[4] = {TL_D, TL_BT, 1, 1};
    if (make_tmap(&tm, QKV, 4, dims, str, box)) return 1;
    TattnLongParams p;
    p.T = T; p.heads = heads; p.HW = (int)HW; p.nitems = (int)items; p.Ci = Ci;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.out = (__half*)O; p.ldo = ldo;
    const unsigned grid = (unsigned)std::min<long long>(items, (long long)num_sms());
    temporal_attn_long_kernel<<<grid, TL_THREADS, TattnLongSmem::TOTAL, st>>>(tm, p);
    STAR_LAUNCH_CHECK("temporal_attn_long");
    return 0;
}

int star_temporal_attention(const void* QKV, long long ld, void* O, long long ldo, int B, int T, long long HW,
                            int heads, int Ci, float scale, void* stream) {
    STAR_CHECK_INIT();
    if (T < 1) return fail("star_temporal_attention: T=%d must be >= 1", T);
    if (ld % 8 || ldo % 8 || Ci % 8) return fail("star_temporal_attention: ld/ldo/Ci must be multiples of 8");
    if ((reinterpret_cast<uintptr_t>(QKV) | reinterpret_cast<uintptr_t>(O)) % 16) return fail("star_temporal_attention: pointers must be 16-byte aligned");
    const long long items = (long long)B * HW * heads;
    cudaStream_t st = (cudaStream_t)stream;
    if (T > TA2_MAXT) return temporal_attention_long(QKV, ld, O, ldo, B, T, HW, heads, Ci, scale, items, st);
    const int tp = (T + 15) / 16 * 16;
    const unsigned grid = (unsigned)std::min<long long>((items + TA2_WARPS - 1) / TA2_WARPS, (long long)num_sms() * 2);
    const size_t smem = (size_t)TA2_WARPS * 3 * tp * TA2_PITCH;
#define STAR_TA2(TPV) temporal_attn2_kernel<TPV><<<grid, TA2_WARPS * 32, smem, st>>>((const __half*)QKV, ld, (__half*)O, ldo, B, T, HW, heads, Ci, scale)
    switch (tp) {
        case 16: STAR_TA2(16); break;
        case 32: STAR_TA2(32); break;
        case 48: STAR_TA2(48); break;
        default: STAR_TA2(64); break;
    }
#undef STAR_TA2
    STAR_LAUNCH_CHECK("temporal_attn2");
    return 0;
}

long long star_groupnorm_workspace_bytes(int nsamples, int C) {
    return (long long)nsamples * 32 * 2 * 8 + (long long)nsamples * C * 2 * 4;
}

static Gn2Range gn2_range(int nsamples, long long rows_per_sample, unsigned& grid) {
    Gn2Range rg;
    rg.slabs_per_sample = (rows_per_sample + GN2_SLAB - 1) / GN2_SLAB;
    rg.total_slabs = rg.slabs_per_sample * nsamples;
    grid = (unsigned)std::min<long long>(rg.total_slabs, (long long)num_sms() * 8);
    return rg;
}

// phases & STAR_GN_STATS: statistics + finalize into the workspace; phases & STAR_GN_APPLY: rows [p0, p0 + band) of every
// frame_rows-row frame normalised with the workspace's (a, b) and written compactly to out (the whole sample: in place is fine)
int star_groupnorm(const void* X, const void* gamma, const void* beta, void* out, int nsamples, long long rows_per_sample, int C,
                   float eps, int silu, long long frame_rows, long long p0, long long band, int phases, void* workspace,
                   void* stream) {
    if (C % 256 && C % 32) return fail("star_groupnorm: C must be a multiple of 32");
    if (C % 8) return fail("star_groupnorm: C must be a multiple of 8");
    if (C / 8 > GN_THREADS) return fail("star_groupnorm: C too large");
    if (phases < 1 || phases > (STAR_GN_STATS | STAR_GN_APPLY)) return fail("star_groupnorm: phases must be 1, 2 or 3");
    const bool whole = p0 == 0 && band == rows_per_sample && frame_rows == rows_per_sample;
    if (frame_rows < 1 || rows_per_sample % frame_rows || p0 < 0 || band < 1 || p0 + band > frame_rows)
        return fail("star_groupnorm: band [%lld, %lld) of %lld-row frames does not tile %lld-row samples", p0, p0 + band, frame_rows,
                    rows_per_sample);
    cudaStream_t st = (cudaStream_t)stream;
    double* stats = (double*)workspace;
    float* ab = (float*)((char*)workspace + (size_t)nsamples * 32 * 2 * 8);
    if (C / 8 <= GN2_THREADS) {
        // persistent CTAs over contiguous slab ranges: statistics / (a, b) stay in registers across slabs
        unsigned grid2;
        const Gn2Range rg = gn2_range(nsamples, rows_per_sample, grid2);
        if (phases & STAR_GN_STATS) {
            STAR_CUDA(cudaMemsetAsync(stats, 0, (size_t)nsamples * 32 * 2 * 8, st));
            const int lanes2 = GN2_THREADS / (C / 8);
            const size_t smem2 = (size_t)lanes2 * C * 2 * sizeof(float);
            gn_stats2_kernel<<<grid2, GN2_THREADS, smem2, st>>>((const __half*)X, stats, rows_per_sample, C, rg);
            STAR_LAUNCH_CHECK("gn_stats2");
            gn_finalize_kernel<<<nsamples, 256, 0, st>>>(stats, (const __half*)gamma, (const __half*)beta, ab, rows_per_sample, C, eps);
            STAR_LAUNCH_CHECK("gn_finalize");
        }
        if (!(phases & STAR_GN_APPLY)) return 0;
        if (band == frame_rows) {
            gn_apply2_kernel<<<grid2, GN2_THREADS, 0, st>>>((const __half*)X, ab, (__half*)out, rows_per_sample, C, silu, rg);
            STAR_LAUNCH_CHECK("gn_apply2");
            return 0;
        }
        const long long frames = (long long)nsamples * (rows_per_sample / frame_rows);
        gn_apply_band_kernel<<<grid_for(frames * band * (C / 8), 256), 256, 0, st>>>((const __half*)X, ab, (__half*)out,
                                                                                     rows_per_sample / frame_rows, frame_rows, p0,
                                                                                     band, frames, C, silu);
        STAR_LAUNCH_CHECK("gn_apply_band");
        return 0;
    }
    if (phases != (STAR_GN_STATS | STAR_GN_APPLY) || !whole) return fail("star_groupnorm: C > 2048 runs both phases over whole samples");
    STAR_CUDA(cudaMemsetAsync(stats, 0, (size_t)nsamples * 32 * 2 * 8, st));
    const long long total_rows = rows_per_sample * nsamples;
    const int lanes = std::max(1, GN_THREADS / (C / 8));
    const size_t smem = (size_t)lanes * C * 2 * sizeof(float);
    dim3 grid((unsigned)((rows_per_sample + GN_SLAB - 1) / GN_SLAB), nsamples);
    gn_stats_kernel<<<grid, GN_THREADS, smem, st>>>((const __half*)X, stats, rows_per_sample, C);
    STAR_LAUNCH_CHECK("gn_stats");
    gn_finalize_kernel<<<nsamples, 256, 0, st>>>(stats, (const __half*)gamma, (const __half*)beta, ab, rows_per_sample, C, eps);
    STAR_LAUNCH_CHECK("gn_finalize");
    gn_apply_kernel<<<grid_for(total_rows * (C / 8), 256), 256, 0, st>>>((const __half*)X, ab, (__half*)out, rows_per_sample,
                                                                          total_rows, C, silu);
    STAR_LAUNCH_CHECK("gn_apply");
    return 0;
}

// SpatialNorm3D of the CogVideoX 3-D VAE decoder (cp_enc_dec.py:451-510): out = GroupNorm32(X) * Ymod[src] + Bmod[src] (+ SiLU)
// over ONE clip of T x H x W rows; Ymod / Bmod = conv_y(zq) / conv_b(zq) at latent resolution (Tl, Hl, Wl) (see
// gn_apply_mod_kernel), row pitch ldmod.  Workspace: star_groupnorm_workspace_bytes(1, C).
int star_groupnorm_mod(const void* X, const void* gamma, const void* beta, const void* Ymod, const void* Bmod, long long ldmod,
                       void* out, int T, int H, int W, int Tl, int Hl, int Wl, int C, float eps, int silu, void* workspace, void* stream) {
    if (C % 32) return fail("star_groupnorm_mod: C must be a multiple of 32");
    if (C / 8 > GN2_THREADS) return fail("star_groupnorm_mod: C too large");
    if (H % Hl || W % Wl) return fail("star_groupnorm_mod: feature size must be a multiple of the latent size");
    if (ldmod % 8 || ldmod < C) return fail("star_groupnorm_mod: ldmod must be a multiple of 8 and >= C");
    const bool split = T > 1 && (T & 1);
    if (split ? ((T - 1) % std::max(1, Tl - 1) != 0 || Tl < 2) : (T % Tl != 0))
        return fail("star_groupnorm_mod: T=%d is not an integer multiple of the latent T=%d", T, Tl);
    const long long rows = (long long)T * H * W;
    if (rows > 0x7fffffffll) return fail("star_groupnorm_mod: more than 2^31 rows");
    cudaStream_t st = (cudaStream_t)stream;
    double* stats = (double*)workspace;
    float* ab = (float*)((char*)workspace + (size_t)32 * 2 * 8);
    STAR_CUDA(cudaMemsetAsync(stats, 0, (size_t)32 * 2 * 8, st));
    Gn2Range rg;
    rg.slabs_per_sample = (rows + GN2_SLAB - 1) / GN2_SLAB;
    rg.total_slabs = rg.slabs_per_sample;
    const int lanes2 = GN2_THREADS / (C / 8);
    const size_t smem2 = (size_t)lanes2 * C * 2 * sizeof(float);
    const unsigned grid2 = (unsigned)std::min<long long>(rg.total_slabs, (long long)num_sms() * 8);
    gn_stats2_kernel<<<grid2, GN2_THREADS, smem2, st>>>((const __half*)X, stats, rows, C, rg);
    STAR_LAUNCH_CHECK("gn_stats2");
    gn_finalize_kernel<<<1, 256, 0, st>>>(stats, (const __half*)gamma, (const __half*)beta, ab, rows, C, eps);
    STAR_LAUNCH_CHECK("gn_finalize");
    auto log2_exact = [](int q) { int s = 0; while ((1 << s) < q) ++s; return (1 << s) == q ? s : -1; };
    // the scales F.interpolate computes (fp32 source / destination sizes), here on the host: device division is approximate
    const float tscale = split ? (float)(Tl - 1) / (float)(T - 1) : (float)Tl / (float)T;
    GnModGeom gm{T, H, W, Tl, Hl, Wl, split ? 1 : 0, log2_exact(H / Hl), log2_exact(W / Wl), tscale, (float)Hl / (float)H,
                 (float)Wl / (float)W};
    gn_apply_mod_kernel<<<grid2, GN2_THREADS, 0, st>>>((const __half*)X, ab, (const __half*)Ymod, (const __half*)Bmod,
                                                       ldmod, (__half*)out, rows, C, silu, rg, gm);
    STAR_LAUNCH_CHECK("gn_apply_mod");
    return 0;
}

int star_layernorm(const void* X, const void* gamma, const void* beta, void* out, long long rows, int C, float eps,
                   int gate_mode, const void* gate, float w0, float w1, void* stream) {
    if (C % 8 || C / 8 > 32 * 12) return fail("star_layernorm: unsupported C=%d", C);
    if (C == 320 || C == 640) {
        const int rpw = C == 320 ? 4 : 2;
        const long long groups = (rows + rpw - 1) / rpw;
        const unsigned g2 = (unsigned)std::min<long long>((groups + 7) / 8, (long long)num_sms() * 6);
        if (C == 320)
            layernorm_sub_kernel<8><<<g2, 256, 0, (cudaStream_t)stream>>>((const __half*)X, (const __half*)gamma, (const __half*)beta,
                                                                          (__half*)out, rows, eps, gate_mode, (const __half*)gate, w0, w1);
        else
            layernorm_sub_kernel<16><<<g2, 256, 0, (cudaStream_t)stream>>>((const __half*)X, (const __half*)gamma, (const __half*)beta,
                                                                           (__half*)out, rows, eps, gate_mode, (const __half*)gate, w0, w1);
        STAR_LAUNCH_CHECK("layernorm_sub");
        return 0;
    }
    const int wpb = 8;
    const long long want = (rows + wpb - 1) / wpb;
    const unsigned grid = (unsigned)std::min<long long>(want, (long long)num_sms() * 6);
    const int oct = (C / 8 + 31) / 32;
#define STAR_LN_LAUNCH(N)                                                                                          \
    layernorm_kernel<N><<<grid, wpb * 32, 0, (cudaStream_t)stream>>>((const __half*)X, (const __half*)gamma,          \
                                                                     (const __half*)beta, (__half*)out, rows, C, eps, \
                                                                     gate_mode, (const __half*)gate, w0, w1)
    if (oct <= 2) STAR_LN_LAUNCH(2);
    else if (oct <= 3) STAR_LN_LAUNCH(3);
    else if (oct <= 5) STAR_LN_LAUNCH(5);
    else STAR_LN_LAUNCH(12);
#undef STAR_LN_LAUNCH
    STAR_LAUNCH_CHECK("layernorm");
    return 0;
}

int star_liem_spatial_gate(const void* X, const void* w98, void* mm_ws, void* gate, int BT, int H, int W, int C,
                           long long r0, long long n, void* stream) {
    if (C % 8) return fail("star_liem_spatial_gate: C must be a multiple of 8");
    cudaStream_t st = (cudaStream_t)stream;
    const long long rows = (long long)BT * H * W;
    if (r0 < 0 || n < 0 || r0 + n > rows) return fail("star_liem_spatial_gate: tokens [%lld, %lld) outside the clip's %lld", r0, r0 + n, rows);
    if (n == 0) return 0;
    if (X) {
        liem_reduce_kernel<<<(unsigned)std::min<long long>((n + 7) / 8, (long long)num_sms() * 8), 256, 0, st>>>(
            (const __half*)X, (__half*)mm_ws + 2 * r0, n, C);
        STAR_LAUNCH_CHECK("liem_reduce");
    }
    if (!gate) return 0;
    if (r0 == 0 && n == rows) {
        liem_conv7_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>((const __half*)mm_ws, (const __half*)w98, (__half*)gate,
                                                                           BT, H, W);
        STAR_LAUNCH_CHECK("liem_conv7");
    } else {
        liem_conv7_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const __half*)mm_ws, (const __half*)w98,
                                                                             (__half*)gate, H, W, r0, n);
        STAR_LAUNCH_CHECK("liem_conv7_rows");
    }
    return 0;
}

int star_row_gate(const void* X, void* out, long long rows, int C, int mode, const void* gate, float w0, float w1,
                  void* stream) {
    if (C % 8) return fail("star_row_gate: C must be a multiple of 8");
    if (mode != 1 && mode != 2) return fail("star_row_gate: mode must be 1 (external gate) or 2 (temporal LIEM)");
    const unsigned grid = (unsigned)std::min<long long>((rows + 7) / 8, (long long)num_sms() * 8);
    row_gate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)X, (__half*)out, rows, C, mode, (const __half*)gate, w0, w1);
    STAR_LAUNCH_CHECK("row_gate");
    return 0;
}

int star_qk_ln_rope(void* QKV, long long ld, long long rows, int heads, int koff, const void* qg, const void* qb,
                    const void* kg, const void* kb, const void* cos_f32, const void* sin_f32, int seq, int text_len,
                    float eps, void* stream) {
    if (ld % 8 || koff % 8) return fail("star_qk_ln_rope: ld and koff must be multiples of 8");
    const long long threads = rows * heads * 2 * 8;
    qk_ln_rope_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (__half*)QKV, ld, rows, heads, koff, (const __half*)qg, (const __half*)qb, (const __half*)kg, (const __half*)kb,
        (const float*)cos_f32, (const float*)sin_f32, seq, text_len, eps);
    STAR_LAUNCH_CHECK("qk_ln_rope");
    return 0;
}

int star_concat_add(const void* a, int Ca, const void* b, const void* c, int Cb, void* out, long long rows,
                    void* stream) {
    if (Ca % 8 || Cb % 8) return fail("star_concat_add: channel counts must be multiples of 8");
    const long long n = rows * ((Ca + Cb) / 8);
    concat_add_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)a, Ca, (const __half*)b,
                                                                           (const __half*)c, Cb, (__half*)out, rows);
    STAR_LAUNCH_CHECK("concat_add");
    return 0;
}

int star_add(const void* a, const void* b, void* out, long long n, void* stream) {
    if (n % 8) return fail("star_add: n must be a multiple of 8");
    add_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)a, (const __half*)b, (__half*)out, n / 8);
    STAR_LAUNCH_CHECK("add");
    return 0;
}

int star_time_avgpool2(const void* X, void* out, int T, long long HW, int C, void* stream) {
    if (C % 8) return fail("star_time_avgpool2: C must be a multiple of 8");
    if (T < 2) return fail("star_time_avgpool2: needs at least two frames");
    const long long per8 = HW * C / 8;
    const int To = (T & 1) ? (T + 1) / 2 : T / 2;
    time_avgpool2_kernel<<<grid_for(per8 * To, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)X, (__half*)out, T, per8);
    STAR_LAUNCH_CHECK("time_avgpool2");
    return 0;
}

int star_upsample2x(const void* X, void* out, int BT, int H, int W, int C, int crop_rows, void* stream) {
    if (C % 8) return fail("star_upsample2x: C must be a multiple of 8");
    if (crop_rows != 0 && crop_rows != 1) return fail("star_upsample2x: crop_rows must be 0 or 1");
    const long long n = (long long)BT * (2 * H - 2 * crop_rows) * (2 * W) * (C / 8);
    upsample2x_crop_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)X, (__half*)out, BT, H, W, C, crop_rows);
    STAR_LAUNCH_CHECK("upsample2x");
    return 0;
}

int star_upsample2x_crop(const void* X, void* out, int BT, int H, int W, int C, void* stream) {
    return star_upsample2x(X, out, BT, H, W, C, 1, stream);
}

int star_softmax_rows(void* S, long long ld, long long rows, int cols, int ctas_per_row, void* stream) {
    STAR_CHECK_INIT();
    if (rows <= 0) return 0;
    if (ld % 8 || reinterpret_cast<uintptr_t>(S) % 16) return fail("star_softmax_rows: rows must be 16-byte aligned (ld %% 8 == 0)");
    if (cols <= 0 || cols > ld) return fail("star_softmax_rows: need 0 < cols <= ld");
    if (ctas_per_row < 1 || ctas_per_row > 8) return fail("star_softmax_rows: ctas_per_row=%d outside [1, 8], the portable cluster size", ctas_per_row);
    if (cols > ctas_per_row * SOFTMAX_SEG_MAX)
        return fail("star_softmax_rows: %d columns do not fit in shared memory (%d CTAs of %d columns per row)", cols,
                    ctas_per_row, SOFTMAX_SEG_MAX);
    if (rows * ctas_per_row > 0x7fffffffll) return fail("star_softmax_rows: too many rows");
    // segments of a multiple of 8 columns keep every CTA's 128-bit loads aligned, and stay <= SOFTMAX_SEG_MAX (one too)
    const int seg = ((cols + ctas_per_row - 1) / ctas_per_row + 7) / 8 * 8;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)ctas_per_row;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)(rows * ctas_per_row));
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = (size_t)seg * 2;
    cfg.stream = (cudaStream_t)stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    STAR_CUDA(cudaLaunchKernelEx(&cfg, softmax_rows_kernel, (__half*)S, ld, cols, seg));
    STAR_LAUNCH_CHECK("softmax_rows");
    return 0;
}

int star_vae_head(const void* X, long long ldx, const void* W27, const void* bias3, void* out, int B, int T,
                  long long HW, void* stream) {
    if (ldx < 3) return fail("star_vae_head: ldx must be >= 3");
    const long long n = (long long)B * T * HW;
    vae_head_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)X, ldx, (const __half*)W27,
                                                                        (const __half*)bias3, (__half*)out, B, T, HW);
    STAR_LAUNCH_CHECK("vae_head");
    return 0;
}

int star_nchw5_to_tokens(const void* x_f32, void* out, int B, int C, int F, long long HW, void* stream) {
    const long long n = (long long)B * F * HW;
    nchw5_to_tokens_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x_f32, (__half*)out, B, C, F, HW);
    STAR_LAUNCH_CHECK("nchw5_to_tokens");
    return 0;
}

int star_tokens_to_nchw5(const void* x, long long ldx, void* out, int B, int C, int F, long long HW, void* stream) {
    const long long n = (long long)B * F * HW;
    tokens_to_nchw5_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, ldx, (__half*)out, B, C, F, HW);
    STAR_LAUNCH_CHECK("tokens_to_nchw5");
    return 0;
}

int star_bilinear_pad(const void* x_f32, void* out_f32, long long NC, int h, int w, int H, int W, int pad_l, int pad_r,
                      int pad_t, int pad_b, float pad_value, void* stream) {
    if (NC <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || pad_l < 0 || pad_r < 0 || pad_t < 0 || pad_b < 0)
        return fail("star_bilinear_pad: bad geometry");
    const int Hp = H + pad_t + pad_b, Wp = W + pad_l + pad_r;
    const long long n = NC * Hp * Wp;
    bilinear_pad_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x_f32, (float*)out_f32, NC, h, w, H, W,
                                                                            pad_l, pad_t, Hp, Wp, (float)h / (float)H,
                                                                            (float)w / (float)W, pad_value);
    STAR_LAUNCH_CHECK("bilinear_pad");
    return 0;
}

long long star_adain_workspace_bytes(int C, int F) { return (long long)C * F * 2 * 2 * 8; }

int star_adain_color_fix(const void* video_f32, const void* source_f32, void* out_f32, void* out_u8, int C, int F, long long HW,
                         long long src_hw, void* workspace, void* stream) {
    if (C < 1 || C > 4 || F < 1 || HW < 2 || src_hw < 2) return fail("star_adain_color_fix: bad geometry (C <= 4)");
    if ((out_f32 == nullptr) == (out_u8 == nullptr)) return fail("star_adain_color_fix: pass exactly one of out_f32 / out_u8");
    // plane_stats_kernel runs one grid row per (channel, frame) plane: gridDim.y = C * F
    if ((long long)C * F > 65535) return fail("star_adain_color_fix: C * F = %lld planes exceed the 65535 grid rows of the statistics launch", (long long)C * F);
    cudaStream_t st = (cudaStream_t)stream;
    double* tgt = (double*)workspace;
    double* src = tgt + (size_t)C * F * 2;
    STAR_CUDA(cudaMemsetAsync(workspace, 0, (size_t)star_adain_workspace_bytes(C, F), st));
    const unsigned gt = (unsigned)std::min<long long>((HW + 255) / 256, 256), gs = (unsigned)std::min<long long>((src_hw + 255) / 256, 256);
    plane_stats_kernel<<<dim3(gt, C * F), 256, 0, st>>>((const float*)video_f32, HW, 1, tgt);
    STAR_LAUNCH_CHECK("plane_stats(target)");
    plane_stats_kernel<<<dim3(gs, C * F), 256, 0, st>>>((const float*)source_f32, src_hw, 0, src);
    STAR_LAUNCH_CHECK("plane_stats(source)");
    adain_apply_kernel<<<dim3((unsigned)std::min<long long>((HW + 255) / 256, 1024), F), 256, 0, st>>>(
        (const float*)video_f32, (float*)out_f32, (unsigned char*)out_u8, C, F, HW, src_hw, tgt, src);
    STAR_LAUNCH_CHECK("adain_apply");
    return 0;
}

long long star_cfg_x0_workspace_bytes(int samples) { return (long long)samples * 4 * 8; }

int star_cfg_x0(const void* y_out, const void* u_out, const void* xt_f32, void* x0_f32, void* guided_out,
                float guide_scale, float guide_rescale, const void* alpha_f32, const void* sigma_f32, int samples,
                long long per_sample, void* workspace, void* stream) {
    if (samples <= 0 || per_sample <= 1) return fail("star_cfg_x0: empty problem");
    if (samples > 65535) return fail("star_cfg_x0: too many samples");
    cudaStream_t st = (cudaStream_t)stream;
    const int has_rescale = guide_rescale >= 0.f;
    double* stats = (double*)workspace;
    const unsigned gx = (unsigned)std::min<long long>((per_sample + 255) / 256, (long long)num_sms() * 8);
    if (has_rescale) {
        if (!workspace) return fail("star_cfg_x0: the std-ratio rescale needs a workspace");
        STAR_CUDA(cudaMemsetAsync(stats, 0, (size_t)samples * 4 * 8, st));
        cfg_stats_kernel<<<dim3(gx, samples), 256, 0, st>>>((const __half*)y_out, (const __half*)u_out, guide_scale, per_sample, stats);
        STAR_LAUNCH_CHECK("cfg_stats");
    }
    cfg_x0_kernel<<<dim3(gx, samples), 256, 0, st>>>((const __half*)y_out, (const __half*)u_out, (const float*)xt_f32,
                                                     (float*)x0_f32, (__half*)guided_out, guide_scale, guide_rescale,
                                                     has_rescale, (const float*)alpha_f32, (const float*)sigma_f32, per_sample, stats);
    STAR_LAUNCH_CHECK("cfg_x0");
    return 0;
}

int star_cfg_x0_blend(const void* y_out, const void* u_out, const void* xt_f32, void* acc_f32, float guide_scale,
                      float guide_rescale, const void* alpha_f32, const void* sigma_f32, const void* wy_f32, const void* wx_f32,
                      int samples, int C, int Ft, int th, int tw, int F, int H, int W, int f0, int lo, int hi, int r0, int c0,
                      void* workspace, void* stream) {
    if (!y_out || !u_out || !xt_f32 || !acc_f32 || !alpha_f32 || !sigma_f32 || !wy_f32 || !wx_f32)
        return fail("star_cfg_x0_blend: null pointer");
    if (samples <= 0 || samples > 65535) return fail("star_cfg_x0_blend: samples=%d outside [1, 65535]", samples);
    if (C < 1 || Ft < 1 || th < 1 || tw < 1) return fail("star_cfg_x0_blend: empty tile %dx%dx%dx%d", C, Ft, th, tw);
    if (f0 < 0 || r0 < 0 || c0 < 0 || (long long)f0 + Ft > F || (long long)r0 + th > H || (long long)c0 + tw > W)
        return fail("star_cfg_x0_blend: window frames [%d, %lld) rows [%d, %lld) cols [%d, %lld) outside the clip %dx%dx%d",
                    f0, (long long)f0 + Ft, r0, (long long)r0 + th, c0, (long long)c0 + tw, F, H, W);
    if (lo < 0 || hi > Ft || lo >= hi) return fail("star_cfg_x0_blend: kept frames [%d, %d) outside the tile's %d", lo, hi, Ft);
    // tile offsets are 32-bit in the kernel; clip offsets 64-bit
    const long long per_sample = (long long)C * Ft * th * tw;
    if (per_sample <= 1 || per_sample >= (1ll << 31)) return fail("star_cfg_x0_blend: %lld elements per tile sample outside [2, 2^31)", per_sample);
    const double clip = (double)samples * C * F * H * W;
    if (clip >= 9.0e18) return fail("star_cfg_x0_blend: clip of %.3g elements exceeds 64-bit indexing", clip);
    if (((uintptr_t)y_out | (uintptr_t)u_out) % 2 || ((uintptr_t)xt_f32 | (uintptr_t)acc_f32 | (uintptr_t)alpha_f32 |
                                                      (uintptr_t)sigma_f32 | (uintptr_t)wy_f32 | (uintptr_t)wx_f32) % 4)
        return fail("star_cfg_x0_blend: misaligned pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int has_rescale = guide_rescale >= 0.f;
    double* stats = (double*)workspace;
    if (has_rescale) {
        if (!workspace) return fail("star_cfg_x0_blend: the std-ratio rescale needs a workspace");
        const unsigned gs = (unsigned)std::min<long long>((per_sample + 255) / 256, (long long)num_sms() * 8);
        STAR_CUDA(cudaMemsetAsync(stats, 0, (size_t)samples * 4 * 8, st));
        cfg_stats_kernel<<<dim3(gs, samples), 256, 0, st>>>((const __half*)y_out, (const __half*)u_out, guide_scale, per_sample, stats);
        STAR_LAUNCH_CHECK("cfg_stats");
    }
    const long long kept = (long long)C * (hi - lo) * th * tw;
    const unsigned gx = (unsigned)std::min<long long>((kept + 255) / 256, (long long)num_sms() * 8);
    CfgBlendGeom q{C, Ft, th, tw, lo, hi, F, H, W, f0, r0, c0};
    cfg_x0_blend_kernel<<<dim3(gx, samples), 256, 0, st>>>((const __half*)y_out, (const __half*)u_out, (const float*)xt_f32,
                                                           (float*)acc_f32, guide_scale, guide_rescale, has_rescale,
                                                           (const float*)alpha_f32, (const float*)sigma_f32, (const float*)wy_f32,
                                                           (const float*)wx_f32, q, stats);
    STAR_LAUNCH_CHECK("cfg_x0_blend");
    return 0;
}

int star_sinusoidal(const void* t_i64, void* out, int B, int dim, void* stream) {
    const int n = B * (dim / 2);
    sinusoidal_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>((const long long*)t_i64, (__half*)out, B, dim);
    STAR_LAUNCH_CHECK("sinusoidal");
    return 0;
}

int star_silu(const void* x, void* out, long long n, void* stream) {
    silu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)out, n);
    STAR_LAUNCH_CHECK("silu");
    return 0;
}

}  // extern "C"
