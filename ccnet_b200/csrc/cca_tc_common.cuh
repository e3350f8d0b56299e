// Pieces shared by the wgmma statistics, forward and backward kernels (channels-last; fp32 I/O as a bf16x3 split, or bf16 or
// f16 I/O).
#pragma once
#include <initializer_list>
#include <mutex>
#include <type_traits>
#include <utility>

#include "cca_common.cuh"
#include "cca_items.cuh"
#include "cca_sm90.cuh"

namespace cca {
namespace tc {
using namespace sm90;

constexpr int kNC = 64;   // channels per chunk (forward ring slot = [LK px][64 ch] fp32 = two swizzled TMA tiles; the backward's
                          // ring slots are one tile, cca_tc_bwd.cuh)

// Thread layout of the attention kernels (three warpgroups):
//   warpgroup 0           : TMA producer (one elected lane of warp 0), the rest idle
//   warpgroups 1, 2       : consumers.  Consumer warpgroup w owns query rows [64w, 64w + 64) of an item's 128-row tile in
//                           the wgmma accumulator layout; both convert fp32 tiles to bf16 operand planes together (256 threads)
constexpr int kThreads = 384;
constexpr int kConsumers = 256;
constexpr int kBarConsumers = 1;   // named barrier of the 256 consumer threads
constexpr int kBarConvert = 2;     // named barrier inside a conversion
// Register split (setmaxnreg): the producer warpgroup only runs one TMA lane, so it gives its registers to the consumers.  The
// kernels are launched with 168 registers per thread (384 threads, one CTA per SM); the split must fit that same pool.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(128 * kProducerRegs + kConsumers * kConsumerRegs <= kThreads * 168, "register split exceeds the launch allocation");

// I/O element type E of the kernels:
//   float        : fp32 I/O, every operand split into bf16 hi + lo (3 bf16 MMAs per product).
//   __nv_bfloat16: bf16 I/O, operands used as they are (1 MMA per product); a 64-channel chunk is ONE 128-byte-wide TMA tile.
//   __half       : f16 I/O, the layout of bf16 I/O with f16 MMAs and f16 packing of P, dS and the staged outputs.
template <typename E> constexpr bool kH16 = sizeof(E) == 2;                      // 16-bit I/O (bf16 or f16)
template <typename E> constexpr bool kF16 = std::is_same<E, __half>::value;
template <typename E> constexpr int kDtype = kF16<E> ? CCA_F16 : (kH16<E> ? CCA_BF16 : CCA_F32);
template <int LK, typename E> struct Tiles {
    static constexpr bool H16 = kH16<E>;
    static constexpr int kTile = LK * 128;             // [LK px][128 B] = 32 fp32 or 64 bf16 / f16 channels, SWIZZLE_128B
    static constexpr int kSlot = H16 ? kTile : 2 * kTile;  // 64 channels
    static constexpr int kPlane = LK * 16;             // operand plane: LK rows x 16 B (8 bf16)
    // fp32 I/O: a converted slot holds its 8-channel planes as  hi0 lo0 hi1 lo1 ... hi7 lo7  (each 32-channel TMA box is rewritten
    // inside its own bytes, so the two boxes of a slot are converted by two independent thread groups)
    static constexpr int kPStride = 2 * kPlane;        // hi plane p -> hi plane p+1 (and lo -> lo)
    static constexpr int kLoOff = kPlane;              // hi plane p -> lo plane p
    static constexpr int kTerms = H16 ? 1 : 2;         // operand copies kept: hi (+ lo)
    static constexpr int kOp = kTerms * 8 * kPlane;    // 8 planes = 64 channels, per copy
    static constexpr int kPP = LK / 8;                 // planes of a [LK x LK] pixel-pixel matrix (P, dS)
    static constexpr int kP = kTerms * kPP * kPlane;
};

__device__ __forceinline__ uint32_t pack_bf16(float a, float b)
{
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // low half = a, high half = b
    return r;
}
// (a, b) -> packed bf16 hi pair and lo pair, x = hi + lo up to ~2^-17 |x|
__device__ __forceinline__ void split2(float a, float b, uint32_t &hi, uint32_t &lo)
{
    hi = pack_bf16(a, b);
    const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xFFFF0000u);
    lo = pack_bf16(a - ah, b - bh);
}
__device__ __forceinline__ void split8(const float *v, uint4 &hi, uint4 &lo)
{
    split2(v[0], v[1], hi.x, lo.x); split2(v[2], v[3], hi.y, lo.y);
    split2(v[4], v[5], hi.z, lo.z); split2(v[6], v[7], hi.w, lo.w);
}
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
// the same for a 16-bit operand type (F16: f16, else bf16): (a, b) -> packed pair (low half = a), and the halves back
template <bool F16> __device__ __forceinline__ uint32_t pack2(float a, float b)
{
    if constexpr (F16) {
        uint32_t r;
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
        return r;
    } else {
        return pack_bf16(a, b);
    }
}
template <bool F16> __device__ __forceinline__ float lo2(uint32_t w)
{
    if constexpr (F16) return __half2float(__ushort_as_half((unsigned short)(w & 0xFFFFu)));
    else return bf_lo(w);
}
template <bool F16> __device__ __forceinline__ float hi2(uint32_t w)
{
    if constexpr (F16) return __half2float(__ushort_as_half((unsigned short)(w >> 16)));
    else return bf_hi(w);
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void consumers_sync() { named_bar_sync(kBarConsumers, kConsumers); }

// Conversion of one staged slot (NB swizzled 32-channel fp32 TMA boxes: [LK px][64 ch] for NB = 2, [LK px][32 ch] for NB = 1)
// into bf16 hi/lo operand planes [8-channel chunk][pixel][16 B], IN PLACE, by the 256 consumer threads (thread t: pixel row
// t & 127, 16-channel half t >> 7 of each box).  Every thread reads its NB x 64 B, the consumers meet, then overwrite; the
// planes are made visible to wgmma (async proxy) and every consumer has passed the closing barrier on return.
// With `dot` (the O tile of the same pixels, same layout): returns this thread's part of sum_c slot[r][c] * dot[r][c].
// With `src` (fp32): box bx is read from src[bx] instead, and `slot` is only the destination of the NB converted boxes (NB = 4:
// two [LK px][64 ch] slots back to back).
// 16-bit slots (one 64-channel box) need no conversion; only the dot product is computed.
template <int LK, typename E, int NB = 2>
__device__ __forceinline__ float convert_slot(uint8_t *slot, int t, const uint8_t *dot = nullptr, const uint8_t *const *src = nullptr)
{
    using T = Tiles<LK, E>;
    constexpr bool H16 = T::H16, F16 = kF16<E>;
    const int r = t & 127, hq = t >> 7;
    const int rr = r < LK ? r : LK - 1, sw = rr & 7;
    float acc = 0.f;
    if constexpr (H16) {
        if (dot) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = (hq * 4 + j) ^ sw;
                const uint4 x = *reinterpret_cast<const uint4 *>(slot + rr * 128 + c * 16);
                const uint4 y = *reinterpret_cast<const uint4 *>(dot + rr * 128 + c * 16);
                const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) acc += lo2<F16>(xw[e]) * lo2<F16>(yw[e]) + hi2<F16>(xw[e]) * hi2<F16>(yw[e]);
            }
        }
        return r < LK ? acc : 0.f;
    } else {
        static_assert(NB == 1 || NB == 2 || NB == 4, "boxes per slot");
        float4 raw[4 * NB];
#pragma unroll
        for (int bx = 0; bx < NB; ++bx)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                raw[4 * bx + j] = *reinterpret_cast<const float4 *>((src ? src[bx] : slot + bx * T::kTile) + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
        if (dot) {
#pragma unroll
            for (int bx = 0; bx < NB; ++bx)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 o = *reinterpret_cast<const float4 *>(dot + bx * T::kTile + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
                    const float4 x = raw[4 * bx + j];
                    acc += x.x * o.x + x.y * o.y + x.z * o.z + x.w * o.w;
                }
        }
        named_bar_sync(kBarConvert, kConsumers);
        if (r < LK) {
#pragma unroll
            for (int bx = 0; bx < NB; ++bx) {
                uint8_t *d = slot + bx * T::kTile + r * 16 + hq * 2 * T::kPStride;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const float4 a = raw[4 * bx + 2 * j], b = raw[4 * bx + 2 * j + 1];
                    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                    uint4 hi, lo;
                    split8(v, hi, lo);
                    *reinterpret_cast<uint4 *>(d + j * T::kPStride) = hi;
                    *reinterpret_cast<uint4 *>(d + j * T::kPStride + T::kLoOff) = lo;
                }
            }
        }
        fence_proxy_async();
        consumers_sync();
        return r < LK ? acc : 0.f;
    }
}

// Operand descriptors of a [LK px][64 ch] slot (16-bit tile or fp32 planes; `lo`: the lo planes), 16-element k-step ks.  A
// one-box fp32 slot ([LK px][32 ch], converted with NB = 1) has the layout of the first half of a two-box slot: the same
// descriptors serve it with ks < 2 (K-major) or N = 32 (MN-major).
//   channels as the contraction (K-major, rows = pixels starting at row0)
template <int LK, typename E> __device__ __forceinline__ uint64_t desc_kmaj(uint32_t slot, int row0, int ks, bool lo)
{
    using T = Tiles<LK, E>;
    if constexpr (T::H16) return smem_desc(slot + row0 * 128 + ks * 32, 16, 1024, kSw128);
    else return smem_desc(slot + row0 * 16 + ks * 2 * T::kPStride + (lo ? T::kLoOff : 0), T::kPStride, 128);
}
//   pixels as the contraction (MN-major: the 64 channels are the N dimension)
template <int LK, typename E> __device__ __forceinline__ uint64_t desc_mnmaj(uint32_t slot, int ks, bool lo)
{
    using T = Tiles<LK, E>;
    if constexpr (T::H16) return smem_desc(slot + ks * 2048, 16, 1024, kSw128);
    else return smem_desc(slot + ks * 256 + (lo ? T::kLoOff : 0), 128, T::kPStride);
}

// ---- host: TMA tensor maps over channels-last tensors -------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeFn get_encode()
{
    static EncodeFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        cudaDriverEntryPointQueryResult qr;
        void *p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeFn>(p);
    });
    return fn;
}
// NHWC tensor [B,H,W,C] of cca_dtype `dtype`; box = [128 bytes of channels] x [LK pixels along W (row pass) or H (column
// pass)].  The map's element type is also the arithmetic type of the TMA reduce-adds through it.
inline bool make_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int LK, bool col, int dtype)
{
    EncodeFn enc = get_encode();
    if (!enc) return false;
    const bool h16 = dtype != CCA_F32;
    const cuuint64_t es_bytes = h16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * es_bytes, (cuuint64_t)W * C * es_bytes, (cuuint64_t)H * W * C * es_bytes};
    cuuint32_t box[4] = {h16 ? 64u : 32u, col ? 1u : (cuuint32_t)LK, col ? (cuuint32_t)LK : 1u, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    const CUtensorMapDataType et = dtype == CCA_F16    ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                   : dtype == CCA_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                       : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    return enc(m, et, 4, const_cast<void *>(base), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// LK template (padded tile length) for the longest tile of a problem
inline int lk_for(int tile) { return tile <= 80 ? 80 : (tile <= 112 ? 112 : 0); }
// f(std::integral_constant<int, LK>{}): the LK instantiation that serves the lines of d
template <typename F> decltype(auto) with_tile(Dims d, F &&f)
{
    if (lk_for(max_tile(make_space(d.B, d.H, d.W))) == 80) return f(std::integral_constant<int, 80>{});
    return f(std::integral_constant<int, 112>{});
}
// f(E{}, std::integral_constant<int, LK>{}): the instantiation that serves `dtype` on the lines of d
template <typename F> decltype(auto) with_elem_tile(int dtype, Dims d, F &&f)
{
    return with_elem(dtype, [&](auto e) { return with_tile(d, [&](auto lk) { return f(e, lk); }); });
}
// Cached tensor maps (cca_tc_host.cu): encoding costs ~1 us of driver time per map and an op call needs 8-15 of them;
// a map only depends on (base, shape, box, dtype), so it stays valid for as long as that address holds such a tensor.
bool get_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int LK, bool col, int dtype);
// One tensor of a launch: [B, H, W, C] at base, boxes of box_col pixels down a column and box_row pixels along a row
struct MapSpec {
    const void *base;
    int B, C, box_col, box_row;
};
// m[2t], m[2t + 1]: the column and row maps of tensor t (H, W from d); cudaErrorInvalidValue and *why set if one fails
cudaError_t get_maps(CUtensorMap *m, std::initializer_list<MapSpec> tensors, Dims d, int dtype, const char **why);
// SM count of the CURRENT device (cached per device id)
int sm_count();
// One launch: sets the kernel's dynamic shared memory limit when it uses any, lets it start ahead of the previous launch on
// the stream (programmatic dependent launch; the kernel waits with griddepcontrol.wait) when `pdl` and tc_pdl() are on,
// and counts it.
template <typename... Params, typename... Args>
cudaError_t launch_kernel(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, bool pdl, cudaStream_t st, Args &&...args)
{
    cudaError_t e;
    if (smem > 0 && (e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
        return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl && tc_pdl() ? 1 : 0;
    e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}
// persistent item kernels: one CTA per SM, fewer if there are fewer items
inline int item_grid(const ItemSpace &sp)
{
    const int sms = sm_count();
    return sp.total < sms ? sp.total : sms;
}
// dst[t] = sum of the nparts planes [nparts][n[t]] at src[t], added in plane order, for count <= 3 tensors; launched with
// programmatic dependent launch after the kernel that writes the planes (cca_tc_det.cu)
cudaError_t planes_sum(const float *const *src, float *const *dst, const long *n, int count, int nparts, cudaStream_t st);

// ---- workspace layouts: each computes its buffers' places once, for the op that carves them and (base nullptr) for the
// size query.  Sizes are part of the C ABI (callers allocate by them) and must not change.
inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
template <typename T> T *ws_at(void *base, size_t off) { return reinterpret_cast<T *>(reinterpret_cast<uintptr_t>(base) + off); }
// forward (2D, and the 3D op on the frames view with extra_parts = 1 for its time plane): [nparts + extra_parts][B*H*W] fp32
// partial lse planes, then [B] per-sample counters of the values kernel, each rounded up to 16 bytes; the planes-mode
// buffers (planes_ws) follow at `planes`
struct FwdWs {
    float *parts;
    unsigned int *cdone;
    void *planes;
    size_t bytes;
};
inline FwdWs fwd_ws(Dims d, int extra_parts, void *base)
{
    const size_t npix = (size_t)d.B * d.H * d.W;
    const size_t parts = align16((make_space(d.B, d.H, d.W).nparts + extra_parts) * npix * sizeof(float));
    const size_t bytes = parts + align16((size_t)d.B * sizeof(unsigned int));
    return {ws_at<float>(base, 0), ws_at<unsigned int>(base, parts), ws_at<void>(base, bytes), bytes};
}
// backward (2D, and the 3D op on the frames view): delta [B*H*W] fp32, then [3*B] per-sample counters, each rounded up to
// 16 bytes; the planes-mode buffers follow at `planes`
struct BwdWs {
    float *delta;
    unsigned int *counters;
    void *planes;
    size_t bytes;
};
inline BwdWs bwd_ws(Dims d, void *base)
{
    const size_t delta = align16((size_t)d.B * d.H * d.W * sizeof(float));
    const size_t bytes = delta + align16(3 * (size_t)d.B * sizeof(unsigned int));
    return {ws_at<float>(base, 0), ws_at<unsigned int>(base, delta), ws_at<void>(base, bytes), bytes};
}
// planes mode (deterministic, tiled lines): one [nparts*B, H, W, c] fp32 plane buffer per entry of `channels`, each at a
// 256-byte boundary (TMA needs 16) from `at` rounded up to 256; the extra 256 bytes pay for that rounding
struct PlanesWs {
    float *p[3];
    size_t bytes;
};
inline PlanesWs planes_ws(Dims d, std::initializer_list<int> channels, void *at)
{
    const size_t per = (size_t)make_space(d.B, d.H, d.W).nparts * d.B * d.H * d.W * sizeof(float);
    void *base = reinterpret_cast<void *>(align256(reinterpret_cast<uintptr_t>(at)));
    PlanesWs w = {};
    size_t off = 0;
    int i = 0;
    for (int c : channels) {
        w.p[i++] = ws_at<float>(base, off);
        off += align256(per * c);
    }
    w.bytes = off + 256;
    return w;
}
// attention-map backward: rho [B*H*W] fp32 rounded up to 256 bytes, then (det, tiled lines) the dQ and dK planes
struct AttnBwdWs {
    float *rho;
    PlanesWs planes;
    size_t bytes;
};
inline AttnBwdWs attn_bwd_ws(Dims d, bool det, void *base)
{
    const size_t rho = align256((size_t)d.B * d.H * d.W * sizeof(float));
    AttnBwdWs w = {ws_at<float>(base, 0), planes_ws(d, {d.Cq, d.Cq}, ws_at<void>(base, rho)), rho};
    if (det && tc_tiled(d)) w.bytes += w.planes.bytes;
    return w;
}

// the shapes the kernels are written for (no device query)
inline bool shape_fits(Dims d, int dtype)
{
    if (dtype != CCA_F32 && dtype != CCA_BF16 && dtype != CCA_F16) return false;
    if (d.Cq % 16 != 0 || d.Cq > 64 || d.Cq < 16 || d.C % kNC != 0) return false;
    return d.H <= 112 * 8 && d.W <= 112 * 8;                 // cca_items.cuh: at most kMaxNT tiles of kMaxTile pixels per line
}
inline bool shape_supported(Dims d, int dtype) { return shape_fits(d, dtype) && get_encode() != nullptr; }

}  // namespace tc
}  // namespace cca
