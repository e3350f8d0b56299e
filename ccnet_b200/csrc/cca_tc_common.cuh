// Pieces shared by the wgmma statistics, forward and backward kernels (channels-last, fp32 I/O as a bf16x3 split, or bf16 I/O).
#pragma once
#include <mutex>

#include "cca_common.cuh"
#include "cca_sm90.cuh"

namespace cca {
namespace tc {
using namespace sm90;

constexpr int kNC = 64;   // channels per chunk (one ring slot = [LK px][64 ch] fp32 = two swizzled TMA tiles)

// Thread layout of the attention kernels (three warpgroups):
//   warpgroup 0           : TMA producer (one elected lane of warp 0), the rest idle
//   warpgroups 1, 2       : consumers.  Consumer warpgroup w owns query rows [64w, 64w + 64) of an item's 128-row tile in
//                           the wgmma accumulator layout; both convert fp32 tiles to bf16 operand planes together (256 threads)
constexpr int kThreads = 384;
constexpr int kConsumers = 256;
constexpr int kBarConsumers = 1;   // named barrier of the 256 consumer threads
constexpr int kBarConvert = 2;     // named barrier inside a conversion

// BF = false: fp32 I/O, every operand split into bf16 hi + lo (3 MMAs per product).
// BF = true : bf16 I/O, operands used as they are (1 MMA per product); a 64-channel chunk is ONE 128-byte-wide TMA tile.
template <int LK, bool BF = false> struct Tiles {
    static constexpr int kTile = LK * 128;             // [LK px][128 B] = 32 fp32 or 64 bf16 channels, SWIZZLE_128B
    static constexpr int kSlot = BF ? kTile : 2 * kTile; // 64 channels
    static constexpr int kPlane = LK * 16;             // operand plane: LK rows x 16 B (8 bf16)
    // fp32 I/O: a converted slot holds its 8-channel planes as  hi0 lo0 hi1 lo1 ... hi7 lo7  (each 32-channel TMA box is rewritten
    // inside its own bytes, so the two boxes of a slot are converted by two independent thread groups)
    static constexpr int kPStride = 2 * kPlane;        // hi plane p -> hi plane p+1 (and lo -> lo)
    static constexpr int kLoOff = kPlane;              // hi plane p -> lo plane p
    static constexpr int kTerms = BF ? 1 : 2;          // operand copies kept: hi (+ lo)
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

__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void consumers_sync() { named_bar_sync(kBarConsumers, kConsumers); }

// Conversion of one staged slot ([LK px][64 ch] fp32 as two swizzled 32-channel TMA boxes) into bf16 hi/lo operand planes
// [8-channel chunk][pixel][16 B], IN PLACE, by the 256 consumer threads (thread t: pixel row t & 127, 32-channel half t >> 7 of
// the slot, i.e. 16 channels of each box).  Every thread reads its 2 x 64 B, the consumers meet, then overwrite; the planes are
// made visible to wgmma (async proxy) and every consumer has passed the closing barrier on return.
// With `dot` (the O tile of the same pixels, same layout): returns this thread's part of sum_c slot[r][c] * dot[r][c].
// bf16 slots need no conversion; only the dot product is computed.
template <int LK, bool BF>
__device__ __forceinline__ float convert_slot(uint8_t *slot, int t, const uint8_t *dot = nullptr)
{
    using T = Tiles<LK, BF>;
    const int r = t & 127, hq = t >> 7;
    const int rr = r < LK ? r : LK - 1, sw = rr & 7;
    float acc = 0.f;
    if constexpr (BF) {
        if (dot) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = (hq * 4 + j) ^ sw;
                const uint4 x = *reinterpret_cast<const uint4 *>(slot + rr * 128 + c * 16);
                const uint4 y = *reinterpret_cast<const uint4 *>(dot + rr * 128 + c * 16);
                const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) acc += bf_lo(xw[e]) * bf_lo(yw[e]) + bf_hi(xw[e]) * bf_hi(yw[e]);
            }
        }
        return r < LK ? acc : 0.f;
    } else {
        float4 raw[8];
#pragma unroll
        for (int bx = 0; bx < 2; ++bx)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                raw[4 * bx + j] = *reinterpret_cast<const float4 *>(slot + bx * T::kTile + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
        if (dot) {
#pragma unroll
            for (int bx = 0; bx < 2; ++bx)
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
            for (int bx = 0; bx < 2; ++bx) {
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

// Operand descriptors of a [LK px][64 ch] slot (bf16 tile or fp32 planes; `lo`: the lo planes), 16-element k-step ks:
//   channels as the contraction (K-major, rows = pixels starting at row0)
template <int LK, bool BF> __device__ __forceinline__ uint64_t desc_kmaj(uint32_t slot, int row0, int ks, bool lo)
{
    using T = Tiles<LK, BF>;
    if constexpr (BF) return smem_desc(slot + row0 * 128 + ks * 32, 16, 1024, kSw128);
    else return smem_desc(slot + row0 * 16 + ks * 2 * T::kPStride + (lo ? T::kLoOff : 0), T::kPStride, 128);
}
//   pixels as the contraction (MN-major: the 64 channels are the N dimension)
template <int LK, bool BF> __device__ __forceinline__ uint64_t desc_mnmaj(uint32_t slot, int ks, bool lo)
{
    using T = Tiles<LK, BF>;
    if constexpr (BF) return smem_desc(slot + ks * 2048, 16, 1024, kSw128);
    else return smem_desc(slot + ks * 256 + (lo ? T::kLoOff : 0), 128, T::kPStride);
}

// global row stores of the accumulator layout: two consecutive channels per thread
__device__ __forceinline__ void put2(float *p, float a, float b, bool add)
{
    if (add) atomicAdd(reinterpret_cast<float2 *>(p), make_float2(a, b));
    else *reinterpret_cast<float2 *>(p) = make_float2(a, b);
}
__device__ __forceinline__ void put2(__nv_bfloat16 *p, float a, float b, bool add)
{
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    if (add) atomicAdd(reinterpret_cast<__nv_bfloat162 *>(p), v);
    else *reinterpret_cast<__nv_bfloat162 *>(p) = v;
}

// ---- host: TMA tensor maps over channels-last fp32 tensors -------------------------------------
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
// NHWC tensor [B,H,W,C] (fp32 or bf16); box = [128 bytes of channels] x [LK pixels along W (row pass) or H (column pass)]
inline bool make_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int LK, bool col, bool bf16 = false)
{
    EncodeFn enc = get_encode();
    if (!enc) return false;
    const cuuint64_t es_bytes = bf16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * es_bytes, (cuuint64_t)W * C * es_bytes, (cuuint64_t)H * W * C * es_bytes};
    cuuint32_t box[4] = {bf16 ? 64u : 32u, col ? 1u : (cuuint32_t)LK, col ? (cuuint32_t)LK : 1u, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    return enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void *>(base), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// LK template (padded tile length) for the longest tile of a problem
inline int lk_for(int tile) { return tile <= 80 ? 80 : (tile <= 112 ? 112 : 0); }
// Cached tensor maps (cca_tc_host.cu): encoding costs ~1 us of driver time per map and an op call needs 8-15 of them;
// a map only depends on (base, shape, box, dtype), so it stays valid for as long as that address holds such a tensor.
bool get_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int LK, bool col, bool bf16);
// SM count of the CURRENT device (cached per device id)
int sm_count();
inline bool shape_supported(Dims d, int dtype)
{
    if (dtype != CCA_F32 && dtype != CCA_BF16) return false;
    if (d.Cq % 16 != 0 || d.Cq > 64 || d.Cq < 16 || d.C % kNC != 0) return false;
    if (d.H > 112 * 8 || d.W > 112 * 8) return false;        // cca_items.cuh: at most kMaxNT tiles of kMaxTile pixels per line
    return get_encode() != nullptr;
}

}  // namespace tc
}  // namespace cca
