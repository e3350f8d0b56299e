// wgmma / TMA kernels of the criss-cross attention MAP for sm_90a (channels-last q, k): the reference's
//     attn[b,h,w,g] = softmax over g of cat(e_col, e_row)          (cc_attention/functions.py:40, `concate`)
// as an fp32 [B,H,W,H+W] tensor (g < H: column key (g, w), self entry 0; g >= H: row key (h, g - H)), and its gradient
// with respect to q and k.
//
// Forward: the statistics pre-pass (cca_tc_stats.cuh, unchanged) leaves the partial log-sum-exp planes; the map kernel walks
// the same items with the same roles (TMA ring of Q and K tiles, S = Q K^T with wgmma), combines each query row's lse from the
// planes as the values kernel does (combine_lse2) and writes P = exp2(S log2e - lse2) for rows < lq and columns < lk.  An
// item's P tile is exactly one block of the map, so every element is written once: the forward is deterministic.
// The rows of the map are (H+W)*4 bytes apart, which is 16-byte aligned only when (H+W) % 4 == 0, so TMA stores do not fit
// in general; each thread stores its accumulator pairs as float2 (the four threads of a row fill one 32-byte sector).
//
// Backward (the map depends on q and k only):
//     rho[p] = sum_j attn[p,j] dattn[p,j]       (cca_attn_rho_kernel, cca_simt_attn.cu: one warp per pixel, fixed order)
//     dS     = attn * (dattn - rho)             (per item, from the attn / dattn tiles in the accumulator layout)
//     dQ     = dS K      dK = dS^T Q            (the dQ / dK part of cca_tc_bwd.cuh: staging in the K slot / dS planes,
//                                                 TMA reduce-add onto outputs the rho pass cleared)
// One tile per line: every dq / dk element receives exactly two adds onto zero, which commute, so the result is
// bit-reproducible.  Planes mode (PL, fp32, CCA_FLAG_DETERMINISTIC on tiled lines): items STORE dQ into plane
// part_index and dK into plane qtile_part_index of [nparts*B, H, W, Cq] buffers, and planes_sum adds them in plane order.
#pragma once
#include "cca_items.cuh"
#include "cca_tc_common.cuh"
#include "cca_tc_stats.cuh"

namespace cca {
namespace tc {

struct AttnFwdParams {
    ItemSpace sp;
    int Cq;
    long npix;
    const float *parts;   // [nparts][B*H*W] partial log2-sum-exp2 (statistics pre-pass)
    float *attn;          // [B,H,W,H+W]
};

// Final log2-sum-exp2 of pixel `pix` from the statistics pre-pass's partial planes ([nparts][npix]), combined as the values
// kernel combines them (cca_tc_fwd.cuh), so that the map is normalised exactly as `out` is; the first kPre planes are passed
// in already loaded (pv), the rest are read here.
template <int kPre>
__device__ __forceinline__ float combine_lse2(const float *pv, const float *parts, long npix, int nparts, long pix)
{
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < kPre; ++i)
        if (i < nparts) m = fmaxf(m, pv[i]);
    for (int i = kPre; i < nparts; ++i) m = fmaxf(m, __ldcg(parts + (long)i * npix + pix));
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kPre; ++i)
        if (i < nparts) sum += exp2f(pv[i] - m);
    for (int i = kPre; i < nparts; ++i) sum += exp2f(__ldcg(parts + (long)i * npix + pix) - m);
    return m + log2f(sum);
}

// (row, c) and (row, c + 1) of a map row, c even: one float2 when both exist and the pair is 8-byte aligned
__device__ __forceinline__ void store_pair(float *row, int c, int lk, bool a8, float x0, float x1)
{
    if (c + 1 < lk && a8) {
        *reinterpret_cast<float2 *>(row + c) = make_float2(x0, x1);
    } else {
        row[c] = x0;
        if (c + 1 < lk) row[c + 1] = x1;
    }
}
__device__ __forceinline__ float2 load_pair(const float *row, int c, int lk, bool a8)
{
    if (c + 1 < lk && a8) return __ldg(reinterpret_cast<const float2 *>(row + c));
    return make_float2(__ldg(row + c), c + 1 < lk ? __ldg(row + c + 1) : 0.f);
}

// Row length of the map: H + W entries in 2D.  The 3D map (cca_tc_attn3d.cu) runs these kernels on the frames view of a
// clip batch with rows of H + W + T entries, its params type carrying T; the item arithmetic is the same.
__device__ __forceinline__ long map_row(const AttnFwdParams &p) { return (long)p.sp.H + p.sp.W; }

// (the kernels' bodies, shared by the 2D and 3D map kernels)
template <int LK, typename E, typename P>
__device__ __forceinline__ void attn_fwd(const CUtensorMap &mqc, const CUtensorMap &mqr, const CUtensorMap &mkc,
                                         const CUtensorMap &mkr, const P &p)
{
    using T = Tiles<LK, E>;
    using S = StatsSmem<LK, E>;          // the same Q + K ring as the statistics pre-pass
    constexpr bool H16 = kH16<E>, F16 = kF16<E>;
    constexpr int kNS = S::kNS;
    constexpr int TERMS = H16 ? 1 : 3;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + S::off_bar), *empty = full + kNS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KQ = p.Cq / 16;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item(p.sp, (int)blockIdx.x + k * (int)gridDim.x); };

    if (tid == 0) {
        for (int i = 0; i < kNS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumers); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr);
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {                 // q and k are inputs: the loads need not wait for the statistics kernel
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                const int slot = k % kNS;
                mbar_wait(&empty[slot], ((k / kNS) & 1) ^ 1);
                uint8_t *dst = smem + S::off_ld + slot * 2 * T::kSlot;
                mbar_expect_tx(&full[slot], 2 * T::kSlot);
                for (int t = 0; t < 2; ++t) {
                    const CUtensorMap *m = t == 0 ? (it.col ? &mqc : &mqr) : (it.col ? &mkc : &mkr);
                    const int start = t == 0 ? it.q0 : it.k0;
                    const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                    tma_load_4d(dst + t * T::kSlot, m, &full[slot], 0, cw, ch, it.b);
                    if constexpr (!H16) tma_load_4d(dst + t * T::kSlot + T::kTile, m, &full[slot], 32, cw, ch, it.b);
                }
            }
        }
    } else if (tid >= 128) {
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
        const long hw2 = map_row(p);
        const uint32_t ld_base = smem_u32(smem + S::off_ld);
        pdl_wait();                      // the partial planes come from the statistics kernel
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const int slot = k % kNS;
            constexpr int kPre = 4;
            float pv[2][kPre];
            long pix[2];
            bool rok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                rok[h] = r < it.lq;
                pix[h] = item_pixel(p.sp, it, rok[h] ? r : 0);
#pragma unroll
                for (int i = 0; i < kPre; ++i)
                    pv[h][i] = rok[h] && i < p.sp.nparts ? __ldcg(p.parts + (long)i * p.npix + pix[h]) : 0.f;
            }
            mbar_wait(&full[slot], (k / kNS) & 1);
            uint8_t *qs = smem + S::off_ld + slot * 2 * T::kSlot;
            if constexpr (!H16) {
                convert_slot<LK, E>(qs, t);
                convert_slot<LK, E>(qs + T::kSlot, t);
            }
            const uint32_t qb = ld_base + slot * 2 * T::kSlot, kb = qb + T::kSlot;
            float acc[LK / 2];
            wg_fence();
            for (int ks = 0; ks < KQ; ++ks) {
                wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, false), desc_kmaj<LK, E>(kb, 0, ks, false), ks > 0, 0, 0);
                if constexpr (TERMS == 3) {
                    wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, false), desc_kmaj<LK, E>(kb, 0, ks, true), 1, 0, 0);
                    wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, true), desc_kmaj<LK, E>(kb, 0, ks, false), 1, 0, 0);
                }
            }
            wg_commit();
            float nlse[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) nlse[h] = rok[h] ? -combine_lse2<kPre>(pv[h], p.parts, p.npix, p.sp.nparts, pix[h]) : 0.f;
            wg_wait<0>();
            wg_acc_fence<LK / 2>(acc);
            mbar_arrive(&empty[slot]);
            // rows rbase (h = 0), rbase + 8 (h = 1) of this thread, columns 8j + cq + e
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!rok[h]) continue;
                const int self = it.col ? it.q0 + rbase + 8 * h - it.k0 : -1;
                float *row = p.attn + pix[h] * hw2 + (it.col ? 0 : p.sp.H) + it.k0;
                const bool a8 = (reinterpret_cast<uintptr_t>(row) & 7) == 0;
#pragma unroll
                for (int j = 0; j < LK / 8; ++j) {
                    const int c = 8 * j + cq;
                    if (c < it.lk) {
                        const float p0 = c == self ? 0.f : exp2f(fmaf(acc[4 * j + 2 * h], kLog2e, nlse[h]));
                        const float p1 = c + 1 == self ? 0.f : exp2f(fmaf(acc[4 * j + 2 * h + 1], kLog2e, nlse[h]));
                        store_pair(row, c, it.lk, a8, p0, p1);
                    }
                }
            }
        }
    }
}

template <int LK, typename E>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_attn_fwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                       const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr, AttnFwdParams p)
{
    attn_fwd<LK, E>(mqc, mqr, mkc, mkr, p);
}

struct AttnBwdParams {
    ItemSpace sp;
    int Cq;
    const float *attn, *dattn;   // [B,H,W,H+W]
    const float *rho;            // [B,H,W]
};

// Shared memory: the dS planes (hi, lo; dK is staged there), then a ring of Q + K stages (one converted [LK px][64 ch] slot
// each, as in the statistics pre-pass; dQ is staged in the K slot).  A stage goes back to the producer once the dQ copy has
// read it.
template <int LK, typename E> struct AttnBwdSmem {
    using T = Tiles<LK, E>;
    static constexpr int off_p = 0;
    // (pad: 64-row dS^T operands read up to 16 planes; TMA destinations with SWIZZLE_128B must be 1024-byte aligned)
    static constexpr int off_ld = (off_p + T::kP + (16 - LK / 8) * T::kPlane + 1023) / 1024 * 1024;
    static constexpr int kBudget = 232448;
    static constexpr int kFit = (kBudget - off_ld - 1024) / (2 * T::kSlot);
    static constexpr int kNS = kFit < 4 ? kFit : 4;
    static constexpr int off_bar = off_ld + kNS * 2 * T::kSlot;
    static constexpr int kBytes = off_bar + 8 * 2 * kNS;
    static_assert(kNS >= 2, "ring depth");
    static_assert(off_p % 1024 == 0 && T::kP >= T::kSlot, "dK staging in the dS planes");
    static_assert(kBytes <= kBudget, "shared memory budget");
};

__device__ __forceinline__ long map_row(const AttnBwdParams &p) { return (long)p.sp.H + p.sp.W; }

template <int LK, typename E, bool PL, typename P>
__device__ __forceinline__ void attn_bwd(const CUtensorMap &mqc, const CUtensorMap &mqr, const CUtensorMap &mkc,
                                         const CUtensorMap &mkr, const CUtensorMap &mdqc, const CUtensorMap &mdqr,
                                         const CUtensorMap &mdkc, const CUtensorMap &mdkr, const P &p)
{
    using T = Tiles<LK, E>;
    using S = AttnBwdSmem<LK, E>;
    constexpr bool H16 = kH16<E>, F16 = kF16<E>;
    constexpr int TERMS = H16 ? 1 : 3;
    constexpr int kNS = S::kNS;
    constexpr int KP = LK / 16;
    constexpr uint32_t LOP = T::kPP * T::kPlane;   // dS planes: hi block -> lo block
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + S::off_bar), *empty = full + kNS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item(p.sp, (int)blockIdx.x + k * (int)gridDim.x); };

    if (tid == 0) {
        for (int i = 0; i < kNS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr);
        prefetch_tmap(&mdqc); prefetch_tmap(&mdqr); prefetch_tmap(&mdkc); prefetch_tmap(&mdkr);
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                const int slot = k % kNS;
                mbar_wait(&empty[slot], ((k / kNS) & 1) ^ 1);
                uint8_t *dst = smem + S::off_ld + slot * 2 * T::kSlot;
                mbar_expect_tx(&full[slot], 2 * T::kSlot);
                for (int t = 0; t < 2; ++t) {
                    const CUtensorMap *m = t == 0 ? (it.col ? &mqc : &mqr) : (it.col ? &mkc : &mkr);
                    const int start = t == 0 ? it.q0 : it.k0;
                    const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                    tma_load_4d(dst + t * T::kSlot, m, &full[slot], 0, cw, ch, it.b);
                    if constexpr (!H16) tma_load_4d(dst + t * T::kSlot + T::kTile, m, &full[slot], 32, cw, ch, it.b);
                }
            }
        }
    } else if (tid >= 128) {
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2);         // accumulator rows rbase, rbase + 8
        const int cq = 2 * (lane & 3);                             // first accumulator column of this thread (+ 8j)
        const long hw2 = map_row(p);
        const uint32_t ld_base = smem_u32(smem + S::off_ld), pb = smem_u32(smem + S::off_p);
        uint8_t *pgen = smem + S::off_p;
        // this thread's accumulator rows (nc channels from 0) -> `tile`, laid out as the output's swizzled TMA box(es)
        auto stage = [&](const float *acc, int nc, uint8_t *tile) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                if (r >= LK) continue;
                uint8_t *row = tile + r * 128;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (8 * j >= nc) break;
                    const int c = 8 * j + cq;
                    const int bx = H16 ? 0 : c >> 5, byte = H16 ? 2 * c : 4 * (c & 31);
                    uint8_t *dst = row + bx * T::kTile + ((((byte >> 4) ^ r) & 7) << 4) + (byte & 15);
                    if constexpr (H16) *reinterpret_cast<uint32_t *>(dst) = pack2<F16>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                    else *reinterpret_cast<float2 *>(dst) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                }
            }
        };
        // (thread 0) the staged boxes -> global: reduce-add onto the cleared outputs, or (PL) store into plane `part`
        auto put = [&](const CUtensorMap *m, const uint8_t *tile, int boxes, int px0, const Item &it, int part) {
            const int cw = it.col ? it.line : px0, ch = it.col ? px0 : it.line;
            const int ob = PL ? part * p.sp.B + it.b : it.b;
            for (int bx = 0; bx < boxes; ++bx) {
                if constexpr (PL) tma_store_4d(m, tile + bx * T::kTile, 32 * bx, cw, ch, ob);
                else tma_reduce_add_4d(m, tile + bx * T::kTile, 32 * bx, cw, ch, ob);
            }
            bulk_commit();
        };
        const int qboxes = H16 ? 1 : (p.Cq > 32 ? 2 : 1);           // dQ / dK boxes of 64 fp32 channels: none wholly past Cq
        pdl_wait();                                                // rho (and the cleared outputs) come from the rho pass
        if (t == 0) fence_proxy_async_global();                    // ... and are visible to the reduce-adds
        int held = -1;                                             // (thread 0) ring stage whose dQ copy may still read it
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const int slot = k % kNS;
            // ---- dS of rows rbase + 8h, columns 8j + cq + e, in registers (0 outside lq x lk and at the self entry)
            float ds[LK / 2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                const bool ok = r < it.lq;
                const long pix = item_pixel(p.sp, it, ok ? r : 0);
                const int self = it.col ? it.q0 + r - it.k0 : -1;
                const long off = pix * hw2 + (it.col ? 0 : p.sp.H) + it.k0;
                const float *arow = p.attn + off, *drow = p.dattn + off;
                // float2 loads only where BOTH rows are 8-byte aligned: attn and dattn come from the caller, who may pass
                // views at any float offset
                const bool a8 = ((reinterpret_cast<uintptr_t>(arow) | reinterpret_cast<uintptr_t>(drow)) & 7) == 0;
                const float rho = ok ? __ldg(p.rho + pix) : 0.f;
#pragma unroll
                for (int j = 0; j < LK / 8; ++j) {
                    const int c = 8 * j + cq;
                    float2 a = make_float2(0.f, 0.f), d = make_float2(0.f, 0.f);
                    if (ok && c < it.lk) { a = load_pair(arow, c, it.lk, a8); d = load_pair(drow, c, it.lk, a8); }
                    ds[4 * j + 2 * h] = c == self ? 0.f : a.x * (d.x - rho);
                    ds[4 * j + 2 * h + 1] = c + 1 == self ? 0.f : a.y * (d.y - rho);
                }
            }
            // ---- the previous item's copies have read the dS planes and its stage: release the stage, reuse the planes
            if (t == 0) {
                bulk_wait_read<0>();
                if (held >= 0) mbar_arrive(&empty[held]);
                held = -1;
            }
            mbar_wait(&full[slot], (k / kNS) & 1);
            uint8_t *qs = smem + S::off_ld + slot * 2 * T::kSlot;
            if constexpr (!H16) {
                convert_slot<LK, E>(qs, t);                        // (each ends with a consumer barrier)
                convert_slot<LK, E>(qs + T::kSlot, t);
            } else {
                consumers_sync();
            }
#pragma unroll
            for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rbase + 8 * h;
                    if (r < LK) {
                        uint8_t *d = pgen + j * T::kPlane + r * 16 + cq * 2;
                        const float s0 = ds[4 * j + 2 * h], s1 = ds[4 * j + 2 * h + 1];
                        if constexpr (H16) {
                            *reinterpret_cast<uint32_t *>(d) = pack2<F16>(s0, s1);
                        } else {
                            uint32_t hi, lo;
                            split2(s0, s1, hi, lo);
                            *reinterpret_cast<uint32_t *>(d) = hi;
                            *reinterpret_cast<uint32_t *>(d + LOP) = lo;
                        }
                    }
                }
            fence_proxy_async();
            consumers_sync();
            // ---- dQ = dS K (rows = query pixels), staged in the K slot; dK = dS^T Q (rows = key pixels), staged in the planes
            const uint32_t qb = ld_base + slot * 2 * T::kSlot, kb = qb + T::kSlot;
            float aq[32], ak[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < KP; ++ks) {
                const uint32_t a = pb + 64 * wg * 16 + ks * 2 * T::kPlane;     // dS, K-major (k = key pixels)
                wgmma_ss_n64<F16>(aq, smem_desc(a, T::kPlane, 128), desc_mnmaj<LK, E>(kb, ks, false), ks > 0, 0, 1);
                if constexpr (TERMS == 3) {
                    wgmma_ss_n64<F16>(aq, smem_desc(a, T::kPlane, 128), desc_mnmaj<LK, E>(kb, ks, true), 1, 0, 1);
                    wgmma_ss_n64<F16>(aq, smem_desc(a + LOP, T::kPlane, 128), desc_mnmaj<LK, E>(kb, ks, false), 1, 0, 1);
                }
            }
            wg_commit();
            wg_wait<0>();
            wg_acc_fence<32>(aq);
            consumers_sync();                                      // both warpgroups' dQ MMAs have read the K slot
            stage(aq, 64, qs + T::kSlot);
            fence_proxy_async();
            consumers_sync();
            if (t == 0) put(it.col ? &mdqc : &mdqr, qs + T::kSlot, qboxes, it.q0, it, part_index(p.sp, it));
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < KP; ++ks) {
                const uint32_t at = pb + 8 * wg * T::kPlane + ks * 256;         // dS^T, MN-major (k = query pixels)
                wgmma_ss_n64<F16>(ak, smem_desc(at, 128, T::kPlane), desc_mnmaj<LK, E>(qb, ks, false), ks > 0, 1, 1);
                if constexpr (TERMS == 3) {
                    wgmma_ss_n64<F16>(ak, smem_desc(at, 128, T::kPlane), desc_mnmaj<LK, E>(qb, ks, true), 1, 1, 1);
                    wgmma_ss_n64<F16>(ak, smem_desc(at + LOP, 128, T::kPlane), desc_mnmaj<LK, E>(qb, ks, false), 1, 1, 1);
                }
            }
            wg_commit();
            wg_wait<0>();
            wg_acc_fence<32>(ak);
            consumers_sync();                                      // both warpgroups' dK MMAs have read dS and Q
            stage(ak, 64, pgen);
            fence_proxy_async();
            consumers_sync();
            if (t == 0) {
                put(it.col ? &mdkc : &mdkr, pgen, qboxes, it.k0, it, qtile_part_index(p.sp, it));
                held = slot;
            }
        }
        if (t == 0) bulk_wait<0>();                                // shared memory must outlive the last bulk reads
    }
}

template <int LK, typename E, bool PL>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_attn_bwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                       const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                       const __grid_constant__ CUtensorMap mdqc, const __grid_constant__ CUtensorMap mdqr,
                       const __grid_constant__ CUtensorMap mdkc, const __grid_constant__ CUtensorMap mdkr, AttnBwdParams p)
{
    attn_bwd<LK, E, PL>(mqc, mqr, mkc, mkr, mdqc, mdqr, mdkc, mdkr, p);
}

// The 3D map (cca_tc_attn3d.cu): the kernels above on the [B*T, H, W, Cq] frames view of NDHWC q, k, writing the column and
// row entries of map rows of H + W + T entries; the forward's lse combine takes one more plane, the time branch's.
struct AttnFwdParams3 : AttnFwdParams {
    int T;
};
struct AttnBwdParams3 : AttnBwdParams {
    int T;
};
__device__ __forceinline__ long map_row(const AttnFwdParams3 &p) { return (long)p.sp.H + p.sp.W + p.T; }
__device__ __forceinline__ long map_row(const AttnBwdParams3 &p) { return (long)p.sp.H + p.sp.W + p.T; }

template <int LK, typename E>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_attn3d_fwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                         const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr, AttnFwdParams3 p)
{
    attn_fwd<LK, E>(mqc, mqr, mkc, mkr, p);
}

template <int LK, typename E, bool PL>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_attn3d_bwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                         const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                         const __grid_constant__ CUtensorMap mdqc, const __grid_constant__ CUtensorMap mdqr,
                         const __grid_constant__ CUtensorMap mdkc, const __grid_constant__ CUtensorMap mdkr, AttnBwdParams3 p)
{
    attn_bwd<LK, E, PL>(mqc, mqr, mkc, mkr, mdqc, mdqr, mdkc, mdkr, p);
}

// ---- host launchers.  X3 = false: the 2D map on d (T unused); X3: the 3D map of clips of T frames on the frames view d
// (d.B = B*T), its lse combining the statistics pass's planes and the time plane after them.
template <int LK, typename E, bool X3>
cudaError_t launch_attn_fwd(const void *q, const void *k, float *attn, const float *parts, Dims d, int T, cudaStream_t st,
                            const char **why)
{
    CUtensorMap m[4];
    if (cudaError_t e = get_maps(m, {{q, d.B, d.Cq, LK, LK}, {k, d.B, d.Cq, LK, LK}}, d, kDtype<E>, why)) return e;
    AttnFwdParams3 p;
    p.sp = make_space(d.B, d.H, d.W);
    p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = parts;
    p.attn = attn;
    p.T = T;
    const int smem = StatsSmem<LK, E>::kBytes;
    if constexpr (!X3) {
        return launch_kernel(cca_tc_attn_fwd_kernel<LK, E>, item_grid(p.sp), kThreads, smem, true, st, m[0], m[1], m[2], m[3],
                             static_cast<const AttnFwdParams &>(p));
    } else {
        p.sp.nparts += 1;                // (the items do not depend on it: only the lse combine reads it)
        return launch_kernel(cca_tc_attn3d_fwd_kernel<LK, E>, item_grid(p.sp), kThreads, smem, true, st, m[0], m[1], m[2], m[3], p);
    }
}

// PL: dq, dk are the [nparts*B, H, W, Cq] fp32 plane buffers
template <int LK, typename E, bool PL, bool X3>
cudaError_t launch_attn_bwd(const float *dattn, const float *attn, const float *rho, const void *q, const void *k, void *dq, void *dk,
                            Dims d, int T, cudaStream_t st, const char **why)
{
    CUtensorMap m[8];
    AttnBwdParams3 p;
    p.sp = make_space(d.B, d.H, d.W);
    // output boxes: one tile of the direction (a store never reaches the next tile)
    const int nb = PL ? p.sp.nparts * d.B : d.B;
    if (cudaError_t e = get_maps(m, {{q, d.B, d.Cq, LK, LK}, {k, d.B, d.Cq, LK, LK}, {dq, nb, d.Cq, p.sp.col.tl, p.sp.row.tl},
                                     {dk, nb, d.Cq, p.sp.col.tl, p.sp.row.tl}},
                                 d, kDtype<E>, why))
        return e;
    p.Cq = d.Cq;
    p.attn = attn; p.dattn = dattn; p.rho = rho;
    p.T = T;
    const int smem = AttnBwdSmem<LK, E>::kBytes;
    if constexpr (!X3)
        return launch_kernel(cca_tc_attn_bwd_kernel<LK, E, PL>, item_grid(p.sp), kThreads, smem, true, st, m[0], m[1], m[2], m[3],
                             m[4], m[5], m[6], m[7], static_cast<const AttnBwdParams &>(p));
    else
        return launch_kernel(cca_tc_attn3d_bwd_kernel<LK, E, PL>, item_grid(p.sp), kThreads, smem, true, st, m[0], m[1], m[2],
                             m[3], m[4], m[5], m[6], m[7], p);
}

// Backward of the 2D map (X3 = false) or of the 3D map's column and row entries on the frames view d: the rho pass over rows
// of H + W (+ T) entries, which also clears dq and dk for the reduce-adds, then the item kernel; in planes mode (det on
// tiled lines; fp32, cca_capi.cu refuses 16-bit I/O there) the items store into the dQ, dK planes and planes_sum adds them.
template <bool X3>
cudaError_t map_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws, Dims d,
                         int T, int dtype, cudaStream_t st, const char **why, bool det)
{
    const long npix = (long)d.B * d.H * d.W;
    const bool planes = det && tc_tiled(d);
    const AttnBwdWs w = attn_bwd_ws(d, planes, ws);
    const long clear = planes ? 0 : npix * d.Cq * (dtype == CCA_F32 ? 4 : 2);
    cudaError_t e = attn_rho(dattn, attn, w.rho, npix, d.H + d.W + (X3 ? T : 0), planes ? nullptr : dq, planes ? nullptr : dk,
                             clear, st);
    if (e != cudaSuccess) return e;
    if (planes) {
        float *pq = w.planes.p[0], *pk = w.planes.p[1];
        e = with_tile(d, [&](auto lk) { return launch_attn_bwd<lk(), float, true, X3>(dattn, attn, w.rho, q, k, pq, pk, d, T, st, why); });
        if (e != cudaSuccess) return e;
        const float *src[2] = {pq, pk};
        float *dst[2] = {reinterpret_cast<float *>(dq), reinterpret_cast<float *>(dk)};
        const long n[2] = {npix * d.Cq, npix * d.Cq};
        return planes_sum(src, dst, n, 2, make_space(d.B, d.H, d.W).nparts, st);
    }
    return with_elem_tile(dtype, d, [&](auto el, auto lk) {
        return launch_attn_bwd<lk(), decltype(el), false, X3>(dattn, attn, w.rho, q, k, dq, dk, d, T, st, why);
    });
}

}  // namespace tc
}  // namespace cca
