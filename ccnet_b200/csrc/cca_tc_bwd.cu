// wgmma / TMA backward kernel of criss-cross attention for sm_90a (channels-last tensors).
//
// Closed form of SURVEY.md 8(a) row a11 (autograd of cc_attention/functions.py:38-47), flash-style: the attention matrix is
// recomputed per item from (q, k, lse), never stored.  Items are those of cca_items.cuh (direction, sample, line, query
// tile, key block); because P = exp(S - lse) uses the FINAL lse, every item is independent and ADDS its contributions:
//   S  = Q K^T                     (K-dim Cq)        P  = exp(S - lse[jq])            [registers -> bf16 planes in smem]
//   dP = dO V^T                    (K-dim C, accumulated in registers over the V/dO chunks)
//   dV[jk,c] += sum_jq P[jq,jk] dO[jq,c]   per chunk  (A = P planes read MN-major = P^T, B = dO chunk)
//   dS = P * (dP - delta[jq])      [planes overwrite P]
//   dQ[jq,c] += sum_jk dS[jq,jk] K[jk,c]   (A = dS planes K-major)     dK[jk,c] += sum_jq dS[jq,jk] Q[jq,c]  (A = dS^T)
// ONE persistent launch walks the items sample by sample (column items, then row items of the same sample): the second
// direction finds q,k,v,dO in L2 and its adds land on dq/dk/dv lines that are still L2-resident.
//
// delta[jq] = sum_c dO[jq,c] O[jq,c] is folded into the items (no separate pass over dO and O): the O chunk of the query
// pixels rides the same ring as V and dO, and the conversion of dO -- which reads every dO element anyway -- accumulates the
// dot products.  Two modes: every item computes delta for itself (no dependency), or only the column items of the first key
// block do, publish it through global memory and a per-sample counter, and the other items of the sample wait for that counter
// right before their dS phase (such items always have a higher index than the producers: no cyclic waits).
//
// Output path (dq, dk, dv need no initialisation by the caller).  One tile per line (H, W <= 112): as in the forward the
// column items STORE their rows, the row items ADD onto them once the per-sample counter cdone[b] says every column item of the
// sample has completed its stores.  Tiled lines: several items contribute to the same dk / dv rows, so a prologue clears the
// outputs and every item adds.
//
// All GEMMs run as bf16x3 split MMAs (hi*hi + hi*lo + lo*hi) with fp32 accumulation in registers (single bf16 MMAs for bf16
// I/O), two consumer warpgroups of 64 rows each (cca_tc_common.cuh).
#include <type_traits>

#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace {
using namespace tc;

struct BwdParams {
    ItemSpace sp;
    int C, Cq;
    long npix;
    const float *lse;
    float *delta;              // [B,H,W] <dout, out> per pixel, written by the producer items (first bytes of the workspace)
    unsigned int *ddone;       // [B] delta producers of sample b done (delta_mode 1)
    int delta_mode;            // 0: every item computes its own delta; 1: column / first-key-block items produce, the rest wait
    int out_mode;              // 1: producers store, consumers add after cdone (one tile per line); 0: cleared outputs, everything adds
    unsigned int *cdone;       // [B] producer items of sample b whose stores have completed (out_mode 1)
    int lag;                   // item order (cca_items.cuh): 1 = consumers trail the producers by one block
    int hints;                 // L2 eviction hints on the loads
    void *dq, *dk, *dv;
};

template <int LK, bool BF> struct BwdSmem {
    using T = Tiles<LK, BF>;
    static constexpr int off_qk = 0;                                // Q slot, K slot (held for the whole item: dQ, dK read them)
    static constexpr int off_p = off_qk + 2 * T::kSlot;             // P / dS planes (hi block, lo block)
    // (pad: 64-row P^T operands read up to 16 planes; TMA destinations with SWIZZLE_128B must be 1024-byte aligned)
    static constexpr int off_ld = (off_p + T::kP + (16 - LK / 8) * T::kPlane + 1023) / 1024 * 1024;
    static constexpr int kNLd = (224 * 1024 - 4096 - off_ld) / T::kSlot < 8 ? (224 * 1024 - 4096 - off_ld) / T::kSlot : 8;
    static constexpr int off_tail = off_ld + kNLd * T::kSlot;       // over-read of the last slot by the second warpgroup
    static constexpr int off_dsum = off_tail + (128 - LK) * 128 + 256;   // float [2][128]: delta halves per pixel row
    static constexpr int off_bar = off_dsum + 1024;
    static constexpr int kBytes = off_bar + 8 * (2 + 2 * kNLd);
    static_assert(kNLd >= 3, "ring depth: V, dO, O of one chunk");
    static_assert(kBytes <= 232448, "shared memory budget");
};

// does this item compute delta itself (its ring carries the O chunks)?
__device__ __forceinline__ bool calc_delta(const BwdParams &p, const Item &it) { return p.delta_mode == 0 || (it.col && it.ik == 0); }

template <int LK, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_bwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                  const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                  const __grid_constant__ CUtensorMap mvc, const __grid_constant__ CUtensorMap mvr,
                  const __grid_constant__ CUtensorMap mdoc, const __grid_constant__ CUtensorMap mdor,
                  const __grid_constant__ CUtensorMap moc, const __grid_constant__ CUtensorMap mor, BwdParams p)
{
    using T = Tiles<LK, BF>;
    using S = BwdSmem<LK, BF>;
    using E = typename std::conditional<BF, __nv_bfloat16, float>::type;
    constexpr int TERMS = BF ? 1 : 3;
    constexpr int kNLd = S::kNLd;
    constexpr int KP = LK / 16;
    constexpr uint32_t LOP = T::kPP * T::kPlane;   // P / dS planes: hi block -> lo block
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + S::off_bar);
    uint64_t *qk_full = bars, *qk_empty = bars + 1, *full = bars + 2, *empty = bars + 2 + kNLd;
    float *dsum = reinterpret_cast<float *>(smem + S::off_dsum);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NCH = p.C / kNC;
    const int KQ = p.Cq / 16;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item_order(p.sp, (int)blockIdx.x + k * (int)gridDim.x, p.lag); };

    if (tid == 0) {
        mbar_init(qk_full, 1); mbar_init(qk_empty, kConsumers);
        for (int i = 0; i < kNLd; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumers); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr); prefetch_tmap(&mvc); prefetch_tmap(&mvr);
        prefetch_tmap(&mdoc); prefetch_tmap(&mdor); prefetch_tmap(&moc); prefetch_tmap(&mor);
    }
    __syncthreads();

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
            auto load = [&](uint8_t *dst, uint64_t *bar, const CUtensorMap *m, int c0, const Item &it, int start, bool last_use) {
                const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                if (p.hints == 1) {     // what the sample's consumers read again stays; O and the consumers' own operands stream
                    const uint64_t pol = (is_producer(it) && !last_use) ? pol_keep : pol_stream;
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b, pol);
                    if constexpr (!BF) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b, pol);
                } else {
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b);
                    if constexpr (!BF) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b);
                }
            };
            uint32_t g = 0;
            auto ring = [&](const CUtensorMap *m, int c0, const Item &it, int start, bool last_use) {
                const int slot = g % kNLd;
                mbar_wait(&empty[slot], ((g / kNLd) & 1) ^ 1);
                mbar_expect_tx(&full[slot], T::kSlot);
                load(smem + S::off_ld + slot * T::kSlot, &full[slot], m, c0, it, start, last_use);
                ++g;
            };
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                const bool calc = calc_delta(p, it);
                mbar_wait(qk_empty, (k & 1) ^ 1);
                mbar_expect_tx(qk_full, 2 * T::kSlot);
                load(smem + S::off_qk, qk_full, it.col ? &mqc : &mqr, 0, it, it.q0, false);
                load(smem + S::off_qk + T::kSlot, qk_full, it.col ? &mkc : &mkr, 0, it, it.k0, false);
                for (int n = 0; n < NCH; ++n) {
                    ring(it.col ? &mvc : &mvr, n * kNC, it, it.k0, false);
                    ring(it.col ? &mdoc : &mdor, n * kNC, it, it.q0, false);
                    if (calc) ring(it.col ? &moc : &mor, n * kNC, it, it.q0, p.delta_mode == 1);   // (mode 1: nobody reads O again)
                }
            }
        }
    } else if (tid >= 128) {
        // =============================== consumers (warpgroup wg = rows [64 wg, 64 wg + 64) of each product) ===============================
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2);         // accumulator rows rbase, rbase + 8
        const int cq = 2 * (lane & 3);                             // first accumulator column of this thread (+ 8j)
        const uint32_t qb = smem_u32(smem + S::off_qk), kb = qb + T::kSlot, ld_base = smem_u32(smem + S::off_ld);
        const uint32_t pb = smem_u32(smem + S::off_p);
        uint8_t *pgen = smem + S::off_p;
        E *const dq = reinterpret_cast<E *>(p.dq), *const dk = reinterpret_cast<E *>(p.dk), *const dv = reinterpret_cast<E *>(p.dv);
        pdl_wait();                                                // prep kernel complete: counters (and the outputs) cleared
        uint32_t g = 0;
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const bool calc = calc_delta(p, it);
            const bool prod = p.out_mode == 1 && is_producer(it);
            Item kit = it;                                         // key pixels of the item as "query rows" (pixel addressing)
            kit.q0 = it.k0;
            long qpix[2], kpix[2];
            bool qok[2], kok[2];
            float nlse[2];
            int self[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                qok[h] = r < it.lq; kok[h] = r < it.lk;
                qpix[h] = item_pixel(p.sp, it, qok[h] ? r : 0);
                kpix[h] = item_pixel(p.sp, kit, kok[h] ? r : 0);
                nlse[h] = qok[h] ? -p.lse[qpix[h]] * kLog2e : 0.f;
                self[h] = it.col ? it.q0 + r - it.k0 : -1;
            }
            // ---------------- S = Q K^T, P = exp(S - lse) -> planes
            mbar_wait(qk_full, k & 1);
            if constexpr (!BF) {
                convert_slot<LK, BF>(smem + S::off_qk, t);
                convert_slot<LK, BF>(smem + S::off_qk + T::kSlot, t);
            }
            {
                float acc[LK / 2];
                wg_fence();
                for (int ks = 0; ks < KQ; ++ks) {
                    wgmma_ss<LK>(acc, desc_kmaj<LK, BF>(qb, 64 * wg, ks, false), desc_kmaj<LK, BF>(kb, 0, ks, false), ks > 0, 0, 0);
                    if constexpr (TERMS == 3) {
                        wgmma_ss<LK>(acc, desc_kmaj<LK, BF>(qb, 64 * wg, ks, false), desc_kmaj<LK, BF>(kb, 0, ks, true), 1, 0, 0);
                        wgmma_ss<LK>(acc, desc_kmaj<LK, BF>(qb, 64 * wg, ks, true), desc_kmaj<LK, BF>(kb, 0, ks, false), 1, 0, 0);
                    }
                }
                wg_commit();
                wg_wait<0>();
                wg_acc_fence<LK / 2>(acc);
#pragma unroll
                for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int r = rbase + 8 * h, c = 8 * j + cq;
                        const bool ok0 = qok[h] && c < it.lk && c != self[h];
                        const bool ok1 = qok[h] && c + 1 < it.lk && c + 1 != self[h];
                        const float p0 = ok0 ? exp2f(fmaf(acc[4 * j + 2 * h], kLog2e, nlse[h])) : 0.f;
                        const float p1 = ok1 ? exp2f(fmaf(acc[4 * j + 2 * h + 1], kLog2e, nlse[h])) : 0.f;
                        if (r < LK) {
                            uint8_t *d = pgen + j * T::kPlane + r * 16 + cq * 2;
                            if constexpr (BF) {
                                *reinterpret_cast<uint32_t *>(d) = pack_bf16(p0, p1);
                            } else {
                                uint32_t hi, lo;
                                split2(p0, p1, hi, lo);
                                *reinterpret_cast<uint32_t *>(d) = hi;
                                *reinterpret_cast<uint32_t *>(d + LOP) = lo;
                            }
                        }
                    }
            }
            fence_proxy_async();
            consumers_sync();
            if (!prod && p.out_mode == 1) wait_count(p.cdone + it.b, (unsigned)p.sp.seg0);   // producers of the sample have stored
            // ---------------- per chunk: dP += dO V^T, dV = P^T dO
            float dp[LK / 2];
            float dacc = 0.f;
            for (int n = 0; n < NCH; ++n) {
                const uint32_t gv = g++, gd = g++, go = calc ? g++ : 0;
                mbar_wait(&full[gv % kNLd], (gv / kNLd) & 1);
                mbar_wait(&full[gd % kNLd], (gd / kNLd) & 1);
                if (calc) mbar_wait(&full[go % kNLd], (go / kNLd) & 1);
                uint8_t *vs = smem + S::off_ld + (gv % kNLd) * T::kSlot, *ds = smem + S::off_ld + (gd % kNLd) * T::kSlot;
                if constexpr (!BF) convert_slot<LK, BF>(vs, t);
                if (calc) {
                    dacc += convert_slot<LK, BF>(ds, t, smem + S::off_ld + (go % kNLd) * T::kSlot);
                    if constexpr (BF) consumers_sync();            // (fp32: the conversion ends on a consumer barrier)
                    mbar_arrive(&empty[go % kNLd]);
                } else if constexpr (!BF) {
                    convert_slot<LK, BF>(ds, t);
                }
                const uint32_t vb = ld_base + (gv % kNLd) * T::kSlot, db = ld_base + (gd % kNLd) * T::kSlot;
                float o[32];
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < kNC / 16; ++ks) {
                    wgmma_ss<LK>(dp, desc_kmaj<LK, BF>(db, 64 * wg, ks, false), desc_kmaj<LK, BF>(vb, 0, ks, false), n > 0 || ks > 0, 0, 0);
                    if constexpr (TERMS == 3) {
                        wgmma_ss<LK>(dp, desc_kmaj<LK, BF>(db, 64 * wg, ks, false), desc_kmaj<LK, BF>(vb, 0, ks, true), 1, 0, 0);
                        wgmma_ss<LK>(dp, desc_kmaj<LK, BF>(db, 64 * wg, ks, true), desc_kmaj<LK, BF>(vb, 0, ks, false), 1, 0, 0);
                    }
                }
#pragma unroll
                for (int ks = 0; ks < KP; ++ks) {
                    const uint32_t pa = pb + 8 * wg * T::kPlane + ks * 256;      // P^T: rows = key pixels [64 wg, +64), k = query rows
                    wgmma_ss_n64(o, smem_desc(pa, 128, T::kPlane), desc_mnmaj<LK, BF>(db, ks, false), ks > 0, 1, 1);
                    if constexpr (TERMS == 3) {
                        wgmma_ss_n64(o, smem_desc(pa, 128, T::kPlane), desc_mnmaj<LK, BF>(db, ks, true), 1, 1, 1);
                        wgmma_ss_n64(o, smem_desc(pa + LOP, 128, T::kPlane), desc_mnmaj<LK, BF>(db, ks, false), 1, 1, 1);
                    }
                }
                wg_commit();
                wg_wait<0>();
                wg_acc_fence<LK / 2>(dp);
                wg_acc_fence<32>(o);
                mbar_arrive(&empty[gv % kNLd]);
                mbar_arrive(&empty[gd % kNLd]);
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (kok[h]) {
                        E *row = dv + kpix[h] * p.C + n * kNC + cq;
#pragma unroll
                        for (int j = 0; j < 8; ++j) put2(row + 8 * j, o[4 * j + 2 * h], o[4 * j + 2 * h + 1], !prod);
                    }
            }
            // ---------------- delta of the query rows
            float dl[2] = {0.f, 0.f};
            if (calc) {
                dsum[(t >> 7) * 128 + (t & 127)] = dacc;
                consumers_sync();
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rbase + 8 * h;
                    dl[h] = dsum[r] + dsum[128 + r];
                    // delta[B,H,W] always ends up in the workspace (the caller's d gamma = sum of it); in mode 1 it is also how
                    // the other items of the sample get it
                    if (qok[h] && is_producer(it) && (lane & 3) == 0) p.delta[qpix[h]] = dl[h];
                }
                if (p.delta_mode == 1) {
                    __threadfence();
                    consumers_sync();
                    if (t == 0) atomicAdd(p.ddone + it.b, 1u);
                }
            } else {
                wait_count(p.ddone + it.b, (unsigned)p.sp.seg0);
#pragma unroll
                for (int h = 0; h < 2; ++h) dl[h] = qok[h] ? __ldcg(p.delta + qpix[h]) : 0.f;
            }
            // ---------------- dS = P * (dP - delta) -> planes (every dV product of both warpgroups has read P)
            consumers_sync();
#pragma unroll
            for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rbase + 8 * h;
                    if (r < LK) {
                        uint8_t *d = pgen + j * T::kPlane + r * 16 + cq * 2;
                        const uint32_t hw = *reinterpret_cast<const uint32_t *>(d);
                        const uint32_t lw = BF ? 0u : *reinterpret_cast<const uint32_t *>(d + LOP);
                        const float p0 = bf_lo(hw) + bf_lo(lw), p1 = bf_hi(hw) + bf_hi(lw);
                        // masked / padded entries have P == 0 exactly; rows past the tile are cleared (their dP is not defined)
                        const float s0 = qok[h] ? p0 * (dp[4 * j + 2 * h] - dl[h]) : 0.f;
                        const float s1 = qok[h] ? p1 * (dp[4 * j + 2 * h + 1] - dl[h]) : 0.f;
                        if constexpr (BF) {
                            *reinterpret_cast<uint32_t *>(d) = pack_bf16(s0, s1);
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
            // ---------------- dQ = dS K (rows = query pixels), dK = dS^T Q (rows = key pixels)
            {
                float aq[32], ak[32];
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < KP; ++ks) {
                    const uint32_t a = pb + 64 * wg * 16 + ks * 2 * T::kPlane;     // dS, K-major (k = key pixels)
                    wgmma_ss_n64(aq, smem_desc(a, T::kPlane, 128), desc_mnmaj<LK, BF>(kb, ks, false), ks > 0, 0, 1);
                    if constexpr (TERMS == 3) {
                        wgmma_ss_n64(aq, smem_desc(a, T::kPlane, 128), desc_mnmaj<LK, BF>(kb, ks, true), 1, 0, 1);
                        wgmma_ss_n64(aq, smem_desc(a + LOP, T::kPlane, 128), desc_mnmaj<LK, BF>(kb, ks, false), 1, 0, 1);
                    }
                    const uint32_t at = pb + 8 * wg * T::kPlane + ks * 256;         // dS^T, MN-major (k = query pixels)
                    wgmma_ss_n64(ak, smem_desc(at, 128, T::kPlane), desc_mnmaj<LK, BF>(qb, ks, false), ks > 0, 1, 1);
                    if constexpr (TERMS == 3) {
                        wgmma_ss_n64(ak, smem_desc(at, 128, T::kPlane), desc_mnmaj<LK, BF>(qb, ks, true), 1, 1, 1);
                        wgmma_ss_n64(ak, smem_desc(at + LOP, 128, T::kPlane), desc_mnmaj<LK, BF>(qb, ks, false), 1, 1, 1);
                    }
                }
                wg_commit();
                wg_wait<0>();
                wg_acc_fence<32>(aq);
                wg_acc_fence<32>(ak);
                mbar_arrive(qk_empty);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int c = 8 * j + cq;
                        if (c < p.Cq) {
                            if (qok[h]) put2(dq + qpix[h] * p.Cq + c, aq[4 * j + 2 * h], aq[4 * j + 2 * h + 1], !prod);
                            if (kok[h]) put2(dk + kpix[h] * p.Cq + c, ak[4 * j + 2 * h], ak[4 * j + 2 * h + 1], !prod);
                        }
                    }
                }
            }
            if (prod) __threadfence();
            consumers_sync();                                      // (also: the planes and dsum are free for the next item)
            if (prod && t == 0) atomicAdd(p.cdone + it.b, 1u);     // publish: all stores of this item are visible
        }
    }
}

// Prologue of the backward: clears the outputs (tiled lines) and the per-sample counters.
__global__ void __launch_bounds__(256) cca_bwd_prep_kernel(uint4 *dq, uint4 *dk, uint4 *dv, long nq16, long nv16,
                                                           unsigned int *counters, int n_counters)
{
    pdl_launch_dependents();
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long)gridDim.x * blockDim.x;
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (long i = tid; i < nq16; i += nth) { dq[i] = z; dk[i] = z; }
    for (long i = tid; i < nv16; i += nth) dv[i] = z;
    for (long i = tid; i < n_counters; i += nth) counters[i] = 0u;
}

template <int LK, bool BF>
cudaError_t launch_bwd(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse, float *delta,
                       unsigned int *counters, void *dq, void *dk, void *dv, Dims d, int delta_mode, cudaStream_t st,
                       const char **why)
{
    CUtensorMap m[10];
    const void *base[5] = {q, k, v, dout, out};
    const int ch[5] = {d.Cq, d.Cq, d.C, d.C, d.C};
    BwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    for (int t = 0; t < 5; ++t)
        for (int r = 0; r < 2; ++r)
            // LK-pixel boxes, zero-filled past the line
            if (!get_map(&m[2 * t + r], base[t], d.B, d.H, d.W, ch[t], LK, r == 0, BF)) {
                if (why) *why = "cuTensorMapEncodeTiled failed";
                return cudaErrorInvalidValue;
            }
    p.C = d.C; p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.lse = lse; p.delta = delta;
    p.ddone = counters; p.cdone = counters + d.B;
    p.delta_mode = delta_mode;
    const bool one_tile = p.sp.col.nt == 1 && p.sp.row.nt == 1;
    p.out_mode = one_tile ? 1 : 0;
    p.lag = tc_lag() != 0 ? 1 : 0;
    p.hints = tc_l2_hints();
    p.dq = dq; p.dk = dk; p.dv = dv;
    const long es = BF ? 2 : 4;
    const long nq = p.out_mode == 1 ? 0 : p.npix * d.Cq * es, nv = p.out_mode == 1 ? 0 : p.npix * d.C * es;
    cca_bwd_prep_kernel<<<p.out_mode == 1 ? 1 : sm_count(), 256, 0, st>>>(
        reinterpret_cast<uint4 *>(dq), reinterpret_cast<uint4 *>(dk), reinterpret_cast<uint4 *>(dv), nq / 16, nv / 16, counters, 3 * d.B);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    auto kern = cca_tc_bwd_kernel<LK, BF>;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem<LK, BF>::kBytes);
    if (e != cudaSuccess) return e;
    const int sms = sm_count();
    const int grid = p.sp.total < sms ? p.sp.total : sms;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = BwdSmem<LK, BF>::kBytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = tc_pdl() ? 1 : 0;
    e = cudaLaunchKernelEx(&cfg, kern, m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8], m[9], p);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace

bool tc_backward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

// Workspace of the backward: delta [B,H,W] fp32, then 3*B unsigned counters.
size_t tc_backward_workspace(Dims d)
{
    const size_t delta = ((size_t)d.B * d.H * d.W * sizeof(float) + 15) & ~(size_t)15;
    return delta + (((size_t)3 * d.B * sizeof(unsigned int) + 15) & ~(size_t)15);
}

// all tensors channels-last (NHWC), fp32 or bf16
cudaError_t tc_backward(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, Dims d, int dtype, cudaStream_t st, const char **why)
{
    float *delta = reinterpret_cast<float *>(ws);
    const size_t delta_bytes = ((size_t)d.B * d.H * d.W * sizeof(float) + 15) & ~(size_t)15;
    unsigned int *counters = reinterpret_cast<unsigned int *>(reinterpret_cast<uint8_t *>(ws) + delta_bytes);
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const int lk = lk_for(max_tile(sp));
    const bool bf = dtype == CCA_BF16;
    int mode = tc_delta_mode();                       // -1: automatic = producers compute delta for their sample (the consumers
    if (mode < 0) mode = 1;                           // only ever wait for lower-indexed items, tiled or not)
    if (bf)
        return lk == 80 ? launch_bwd<80, true>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why)
                        : launch_bwd<112, true>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why);
    return lk == 80 ? launch_bwd<80, false>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why)
                    : launch_bwd<112, false>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why);
}

}  // namespace cca
