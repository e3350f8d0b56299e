// wgmma / TMA forward (values) kernel of criss-cross attention for sm_90a (channels-last tensors).
//
// Layout: q,k [B,H,W,Cq], v,out [B,H,W,C] (torch channels_last).  In this layout an image row and an image column are
// the same object -- L pixels with a fixed pixel stride, each pixel's channels contiguous -- so one kernel serves both
// branches of cc_attention/functions.py:38-47.
//
// Formulation (DESIGN.md 3): the statistics pre-pass (cca_tc_stats.cuh) has left the log-sum-exp of every pixel's logits
// per (direction, key block).  An item (cca_items.cuh: direction, sample, line, query tile, key block) combines those few
// planes into the pixel's final lse and computes its share of the output with the FINAL normalisation,
//     P = exp(S - lse)        O_item = P V_block        out[query pixels] += O_item
// so items never exchange anything: no partial output is written and read back, no per-pixel merge, and lines longer
// than one tile are just more items.  ONE persistent launch walks the items sample by sample: the second direction of a
// sample finds q,k,v in L2 and adds onto output lines that are still L2-resident.
//
// Two touches per output element, ordered: the "producer" items of a sample (column lines, first key block) STORE their
// rows, every other item of the sample ADDS onto them (TMA reduce-add at L2) once the per-sample counter cdone[b] says all
// producers have completed their stores.  Items are walked in one of the two orders of cca_items.cuh (launch_fwd picks it):
// the lagged one -- P(0) | P(1) C(0) | ... -- in which a consumer practically never waits, or sample after sample, which
// keeps one sample's v and out in the L2 instead of two.  Only items with a LOWER index are ever waited for and each
// persistent CTA walks its items in increasing order, so the wait cannot cycle.  With one tile per line every output element
// is one store plus one add: the result is bit-reproducible; with key-block tiling a pixel gets 2*nt-1 adds whose order is
// not fixed.
//
// Roles (cca_tc_common.cuh):
//   producer lane       : Q, K of an item into their own stage; the item's 64-channel V chunks into a ring.  4-D tiled loads,
//                         SWIZZLE_128B, pixels past the line zero-filled.
//   consumer warpgroups : fp32 only: tiles -> bf16 hi + lo planes in place (x = hi + lo to ~2^-17).  S = Q K^T (wgmma, both
//                         operands in shared memory), P = exp2(S log2e - lse2) in registers, re-packed as the 16-bit A operand
//                         of O = P V (wgmma with A from registers, 3 MMAs per k-step for fp32 I/O).
//   chunk pipeline      : two O accumulators.  While chunk n's wgmma group runs, chunk n - 1's O is written into chunk n - 1's
//                         own V slot (its MMAs have retired) in the swizzled layout of the output's TMA box and chunk n + 1's
//                         slot is converted; then chunk n is waited for, one thread stores / reduce-adds chunk n - 1 with TMA,
//                         and chunk n + 1 is issued.  A slot goes back to the producer once its bulk copy has read it,
//                         checked one chunk later.
//
// Planes mode (PL, fp32 only; torch.use_deterministic_algorithms): with key-block tiling the reduce-adds above land in no
// fixed order.  Instead every item STORES its O tile into partial plane part_index(item) -- the (direction, key block)
// index of the lse planes -- of a [nparts*B, H, W, C] buffer; each (pixel, plane) pair is written by exactly one item, so
// nothing waits for anything, and cca_planes_sum_kernel (cca_tc_det.cu) adds the planes in plane order into out.

#pragma once
#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace tc {

// PL: `out` is the [nparts*B, H, W, C] plane buffer (cca_tc_det.cu sums it into the output).  extra_parts: planes of `parts`
// past the statistics pass's own (the time branch of the 3D op, cca_tc_time.cu) that the final lse combines too; the item
// space and the planes-mode output buffer stay those of the 2D problem
struct FwdArgs {
    const void *q, *k, *v;
    void *out;
    float *lse;
    const float *parts;
    unsigned int *cdone;
    Dims d;
    cudaStream_t st;
    const char **why;
    int extra_parts;
};
template <int LK, typename E, bool PL = false> cudaError_t launch_fwd(const FwdArgs &a);

struct FwdParams {
    ItemSpace sp;
    int C, Cq;
    long npix;
    const float *parts;    // [nparts][B*H*W] partial log2-sum-exp2 (statistics pre-pass)
    float *lse;            // [B,H,W] natural-log lse (saved for backward)
    unsigned int *cdone;   // [B] producer items of sample b whose stores have completed (cleared by the statistics kernel)
    int lag;               // item order: 1 = consumers trail the producers by one block, 0 = sample after sample
    int hints;             // L2 eviction hints on the loads and the output stores
};

template <int LK, typename E> struct FwdSmem {
    using T = Tiles<LK, E>;
    static constexpr int off_qk = 0;                               // Q slot, K slot
    static constexpr int off_ld = off_qk + 2 * T::kSlot;           // ring of V chunks
    static constexpr int kNLd = (200 * 1024 - off_ld) / T::kSlot < 8 ? (200 * 1024 - off_ld) / T::kSlot : 8;
    static constexpr int off_tail = off_ld + kNLd * T::kSlot;      // 64-row wgmmas of the second warpgroup read up to
                                                                   // (128 - LK) rows past a tile; they only feed discarded rows
    static constexpr int off_bar = off_tail + (128 - LK) * 128 + 1024;
    static constexpr int kBytes = off_bar + 8 * (2 + 2 * kNLd);
    static_assert(kNLd >= 4, "ring depth: chunks n - 2 (store reading), n - 1 (staged), n (MMAs), n + 1 (converting)");
    static_assert(kBytes <= 232448, "shared memory budget");
};

template <int LK, typename E, bool PL = false>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_fwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                  const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                  const __grid_constant__ CUtensorMap mvc, const __grid_constant__ CUtensorMap mvr,
                  const __grid_constant__ CUtensorMap moc, const __grid_constant__ CUtensorMap mor, FwdParams p)
{
    using T = Tiles<LK, E>;
    using S = FwdSmem<LK, E>;
    constexpr bool H16 = kH16<E>, F16 = kF16<E>;
    constexpr int kNLd = S::kNLd;
    constexpr int TERMS = H16 ? 1 : 3;
    constexpr int KP = LK / 16;               // k-steps of O = P V
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + S::off_bar);
    uint64_t *qk_full = bars, *qk_empty = bars + 1, *full = bars + 2, *empty = bars + 2 + kNLd;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NCH = p.C / kNC;
    const int KQ = p.Cq / 16;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item_order(p.sp, (int)blockIdx.x + k * (int)gridDim.x, p.lag); };

    if (tid == 0) {
        mbar_init(qk_full, 1); mbar_init(qk_empty, kConsumers);
        for (int i = 0; i < kNLd; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }   // empty: the store-issuing thread
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr); prefetch_tmap(&mvc); prefetch_tmap(&mvr);
        prefetch_tmap(&moc); prefetch_tmap(&mor);
    }
    __syncthreads();

    if (tid < 128) {
        // =============================== TMA producer ===============================
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && lane == 0) {
            const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
            auto load = [&](uint8_t *dst, uint64_t *bar, const CUtensorMap *m, int c0, const Item &it, int start) {
                const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                if (p.hints == 1) {     // producers' operands are read again by the sample's consumers; theirs are not
                    const uint64_t pol = is_producer(it) ? pol_keep : pol_stream;
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b, pol);
                    if constexpr (!H16) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b, pol);
                } else {
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b);
                    if constexpr (!H16) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b);
                }
            };
            uint32_t g = 0;
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                mbar_wait(qk_empty, (k & 1) ^ 1);
                mbar_expect_tx(qk_full, 2 * T::kSlot);
                load(smem + S::off_qk, qk_full, it.col ? &mqc : &mqr, 0, it, it.q0);
                load(smem + S::off_qk + T::kSlot, qk_full, it.col ? &mkc : &mkr, 0, it, it.k0);
                for (int n = 0; n < NCH; ++n, ++g) {
                    const int slot = g % kNLd;
                    mbar_wait(&empty[slot], ((g / kNLd) & 1) ^ 1);
                    mbar_expect_tx(&full[slot], T::kSlot);
                    load(smem + S::off_ld + slot * T::kSlot, &full[slot], it.col ? &mvc : &mvr, n * kNC, it, it.k0);
                }
            }
        }
    } else {
        // =============================== consumers (warpgroup wg = query rows [64 wg, 64 wg + 64)) ===============================
        setmaxnreg_inc<kConsumerRegs>();
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2);         // rows rbase, rbase + 8 of the accumulators
        const uint32_t qb = smem_u32(smem + S::off_qk), kb = qb + T::kSlot, ld_base = smem_u32(smem + S::off_ld);
        const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
        // chunk n's O (this thread's rows rbase, rbase + 8; 64 channels) -> its V slot, laid out as the output's swizzled TMA
        // box(es) [tile px][128 B]; accumulator rows past LK are padding and would land in the next slot, so they are skipped
        auto stage = [&](const float (&o)[32], uint8_t *slot) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                if (r >= LK) continue;
                uint8_t *row = slot + r * 128;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    const int bx = H16 ? 0 : c >> 5, byte = H16 ? 2 * c : 4 * (c & 31);
                    uint8_t *dst = row + bx * T::kTile + ((((byte >> 4) ^ r) & 7) << 4) + (byte & 15);
                    if constexpr (H16) *reinterpret_cast<uint32_t *>(dst) = pack2<F16>(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
                    else *reinterpret_cast<float2 *>(dst) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
                }
            }
        };
        pdl_wait();                                                // parts and the counters come from the statistics kernel
        uint32_t g = 0;
        int pending = -1;                                          // (thread 0) slot whose bulk store may still be reading it
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            bool prod = true;                                      // (PL: every item stores)
            if constexpr (!PL) prod = is_producer(it);
            // ---- partial lse planes of rows rbase (h = 0), rbase + 8 (h = 1): the first kPre are loaded here, all at once, and
            // only used once S is in flight, so their L2 latency overlaps the Q / K wait, the conversion and S
            constexpr int kPre = 4;                                // (one tile per line: 2 planes)
            float pv[2][kPre];
            long pix[2];
            int self[2];
            bool rok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                rok[h] = r < it.lq;
                pix[h] = item_pixel(p.sp, it, rok[h] ? r : 0);
                self[h] = it.col ? it.q0 + r - it.k0 : -1;
#pragma unroll
                for (int i = 0; i < kPre; ++i)
                    pv[h][i] = rok[h] && i < p.sp.nparts ? __ldcg(p.parts + (long)i * p.npix + pix[h]) : 0.f;
            }
            // ---- S = Q K^T
            mbar_wait(qk_full, k & 1);
            if constexpr (!H16) {
                convert_slot<LK, E>(smem + S::off_qk, t);
                convert_slot<LK, E>(smem + S::off_qk + T::kSlot, t);
            }
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
            // ---- final lse2 of the two rows while S runs (planes past kPre, if any, are read here)
            float nlse[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float lse2 = 0.f;
                if (rok[h]) {
                    float m = -INFINITY;
#pragma unroll
                    for (int i = 0; i < kPre; ++i)
                        if (i < p.sp.nparts) m = fmaxf(m, pv[h][i]);
                    for (int i = kPre; i < p.sp.nparts; ++i) m = fmaxf(m, __ldcg(p.parts + (long)i * p.npix + pix[h]));
                    float sum = 0.f;
#pragma unroll
                    for (int i = 0; i < kPre; ++i)
                        if (i < p.sp.nparts) sum += exp2f(pv[h][i] - m);
                    for (int i = kPre; i < p.sp.nparts; ++i) sum += exp2f(__ldcg(p.parts + (long)i * p.npix + pix[h]) - m);
                    lse2 = m + log2f(sum);
                    if (!it.col && it.ik == 0 && (lane & 3) == 0) p.lse[pix[h]] = lse2 * kLn2;
                }
                nlse[h] = -lse2;
            }
            wg_wait<0>();
            wg_acc_fence<LK / 2>(acc);
            mbar_arrive(qk_empty);
            // ---- P = exp2(S log2e - lse2) as 16-bit A fragments (fp32 I/O: bf16 hi, lo)
            uint32_t ph[KP][4], pl[KP][4];
#pragma unroll
            for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = 8 * j + 2 * (lane & 3);
                    const bool ok0 = rok[h] && c < it.lk && c != self[h];
                    const bool ok1 = rok[h] && c + 1 < it.lk && c + 1 != self[h];
                    const float p0 = ok0 ? exp2f(fmaf(acc[4 * j + 2 * h], kLog2e, nlse[h])) : 0.f;
                    const float p1 = ok1 ? exp2f(fmaf(acc[4 * j + 2 * h + 1], kLog2e, nlse[h])) : 0.f;
                    // A fragment of k-step j/2: {row r, cols 0-7}, {row r+8, cols 0-7}, {row r, cols 8-15}, {row r+8, cols 8-15}
                    const int reg = (j & 1) * 2 + h;
                    if constexpr (H16) {
                        ph[j / 2][reg] = pack2<F16>(p0, p1);
                        pl[j / 2][reg] = 0u;
                    } else {
                        split2(p0, p1, ph[j / 2][reg], pl[j / 2][reg]);
                    }
                }
            // ---- O = P V, 64 channels at a time.  Chunk n's wgmma group runs while chunk n - 1's O (the other accumulator)
            // is staged and chunk n + 1 is converted; only then is chunk n waited for and chunk n + 1 issued.  One group is in
            // flight at a time: with chunk n + 1 issued before chunk n is waited for, the accumulator that chunk n + 1 later
            // overwrites is read inside chunk n's pipeline stage and ptxas serialises every wgmma (C7514).
            const uint32_t g0 = g;
            g += NCH;
            const CUtensorMap *const mo = it.col ? &moc : &mor;
            const int ow = it.col ? it.line : it.q0, oh = it.col ? it.q0 : it.line;
            auto slot_of = [&](int n) { return (int)((g0 + n) % kNLd); };
            auto prep = [&](int n) {                               // chunk n's V has landed; fp32: split into planes
                mbar_wait(&full[slot_of(n)], ((g0 + n) / kNLd) & 1);
                if constexpr (!H16) convert_slot<LK, E>(smem + S::off_ld + slot_of(n) * T::kSlot, t);
            };
            auto mma = [&](float (&o)[32], int n) {
                const uint32_t vb = ld_base + slot_of(n) * T::kSlot;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < KP; ++ks) {
                    wgmma_rs_n64_tb<F16>(o, ph[ks], desc_mnmaj<LK, E>(vb, ks, false), ks > 0);
                    if constexpr (TERMS == 3) {
                        wgmma_rs_n64_tb<F16>(o, ph[ks], desc_mnmaj<LK, E>(vb, ks, true), 1);
                        wgmma_rs_n64_tb<F16>(o, pl[ks], desc_mnmaj<LK, E>(vb, ks, false), 1);
                    }
                }
                wg_commit();
            };
            auto write = [&](float (&o)[32], int n) {              // chunk n has retired in both warpgroups after the barrier
                wg_acc_fence<32>(o);
                consumers_sync();
                stage(o, smem + S::off_ld + slot_of(n) * T::kSlot);
                fence_proxy_async();
                consumers_sync();
            };
            auto store = [&](int n) {                              // chunk n is staged
                if (t != 0) return;
                if (n == 0 && !prod) fence_proxy_async_global();  // the counter's acquire (below) before the reduce-adds
                const uint8_t *sl = smem + S::off_ld + slot_of(n) * T::kSlot;
                const int ob = PL ? part_index(p.sp, it) * p.sp.B + it.b : it.b;     // sample coordinate of the output box
#pragma unroll
                for (int bx = 0; bx < (H16 ? 1 : 2); ++bx) {
                    const int c0 = n * kNC + 32 * bx;
                    const uint8_t *src = sl + bx * T::kTile;
                    if (p.hints == 1) {                            // producers' rows are added onto by the sample's consumers
                        if (prod) tma_store_4d(mo, src, c0, ow, oh, ob, pol_keep);
                        else tma_reduce_add_4d(mo, src, c0, ow, oh, ob, pol_stream);
                    } else {
                        if (prod) tma_store_4d(mo, src, c0, ow, oh, ob);
                        else tma_reduce_add_4d(mo, src, c0, ow, oh, ob);
                    }
                }
                bulk_commit();
                bulk_wait_read<1>();                               // the previous chunk's store has read its slot
                if (pending >= 0) mbar_arrive(&empty[pending]);
                pending = slot_of(n);
            };
            // before a consumer's first reduce-add: every producer of this sample has stored its rows.  Only the adds need it,
            // so S, P and the first chunks' MMAs overlap the wait.  It sits where no wgmma group is in flight, and all threads
            // wait: a spin in thread 0 alone, while a group is in flight, makes ptxas serialise the wgmmas.
            auto acquire = [&](int n) {
                if (n == 0 && !prod) wait_count(p.cdone + it.b, (unsigned)p.sp.seg0);
            };
            // chunk n in flight in oc, chunk n - 1 retired in op
            auto step = [&](float (&oc)[32], float (&op)[32], int n) {
                if (n > 0) write(op, n - 1);
                const bool more = n + 1 < NCH;
                if (more) prep(n + 1);
                wg_wait<0>();
                if (n > 0) {
                    acquire(n - 1);
                    store(n - 1);
                }
                if (more) mma(op, n + 1);
            };
            float o0[32], o1[32];
            prep(0);
            mma(o0, 0);
            for (int n = 0; n < NCH; n += 2) {
                step(o0, o1, n);
                if (n + 1 < NCH) step(o1, o0, n + 1);
            }
            wg_wait<0>();                                          // (nothing is pending; ptxas cannot tell which step ran last)
            if (NCH & 1) write(o0, NCH - 1);
            else write(o1, NCH - 1);
            acquire(NCH - 1);
            store(NCH - 1);
            if constexpr (!PL) {
                if (prod && t == 0) {                              // publish: all stores of this item are complete
                    bulk_wait<0>();
                    mbar_arrive(&empty[pending]);
                    pending = -1;
                    publish_count(p.cdone + it.b);
                }
            }
        }
        if (t == 0) bulk_wait<0>();                                // shared memory must outlive the last bulk reads
    }
}

template <int LK, typename E, bool PL> cudaError_t launch_fwd(const FwdArgs &a)
{
    CUtensorMap m[8];
    const Dims &d = a.d;
    FwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    // loads: LK-pixel boxes, pixels past the line are zero-filled; output: boxes of one tile of the direction, so a store
    // never reaches into the next tile of a line (pixels past the line are not written)
    const MapSpec out{a.out, PL ? p.sp.nparts * d.B : d.B, d.C, p.sp.col.tl, p.sp.row.tl};
    if (cudaError_t e = get_maps(m, {{a.q, d.B, d.Cq, LK, LK}, {a.k, d.B, d.Cq, LK, LK}, {a.v, d.B, d.C, LK, LK}, out}, d, kDtype<E>,
                                 a.why))
        return e;
    p.sp.nparts += a.extra_parts;        // (after the maps: the planes-mode output holds the 2D problem's planes only)
    p.C = d.C; p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = a.parts; p.lse = a.lse; p.cdone = a.cdone;
    p.hints = tc_l2_hints();
    const int grid = item_grid(p.sp);
    // Item order (default; DESIGN.md 4).  Sample after sample, the first consumers of each sample wait for its last producers,
    // up to about one item per CTA and sample; in the lagged order two samples' v and out are in play in the L2 instead of one.
    // The wait weighs less the more items a sample has per CTA.  Measured on an H100 (132 SMs): sample after sample is faster
    // from 4/3 items per CTA (lines of 89 pixels and more) with 4 samples or more, and slower with fewer items per CTA (lines
    // of 73 and 81) or 2 samples.
    const int lag = tc_lag();
    p.lag = lag >= 0 ? lag : (d.B >= 4 && 3 * p.sp.per_sample >= 4 * grid ? 0 : 1);
    // may start ahead of the statistics kernel's completion (griddepcontrol.wait inside)
    return launch_kernel(cca_tc_fwd_kernel<LK, E, PL>, grid, kThreads, FwdSmem<LK, E>::kBytes, true, a.st, m[0], m[1], m[2], m[3], m[4],
                         m[5], m[6], m[7], p);
}

// The f16 instantiations live in their own translation unit (cca_tc_f16.cu), the planes-mode ones (fp32) in cca_tc_det.cu.
extern template cudaError_t launch_fwd<80, __half>(const FwdArgs &);
extern template cudaError_t launch_fwd<112, __half>(const FwdArgs &);
extern template cudaError_t launch_fwd<80, float, true>(const FwdArgs &);
extern template cudaError_t launch_fwd<112, float, true>(const FwdArgs &);

}  // namespace tc
}  // namespace cca
