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
// outputs and every item adds.  Every output tile is staged in shared memory in the swizzled layout of the output's TMA box and
// written by one thread with a TMA store or a TMA reduce-add at L2: a dV chunk in the dO slot of its chunk, dQ in the K slot,
// dK in the P / dS planes, each once the MMAs that read that memory have retired in both warpgroups.
//
// Planes mode (PL, fp32 only; torch.use_deterministic_algorithms): on tiled lines the reduce-adds above land in no fixed
// order.  Instead every item STORES its tiles into partial planes, [nparts*B, H, W, C or Cq] buffers: dQ into plane
// part_index(item) (direction, key block), dK and dV into plane qtile_part_index(item) (direction, query tile).  Each
// (pixel, plane) pair is written by exactly one item, so there is no clear and no cdone wait (the delta hand-off stays), and
// cca_planes_sum_kernel (cca_tc_det.cu) adds the planes in plane order into dq, dk, dv.
//
// All GEMMs run as bf16x3 split MMAs (hi*hi + hi*lo + lo*hi) with fp32 accumulation in registers (single bf16 / f16 MMAs for
// 16-bit I/O), two consumer warpgroups of 64 rows each (cca_tc_common.cuh).
#pragma once
#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace tc {

// PL: dq, dk, dv are the [nparts*B, H, W, Cq or C] plane buffers (cca_tc_det.cu sums them into the gradients).  delta and
// counters: the workspace's [B,H,W] delta and [3*B] counters
struct BwdArgs {
    const void *dout, *q, *k, *v, *out;
    const float *lse;
    float *delta;
    unsigned int *counters;
    void *dq, *dk, *dv;
    Dims d;
    int delta_mode;
    cudaStream_t st;
    const char **why;
};
template <int LK, typename E, bool PL = false> cudaError_t launch_bwd(const BwdArgs &a);

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
};

// The load ring holds ONE 128-byte TMA box per slot: 32 channels for fp32 (converted in place to hi/lo planes), 64 for 16-bit
// I/O.  Per item it carries Q's boxes, K's boxes, then the V, dO (, O) chunks.  Small slots buy depth: at LK = 112 fp32 the ring
// has 8 slots (2 2/3 chunks of V, dO, O), so chunk n + 1 lands and is converted while chunk n's MMAs run, and the next item's
// Q, K and first chunks land while this item runs its dS, dQ, dK epilogue.  A dV chunk has the footprint of a slot and is
// staged in its chunk's dO slot, which goes back to the producer once the bulk copy has read it.
template <int LK, typename E> struct BwdSmem {
    using T = Tiles<LK, E>;
    static constexpr int kCh = T::H16 ? kNC : kNC / 2;               // channels per ring slot / per chunk
    static constexpr int kRSlot = T::kTile;                         // ring slot bytes: [LK px][128 B]
    static constexpr int off_qk = 0;                                // Q, K of the item, moved here from the ring (dQ, dK read them)
    static constexpr int off_p = off_qk + 2 * T::kSlot;             // P / dS planes (hi block, lo block)
    // (pad: 64-row P^T operands read up to 16 planes; TMA destinations with SWIZZLE_128B must be 1024-byte aligned)
    static constexpr int off_ld = (off_p + T::kP + (16 - LK / 8) * T::kPlane + 1023) / 1024 * 1024;
    static constexpr int kTail = (128 - LK) * 128 + 256;            // over-read of the last slot by the second warpgroup
    static constexpr int kDsum = 1024;                              // float [2][128]: delta halves per pixel row
    static constexpr int kBudget = 232448;                          // 227 KB: the opt-in maximum per block on sm_90
    // every slot also needs its full / empty barriers (8 B each)
    static constexpr int kNLd = (kBudget - off_ld - kTail - kDsum) / (kRSlot + 16);
    static constexpr int off_tail = off_ld + kNLd * kRSlot;
    static constexpr int off_dsum = off_tail + kTail;
    static constexpr int off_bar = off_dsum + kDsum;
    static constexpr int kBytes = off_bar + 8 * 2 * kNLd;
    // The ring is filled in order, so what counts is the span from the oldest slot still held to the newest one waited for.
    // While chunk n's MMAs run, the conversion of chunk n + 1 waits for chunk n + 1's V, dO, O; chunk n - 1's dO slot holds its
    // staged dV until the conversion has ended (the bulk copy is checked then), chunk n's V and dO are in the MMAs.  From
    // chunk n - 1's dO to chunk n + 1's O that is 8 slots; with fewer the producer could not load chunk n + 1: deadlock.
    // An item's Q / K entries are moved out and released before its chunk 0 is converted, and nothing is held across items
    // (the last dV slot goes back at the end of the item), so they add nothing to this span.
    static_assert(kNLd >= 8, "ring depth: chunk n - 1's dO (staged dV) up to chunk n + 1's O");
    // dK is staged in the P / dS planes: two (fp32) or one (16-bit) swizzled [LK px][128 B] boxes, 1024-byte aligned
    static_assert(off_p % 1024 == 0 && T::kP >= T::kSlot, "dK staging in the P / dS planes");
    static_assert(kBytes <= kBudget, "shared memory budget");
};

// does this item compute delta itself (its ring carries the O chunks)?
__device__ __forceinline__ bool calc_delta(const BwdParams &p, const Item &it) { return p.delta_mode == 0 || (it.col && it.ik == 0); }

template <int LK, typename E, bool PL = false>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_bwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                  const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                  const __grid_constant__ CUtensorMap mvc, const __grid_constant__ CUtensorMap mvr,
                  const __grid_constant__ CUtensorMap mdoc, const __grid_constant__ CUtensorMap mdor,
                  const __grid_constant__ CUtensorMap moc, const __grid_constant__ CUtensorMap mor,
                  const __grid_constant__ CUtensorMap mdqc, const __grid_constant__ CUtensorMap mdqr,
                  const __grid_constant__ CUtensorMap mdkc, const __grid_constant__ CUtensorMap mdkr,
                  const __grid_constant__ CUtensorMap mdvc, const __grid_constant__ CUtensorMap mdvr, BwdParams p)
{
    using T = Tiles<LK, E>;
    using S = BwdSmem<LK, E>;
    constexpr bool H16 = kH16<E>, F16 = kF16<E>;
    constexpr int TERMS = H16 ? 1 : 3;
    constexpr int kNLd = S::kNLd;
    constexpr int kCh = S::kCh;
    constexpr int KP = LK / 16;
    constexpr int kQKBoxes = H16 ? 1 : 2;          // ring entries per Q or K operand (64 channels)
    constexpr uint32_t LOP = T::kPP * T::kPlane;   // P / dS planes: hi block -> lo block
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + S::off_bar);
    uint64_t *full = bars, *empty = bars + kNLd;
    float *dsum = reinterpret_cast<float *>(smem + S::off_dsum);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NCH = p.C / kCh;
    const int KQ = p.Cq / 16;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item_order(p.sp, (int)blockIdx.x + k * (int)gridDim.x, p.lag); };

    if (tid == 0) {
        // empty barriers: one arrival per use of a slot (consumer thread 0, after the barrier or bulk read that ends the use)
        for (int i = 0; i < kNLd; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr); prefetch_tmap(&mvc); prefetch_tmap(&mvr);
        prefetch_tmap(&mdoc); prefetch_tmap(&mdor); prefetch_tmap(&moc); prefetch_tmap(&mor);
        prefetch_tmap(&mdqc); prefetch_tmap(&mdqr); prefetch_tmap(&mdkc); prefetch_tmap(&mdkr); prefetch_tmap(&mdvc); prefetch_tmap(&mdvr);
    }
    __syncthreads();

    if (tid < 128) {
        // =============================== TMA producer ===============================
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0 && lane == 0) {
            // the next ring slot <- the 128-byte TMA box from channel c0 on.  The producer waits for nothing but free slots, so it
            // runs ahead into the next item (its Q, K and first chunks) while the consumers finish this one.
            // No L2 eviction hints (loads or output copies): with evict_last on the producers' operands and stores and
            // evict_first on the rest, the backward was 6 % (fp32) and 1.5 % (bf16) slower at 8x512x97x97 (DESIGN.md 4).
            uint32_t g = 0;
            auto ring = [&](const CUtensorMap *m, int c0, const Item &it, int start) {
                const int slot = g % kNLd;
                mbar_wait(&empty[slot], ((g / kNLd) & 1) ^ 1);
                mbar_expect_tx(&full[slot], S::kRSlot);
                uint8_t *dst = smem + S::off_ld + slot * S::kRSlot;
                const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                tma_load_4d(dst, m, &full[slot], c0, cw, ch, it.b);
                ++g;
            };
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                const bool calc = calc_delta(p, it);
                for (int bx = 0; bx < kQKBoxes; ++bx) ring(it.col ? &mqc : &mqr, 32 * bx, it, it.q0);
                for (int bx = 0; bx < kQKBoxes; ++bx) ring(it.col ? &mkc : &mkr, 32 * bx, it, it.k0);
                for (int n = 0; n < NCH; ++n) {
                    ring(it.col ? &mvc : &mvr, n * kCh, it, it.k0);
                    ring(it.col ? &mdoc : &mdor, n * kCh, it, it.q0);
                    if (calc) ring(it.col ? &moc : &mor, n * kCh, it, it.q0);
                }
            }
        }
    } else {
        // =============================== consumers (warpgroup wg = rows [64 wg, 64 wg + 64) of each product) ===============================
        setmaxnreg_inc<kConsumerRegs>();
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2);         // accumulator rows rbase, rbase + 8
        const int cq = 2 * (lane & 3);                             // first accumulator column of this thread (+ 8j)
        const uint32_t qb = smem_u32(smem + S::off_qk), kb = qb + T::kSlot, ld_base = smem_u32(smem + S::off_ld);
        const uint32_t pb = smem_u32(smem + S::off_p);
        uint8_t *pgen = smem + S::off_p;
        // this thread's accumulator rows rbase, rbase + 8 (nc channels from 0) -> `tile`, laid out as the output's swizzled TMA
        // box(es) [tile px][128 B] (fp32: 32-channel boxes T::kTile apart); rows past LK are padding and are skipped
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
        // (thread 0) the staged boxes -> global: producers store, everybody else reduce-adds
        // (PL: `part` is the plane of the box, sample coordinate part * B + b)
        auto put = [&](const CUtensorMap *m, const uint8_t *tile, int boxes, int c0, int px0, const Item &it, bool prod, int part) {
            const int cw = it.col ? it.line : px0, ch = it.col ? px0 : it.line;
            const int ob = PL ? part * p.sp.B + it.b : it.b;
            for (int bx = 0; bx < boxes; ++bx) {
                const uint8_t *src = tile + bx * T::kTile;
                if (prod) tma_store_4d(m, src, c0 + 32 * bx, cw, ch, ob);
                else tma_reduce_add_4d(m, src, c0 + 32 * bx, cw, ch, ob);
            }
            bulk_commit();
        };
        // dQ / dK boxes: 64 channels (fp32: two boxes; a box wholly past Cq is not issued, TMA clips the rest)
        const int qboxes = H16 ? 1 : (p.Cq > 32 ? 2 : 1);
        pdl_wait();                                                // prep kernel complete: counters (and the outputs) cleared
        uint32_t g = 0;
        int pending = -1;                                          // (thread 0) ring slot whose bulk copy may still be reading it
        int unpublished = -1;                                      // (thread 0) sample of the last producer item, not yet published
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const bool calc = calc_delta(p, it);
            const bool prod = PL || (p.out_mode == 1 && is_producer(it));
            long qpix[2];
            bool qok[2];
            float nlse[2];
            int self[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                qok[h] = r < it.lq;
                qpix[h] = item_pixel(p.sp, it, qok[h] ? r : 0);
                nlse[h] = qok[h] ? -p.lse[qpix[h]] * kLog2e : 0.f;
                self[h] = it.col ? it.q0 + r - it.k0 : -1;
            }
            // ---------------- Q, K: the item's first ring entries -> the Q / K region
            // Every thread reads its part, the consumers meet, then write: the previous item's dK MMAs (both warpgroups) and
            // its dQ copy out of the K region (thread 0's wait_group.read at the end of that item) precede that barrier.
            {
                const uint8_t *src[2 * kQKBoxes];
#pragma unroll
                for (int i = 0; i < 2 * kQKBoxes; ++i) {
                    const uint32_t gi = g + i;
                    mbar_wait(&full[gi % kNLd], (gi / kNLd) & 1);
                    src[i] = smem + S::off_ld + (gi % kNLd) * S::kRSlot;
                }
                if constexpr (H16) {                               // a plain copy: both sides are 1024-byte aligned, so the
                    constexpr int kV = T::kTile / 16, kPer = (kV + kConsumers - 1) / kConsumers;     // swizzle carries over
                    uint4 v[2][kPer];
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int j = 0; j < kPer; ++j)
                            if (t + kConsumers * j < kV) v[i][j] = reinterpret_cast<const uint4 *>(src[i])[t + kConsumers * j];
                    consumers_sync();
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int j = 0; j < kPer; ++j)
                            if (t + kConsumers * j < kV) reinterpret_cast<uint4 *>(smem + S::off_qk + i * T::kSlot)[t + kConsumers * j] = v[i][j];
                    fence_proxy_async();
                    consumers_sync();
                } else {
                    convert_slot<LK, E, 4>(smem + S::off_qk, t, nullptr, src);      // Q0 Q1 K0 K1 -> hi/lo planes of Q, K
                }
                if (t == 0)
                    for (int i = 0; i < 2 * kQKBoxes; ++i) mbar_arrive(&empty[(g + i) % kNLd]);
                g += 2 * kQKBoxes;
            }
            // ---------------- S = Q K^T, P = exp(S - lse) -> planes
            {
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
                wg_wait<0>();
                wg_acc_fence<LK / 2>(acc);
                if (t == 0) {                                      // the previous item's dK copy has read the P / dS planes
                    // Deferred publish of the previous item (a producer): its stores have long completed by now.  It must come
                    // before this item's first counter wait (cdone before chunk 0's dV add, ddone before dS): in the lagged
                    // order an item can consume the very sample the CTA's previous item produced, and would wait for itself.
                    if (unpublished >= 0) {
                        bulk_wait<0>();
                        publish_count(p.cdone + unpublished);
                        unpublished = -1;
                    } else {
                        bulk_wait_read<0>();
                    }
                }
                consumers_sync();
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
                            if constexpr (H16) {
                                *reinterpret_cast<uint32_t *>(d) = pack2<F16>(p0, p1);
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
            // ---------------- per chunk: dP += dO V^T, dV = P^T dO
            // Pipelined over the chunks: chunk n's MMAs run while chunk n + 1 is converted (and its delta dot accumulated); then
            // chunk n is waited for and its V slot released, chunk n + 1's dP is issued, chunk n's dV is staged in its dO slot
            // and stored by one thread with TMA while that dP runs, and chunk n + 1's dV is issued.  The dO slot goes back to
            // the producer at the end of the next conversion, when the copy has long read it.  dP and dV are two commit groups
            // so that the staging (which reads the dV accumulator) overlaps the dP group; the one wait per chunk waits for
            // both.  A second dV accumulator (so that a dV group could stay in flight across the wait) makes ptxas treat the
            // groups chained through dP as one pipeline stage, see the other dV accumulator read inside it and serialise every
            // wgmma of the kernel (C7514); at LK = 112 fp32 it also spills.
            float dp[LK / 2];
            float o[kCh / 2];                                      // dV of the chunk
            float dacc = 0.f;
            const uint32_t per = calc ? 3 : 2;                     // ring slots per chunk: V, dO (, O)
            auto rslot = [&](uint32_t gi) { return gi % kNLd; };
            // fp32: chunk n's V and dO boxes -> hi/lo planes in place, in one pass (the layout of convert_slot with one box each).
            // Every thread reads its part of both (and accumulates the delta dot with O), the consumers meet once, then write.
            // There is no closing barrier: the barrier that follows the previous chunk's wait (or the one after chunk 0's
            // conversion) orders these writes before this chunk's MMAs are issued.
            auto convert_chunk = [&](int n) {
                const uint32_t gv = g + per * n, gd = gv + 1, go = gv + 2;
                mbar_wait(&full[rslot(gv)], (gv / kNLd) & 1);
                mbar_wait(&full[rslot(gd)], (gd / kNLd) & 1);
                if (calc) mbar_wait(&full[rslot(go)], (go / kNLd) & 1);
                uint8_t *vs = smem + S::off_ld + rslot(gv) * S::kRSlot, *ds = smem + S::off_ld + rslot(gd) * S::kRSlot;
                const uint8_t *os = smem + S::off_ld + rslot(go) * S::kRSlot;
                if constexpr (H16) {
                    if (calc) {
                        dacc += convert_slot<LK, E, 1>(ds, t, os);
                        consumers_sync();
                        if (t == 0) mbar_arrive(&empty[rslot(go)]);
                    }
                } else {
                    const int r = t & 127, hq = t >> 7;
                    const int rr = r < LK ? r : LK - 1, sw = rr & 7;
                    float4 raw[2][4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        raw[0][j] = *reinterpret_cast<const float4 *>(vs + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
                        raw[1][j] = *reinterpret_cast<const float4 *>(ds + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
                    }
                    if (calc) {
                        float acc = 0.f;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float4 o = *reinterpret_cast<const float4 *>(os + rr * 128 + (((hq * 4 + j) ^ sw) * 16));
                            const float4 x = raw[1][j];
                            acc += x.x * o.x + x.y * o.y + x.z * o.z + x.w * o.w;
                        }
                        dacc += r < LK ? acc : 0.f;
                    }
                    named_bar_sync(kBarConvert, kConsumers);
                    if (calc && t == 0) mbar_arrive(&empty[rslot(go)]);
                    if (r < LK) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            uint8_t *d = (b ? ds : vs) + r * 16 + hq * 2 * T::kPStride;
#pragma unroll
                            for (int j = 0; j < 2; ++j) {
                                const float4 a = raw[b][2 * j], c = raw[b][2 * j + 1];
                                const float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
                                uint4 hi, lo;
                                split8(v, hi, lo);
                                *reinterpret_cast<uint4 *>(d + j * T::kPStride) = hi;
                                *reinterpret_cast<uint4 *>(d + j * T::kPStride + T::kLoOff) = lo;
                            }
                        }
                    }
                    fence_proxy_async();
                }
            };
            auto issue_dp = [&](int n) {
                const uint32_t gv = g + per * n, gd = gv + 1;
                const uint32_t vb = ld_base + rslot(gv) * S::kRSlot, db = ld_base + rslot(gd) * S::kRSlot;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < kCh / 16; ++ks) {
                    wgmma_ss<LK, F16>(dp, desc_kmaj<LK, E>(db, 64 * wg, ks, false), desc_kmaj<LK, E>(vb, 0, ks, false), n > 0 || ks > 0, 0, 0);
                    if constexpr (TERMS == 3) {
                        wgmma_ss<LK, F16>(dp, desc_kmaj<LK, E>(db, 64 * wg, ks, false), desc_kmaj<LK, E>(vb, 0, ks, true), 1, 0, 0);
                        wgmma_ss<LK, F16>(dp, desc_kmaj<LK, E>(db, 64 * wg, ks, true), desc_kmaj<LK, E>(vb, 0, ks, false), 1, 0, 0);
                    }
                }
                wg_commit();
            };
            auto issue_dv = [&](int n) {
                const uint32_t db = ld_base + rslot(g + per * n + 1) * S::kRSlot;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < KP; ++ks) {
                    const uint32_t pa = pb + 8 * wg * T::kPlane + ks * 256;      // P^T: rows = key pixels [64 wg, +64), k = query rows
                    if constexpr (H16) {
                        wgmma_ss_n64<F16>(o, smem_desc(pa, 128, T::kPlane), desc_mnmaj<LK, E>(db, ks, false), ks > 0, 1, 1);
                    } else {
                        wgmma_ss_n32<1, 1>(o, smem_desc(pa, 128, T::kPlane), desc_mnmaj<LK, E>(db, ks, false), ks > 0);
                        wgmma_ss_n32<1, 1>(o, smem_desc(pa, 128, T::kPlane), desc_mnmaj<LK, E>(db, ks, true), 1);
                        wgmma_ss_n32<1, 1>(o, smem_desc(pa + LOP, 128, T::kPlane), desc_mnmaj<LK, E>(db, ks, false), 1);
                    }
                }
                wg_commit();
            };
            auto release = [&]() {                                 // (thread 0) the previous chunk's dV copy has read its slot
                if (t == 0 && pending >= 0) {
                    bulk_wait_read<0>();
                    mbar_arrive(&empty[pending]);
                    pending = -1;
                }
            };
            convert_chunk(0);
            if constexpr (!H16) consumers_sync();
            issue_dp(0);
            issue_dv(0);
            for (int n = 0; n < NCH; ++n) {
                if (n + 1 < NCH) convert_chunk(n + 1);
                release();
                wg_wait<0>();                                      // chunk n's MMAs are complete in this warpgroup
                wg_acc_fence<kCh / 2>(o);
                if (n == 0 && !prod) {                             // before this item's first reduce-add, no group in flight:
                    if (p.out_mode == 1) wait_count(p.cdone + it.b, (unsigned)p.sp.seg0);   // producers of the sample have stored
                    // the counter's acquire (or the prep kernel's clear, tiled lines) before the reduce-adds
                    if (t == 0) fence_proxy_async_global();
                }
                consumers_sync();                                  // ... and in the other: V and dO are free
                if (t == 0) mbar_arrive(&empty[rslot(g + per * n)]);
                if (n + 1 < NCH) issue_dp(n + 1);
                uint8_t *ds = smem + S::off_ld + rslot(g + per * n + 1) * S::kRSlot;
                stage(o, kCh, ds);
                fence_proxy_async();
                consumers_sync();
                if (t == 0) {
                    put(it.col ? &mdvc : &mdvr, ds, 1, n * kCh, it.k0, it, prod, qtile_part_index(p.sp, it));
                    pending = (int)rslot(g + per * n + 1);
                }
                if (n + 1 < NCH) issue_dv(n + 1);
            }
            wg_wait<0>();                                          // (nothing is pending; ptxas cannot tell which step ran last)
            wg_acc_fence<LK / 2>(dp);
            g += per * NCH;
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
                        const uint32_t lw = H16 ? 0u : *reinterpret_cast<const uint32_t *>(d + LOP);
                        const float p0 = lo2<F16>(hw) + lo2<F16>(lw), p1 = hi2<F16>(hw) + hi2<F16>(lw);
                        // masked / padded entries have P == 0 exactly; rows past the tile are cleared (their dP is not defined)
                        const float s0 = qok[h] ? p0 * (dp[4 * j + 2 * h] - dl[h]) : 0.f;
                        const float s1 = qok[h] ? p1 * (dp[4 * j + 2 * h + 1] - dl[h]) : 0.f;
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
            // ---------------- dQ = dS K (rows = query pixels), dK = dS^T Q (rows = key pixels)
            // Two groups (one accumulator set of 32 live at a time): dQ is staged in the K slot (dK reads dS and Q) and its bulk
            // copy runs with the dK MMAs; dK is staged in the P / dS planes once its MMAs have retired.
            {
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
                consumers_sync();                                  // both warpgroups' dQ MMAs have read the K slot
                stage(aq, 64, smem + S::off_qk + T::kSlot);
                fence_proxy_async();
                consumers_sync();
                if (t == 0) put(it.col ? &mdqc : &mdqr, smem + S::off_qk + T::kSlot, qboxes, 0, it.q0, it, prod, part_index(p.sp, it));
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
                consumers_sync();                                  // both warpgroups' dK MMAs have read dS and Q
                stage(ak, 64, pgen);
                fence_proxy_async();
                consumers_sync();                                  // (also: the planes and dsum are free for the next item)
                if (t == 0) {
                    put(it.col ? &mdkc : &mdkr, pgen, qboxes, 0, it.k0, it, prod, qtile_part_index(p.sp, it));
                    bulk_wait_read<1>();                           // the last dV copy and the dQ copy have read their slots
                    if (pending >= 0) mbar_arrive(&empty[pending]);
                    pending = -1;
                    if (!PL && prod) unpublished = it.b;                  // published once its stores are complete, in the next item
                }
            }
        }
        if (t == 0) {
            bulk_wait<0>();                                        // shared memory must outlive the last bulk reads
            if (unpublished >= 0) publish_count(p.cdone + unpublished);
        }
    }
}

// Prologue of the backward: clears the outputs (tiled lines) and the per-sample counters.  (Internal linkage: every
// translation unit that instantiates launch_bwd has its own copy.)
namespace {
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
}  // namespace

template <int LK, typename E, bool PL> cudaError_t launch_bwd(const BwdArgs &a)
{
    CUtensorMap m[16];
    const Dims &d = a.d;
    BwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    // loads: LK-pixel boxes, zero-filled past the line; outputs: boxes of one tile of the direction, so a store never reaches
    // into the next tile of a line (pixels past the line are not written)
    const int nb = PL ? p.sp.nparts * d.B : d.B, bc = p.sp.col.tl, br = p.sp.row.tl;
    if (cudaError_t e = get_maps(m, {{a.q, d.B, d.Cq, LK, LK}, {a.k, d.B, d.Cq, LK, LK}, {a.v, d.B, d.C, LK, LK},
                                     {a.dout, d.B, d.C, LK, LK}, {a.out, d.B, d.C, LK, LK}, {a.dq, nb, d.Cq, bc, br},
                                     {a.dk, nb, d.Cq, bc, br}, {a.dv, nb, d.C, bc, br}},
                                 d, kDtype<E>, a.why))
        return e;
    p.C = d.C; p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.lse = a.lse; p.delta = a.delta;
    p.ddone = a.counters; p.cdone = a.counters + d.B;
    p.delta_mode = a.delta_mode;
    const bool one_tile = p.sp.col.nt == 1 && p.sp.row.nt == 1;
    p.out_mode = one_tile || PL ? 1 : 0;          // (PL: every item stores; 1 only skips the clear below)
    p.lag = tc_lag() != 0 ? 1 : 0;
    const long es = sizeof(E);
    const long nq = p.out_mode == 1 ? 0 : p.npix * d.Cq * es, nv = p.out_mode == 1 ? 0 : p.npix * d.C * es;
    cca_bwd_prep_kernel<<<p.out_mode == 1 ? 1 : sm_count(), 256, 0, a.st>>>(
        reinterpret_cast<uint4 *>(a.dq), reinterpret_cast<uint4 *>(a.dk), reinterpret_cast<uint4 *>(a.dv), nq / 16, nv / 16, a.counters,
        3 * d.B);
    count_launch();
    if (cudaError_t e = cudaGetLastError()) return e;
    return launch_kernel(cca_tc_bwd_kernel<LK, E, PL>, item_grid(p.sp), kThreads, BwdSmem<LK, E>::kBytes, true, a.st, m[0], m[1], m[2],
                         m[3], m[4], m[5], m[6], m[7], m[8], m[9], m[10], m[11], m[12], m[13], m[14], m[15], p);
}

// The f16 instantiations live in their own translation unit (cca_tc_f16.cu), the planes-mode ones (fp32) in cca_tc_det.cu.
extern template cudaError_t launch_bwd<80, __half>(const BwdArgs &);
extern template cudaError_t launch_bwd<112, __half>(const BwdArgs &);
extern template cudaError_t launch_bwd<80, float, true>(const BwdArgs &);
extern template cudaError_t launch_bwd<112, float, true>(const BwdArgs &);

}  // namespace tc
}  // namespace cca
