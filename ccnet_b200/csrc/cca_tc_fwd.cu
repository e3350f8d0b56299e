// wgmma / TMA forward (values) kernel of criss-cross attention for sm_90a (channels-last tensors).
//
// Layout: q,k [B,H,W,Cq], v,out [B,H,W,C] (torch channels_last).  In this layout an image row and an image column are
// the same object -- L pixels with a fixed pixel stride, each pixel's channels contiguous -- so one kernel serves both
// branches of cc_attention/functions.py:38-47.
//
// Formulation (DESIGN.md 3): the statistics pre-pass (cca_tc_stats.cu) has left the log-sum-exp of every pixel's logits
// per (direction, key block).  An item (cca_items.cuh: direction, sample, line, query tile, key block) combines those few
// planes into the pixel's final lse and computes its share of the output with the FINAL normalisation,
//     P = exp(S - lse)        O_item = P V_block        out[query pixels] += O_item
// so items never exchange anything: no partial output is written and read back, no per-pixel merge, and lines longer
// than one tile are just more items.  ONE persistent launch walks the items sample by sample: the second direction of a
// sample finds q,k,v in L2 and adds onto output lines that are still L2-resident.
//
// Two touches per output element, ordered: the "producer" items of a sample (column lines, first key block) STORE their
// rows, every other item of the sample ADDS onto them (vector reductions at L2) once the per-sample counter cdone[b] says all
// producers have completed their stores.  Items are walked in the lagged order of cca_items.cuh -- P(0) | P(1) C(0) | ... --
// so a consumer practically never waits; only items with a LOWER index are ever waited for and each persistent CTA walks its
// items in increasing order, so the wait cannot cycle.  With one tile per line every output element is one store plus one
// add: the result is bit-reproducible; with key-block tiling a pixel gets 2*nt-1 adds whose order is not fixed.
//
// Roles (cca_tc_common.cuh):
//   producer lane       : Q, K of an item into their own stage; the item's 64-channel V chunks into a ring.  4-D tiled loads,
//                         SWIZZLE_128B, pixels past the line zero-filled.
//   consumer warpgroups : fp32 only: tiles -> bf16 hi + lo planes in place (x = hi + lo to ~2^-17).  S = Q K^T (wgmma, both
//                         operands in shared memory), P = exp2(S log2e - lse2) in registers, re-packed as the bf16 A operand of
//                         O = P V (wgmma with A from registers, 3 MMAs per k-step for fp32 I/O), O rows stored / added
//                         straight from the accumulators.
#include <type_traits>

#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace {
using namespace tc;

struct FwdParams {
    ItemSpace sp;
    int C, Cq;
    long npix;
    const float *parts;    // [nparts][B*H*W] partial log2-sum-exp2 (statistics pre-pass)
    float *lse;            // [B,H,W] natural-log lse (saved for backward)
    void *out;             // [B,H,W,C] fp32 or bf16
    unsigned int *cdone;   // [B] producer items of sample b whose stores have completed (cleared by the statistics kernel)
    int lag;               // item order: 1 = consumers trail the producers by one block, 0 = sample after sample
    int hints;             // L2 eviction hints on the loads
};

template <int LK, bool BF> struct FwdSmem {
    using T = Tiles<LK, BF>;
    static constexpr int off_qk = 0;                               // Q slot, K slot
    static constexpr int off_ld = off_qk + 2 * T::kSlot;           // ring of V chunks
    static constexpr int kNLd = (200 * 1024 - off_ld) / T::kSlot < 8 ? (200 * 1024 - off_ld) / T::kSlot : 8;
    static constexpr int off_tail = off_ld + kNLd * T::kSlot;      // 64-row wgmmas of the second warpgroup read up to
                                                                   // (128 - LK) rows past a tile; they only feed discarded rows
    static constexpr int off_bar = off_tail + (128 - LK) * 128 + 1024;
    static constexpr int kBytes = off_bar + 8 * (2 + 2 * kNLd);
    static_assert(kNLd >= 2, "ring depth");
    static_assert(kBytes <= 232448, "shared memory budget");
};

template <int LK, bool BF>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_fwd_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                  const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr,
                  const __grid_constant__ CUtensorMap mvc, const __grid_constant__ CUtensorMap mvr, FwdParams p)
{
    using T = Tiles<LK, BF>;
    using S = FwdSmem<LK, BF>;
    using E = typename std::conditional<BF, __nv_bfloat16, float>::type;
    constexpr int kNLd = S::kNLd;
    constexpr int TERMS = BF ? 1 : 3;
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
        for (int i = 0; i < kNLd; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumers); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr); prefetch_tmap(&mvc); prefetch_tmap(&mvr);
    }
    __syncthreads();

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
            auto load = [&](uint8_t *dst, uint64_t *bar, const CUtensorMap *m, int c0, const Item &it, int start) {
                const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                if (p.hints == 1) {     // producers' operands are read again by the sample's consumers; theirs are not
                    const uint64_t pol = is_producer(it) ? pol_keep : pol_stream;
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b, pol);
                    if constexpr (!BF) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b, pol);
                } else {
                    tma_load_4d(dst, m, bar, c0, cw, ch, it.b);
                    if constexpr (!BF) tma_load_4d(dst + T::kTile, m, bar, c0 + 32, cw, ch, it.b);
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
    } else if (tid >= 128) {
        // =============================== consumers (warpgroup wg = query rows [64 wg, 64 wg + 64)) ===============================
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        const int rbase = 64 * wg + 16 * wq + (lane >> 2);         // rows rbase, rbase + 8 of the accumulators
        const uint32_t qb = smem_u32(smem + S::off_qk), kb = qb + T::kSlot, ld_base = smem_u32(smem + S::off_ld);
        E *const out = reinterpret_cast<E *>(p.out);
        pdl_wait();                                                // parts and the counters come from the statistics kernel
        uint32_t g = 0;
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const bool prod = is_producer(it);
            // ---- S = Q K^T
            mbar_wait(qk_full, k & 1);
            if constexpr (!BF) {
                convert_slot<LK, BF>(smem + S::off_qk, t);
                convert_slot<LK, BF>(smem + S::off_qk + T::kSlot, t);
            }
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
            mbar_arrive(qk_empty);
            // ---- P = exp2(S log2e - lse2) for rows rbase (h = 0), rbase + 8 (h = 1), as bf16 A fragments (hi, lo)
            long pix[2];
            float nlse[2];
            int self[2];
            bool rok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                rok[h] = r < it.lq;
                pix[h] = item_pixel(p.sp, it, rok[h] ? r : 0);
                self[h] = it.col ? it.q0 + r - it.k0 : -1;
                float lse2 = 0.f;
                if (rok[h]) {
                    float m = -INFINITY;
                    for (int i = 0; i < p.sp.nparts; ++i) m = fmaxf(m, __ldcg(p.parts + (long)i * p.npix + pix[h]));
                    float sum = 0.f;
                    for (int i = 0; i < p.sp.nparts; ++i) sum += exp2f(__ldcg(p.parts + (long)i * p.npix + pix[h]) - m);
                    lse2 = m + log2f(sum);
                    if (!it.col && it.ik == 0 && (lane & 3) == 0) p.lse[pix[h]] = lse2 * kLn2;
                }
                nlse[h] = -lse2;
            }
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
                    if constexpr (BF) {
                        ph[j / 2][reg] = pack_bf16(p0, p1);
                        pl[j / 2][reg] = 0u;
                    } else {
                        split2(p0, p1, ph[j / 2][reg], pl[j / 2][reg]);
                    }
                }
            if (!prod) wait_count(p.cdone + it.b, (unsigned)p.sp.seg0);   // every producer of this sample has stored its rows
            // ---- O = P V, 64 channels at a time
            for (int n = 0; n < NCH; ++n, ++g) {
                const int slot = g % kNLd;
                mbar_wait(&full[slot], (g / kNLd) & 1);
                if constexpr (!BF) convert_slot<LK, BF>(smem + S::off_ld + slot * T::kSlot, t);
                const uint32_t vb = ld_base + slot * T::kSlot;
                float o[32];
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < KP; ++ks) {
                    wgmma_rs_n64_tb(o, ph[ks], desc_mnmaj<LK, BF>(vb, ks, false), ks > 0);
                    if constexpr (TERMS == 3) {
                        wgmma_rs_n64_tb(o, ph[ks], desc_mnmaj<LK, BF>(vb, ks, true), 1);
                        wgmma_rs_n64_tb(o, pl[ks], desc_mnmaj<LK, BF>(vb, ks, false), 1);
                    }
                }
                wg_commit();
                wg_wait<0>();
                wg_acc_fence<32>(o);
                mbar_arrive(&empty[slot]);
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (rok[h]) {
                        E *row = out + pix[h] * p.C + n * kNC + 2 * (lane & 3);
#pragma unroll
                        for (int j = 0; j < 8; ++j) put2(row + 8 * j, o[4 * j + 2 * h], o[4 * j + 2 * h + 1], !prod);
                    }
            }
            if (prod) {                                            // publish: all stores of this item are visible
                __threadfence();
                consumers_sync();
                if (t == 0) atomicAdd(p.cdone + it.b, 1u);
            }
        }
    }
}

template <int LK, bool BF>
cudaError_t launch_fwd(const void *q, const void *k, const void *v, void *out, float *lse, const float *parts, unsigned int *cdone,
                       Dims d, cudaStream_t st, const char **why)
{
    CUtensorMap m[6];
    const void *base[3] = {q, k, v};
    const int ch[3] = {d.Cq, d.Cq, d.C};
    FwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    for (int t = 0; t < 3; ++t)
        for (int r = 0; r < 2; ++r)
            // LK-pixel boxes: pixels past the line are zero-filled
            if (!get_map(&m[2 * t + r], base[t], d.B, d.H, d.W, ch[t], LK, r == 0, BF)) {
                if (why) *why = "cuTensorMapEncodeTiled failed";
                return cudaErrorInvalidValue;
            }
    p.C = d.C; p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = parts; p.lse = lse; p.cdone = cdone; p.out = out;
    p.lag = tc_lag() != 0 ? 1 : 0;                 // default (-1): lagged
    p.hints = tc_l2_hints();
    auto kern = cca_tc_fwd_kernel<LK, BF>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FwdSmem<LK, BF>::kBytes);
    if (e != cudaSuccess) return e;
    const int sms = sm_count();
    const int grid = p.sp.total < sms ? p.sp.total : sms;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = FwdSmem<LK, BF>::kBytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = tc_pdl() ? 1 : 0;     // may start ahead of the statistics kernel's completion (griddepcontrol.wait inside)
    e = cudaLaunchKernelEx(&cfg, kern, m[0], m[1], m[2], m[3], m[4], m[5], p);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace

bool tc_forward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

// Workspace of the forward: [nparts][B*H*W] fp32 partial lse planes, then [B] unsigned per-sample counters.
size_t tc_forward_workspace(Dims d)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const size_t parts = (size_t)sp.nparts * d.B * d.H * d.W * sizeof(float);
    return ((parts + 15) & ~(size_t)15) + (((size_t)d.B * sizeof(unsigned int) + 15) & ~(size_t)15);
}

// q,k,v,out are channels-last (NHWC), fp32 or bf16.  Two launches: statistics pre-pass (q,k only), values.
cudaError_t tc_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims d, int dtype,
                       cudaStream_t st, const char **why)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const long npix = (long)d.B * d.H * d.W;
    float *parts = reinterpret_cast<float *>(ws);
    const size_t parts_bytes = ((size_t)sp.nparts * npix * sizeof(float) + 15) & ~(size_t)15;
    unsigned int *cdone = reinterpret_cast<unsigned int *>(reinterpret_cast<uint8_t *>(ws) + parts_bytes);
    const bool bf = dtype == CCA_BF16;
    // statistics; it also clears the per-sample counters of the values kernel
    cudaError_t e = tc_stats(q, k, parts, nullptr, 0, cdone, d.B, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    const int lk = lk_for(max_tile(sp));
    if (bf)
        return lk == 80 ? launch_fwd<80, true>(q, k, v, out, lse, parts, cdone, d, st, why)
                        : launch_fwd<112, true>(q, k, v, out, lse, parts, cdone, d, st, why);
    return lk == 80 ? launch_fwd<80, false>(q, k, v, out, lse, parts, cdone, d, st, why)
                    : launch_fwd<112, false>(q, k, v, out, lse, parts, cdone, d, st, why);
}

}  // namespace cca
