// Thin inline-PTX layer for the Hopper (sm_90a) features the tensor-core kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMAs (wgmma.mma_async) and their shared-memory descriptors, proxy fences.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Debug builds (-DCCA_SPIN_TRAP=1, `python -m ccnet_b200.build --debug`): a broken pipeline traps after a bounded spin
// instead of hanging the GPU.  Release builds wait without a bound (a trap would take the whole CUDA context of a
// training job with it).
#ifndef CCA_SPIN_TRAP
#define CCA_SPIN_TRAP 0
#endif
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
#if CCA_SPIN_TRAP
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) { __trap(); }
    }
#else
    while (!mbar_try_wait(bar, parity)) {}
#endif
}
// Spin until a global counter (bumped with a release by other CTAs) reaches `need`.
__device__ __forceinline__ void wait_count(const unsigned int *cnt, unsigned int need)
{
    unsigned int v;
#if CCA_SPIN_TRAP
    unsigned int spins = 0;
#endif
    for (;;) {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(cnt) : "memory");
        if (v >= need) return;
        __nanosleep(64);
#if CCA_SPIN_TRAP
        if (++spins > (1u << 24)) __trap();
#endif
    }
}
// ---------------------------------------------------------------- programmatic dependent launch
// launch_dependents: the next kernel in the stream (if it was launched with the programmatic-serialization attribute) may be
// scheduled once every CTA of this grid has executed this (or exited); wait: blocks until the grids this one depends on have
// completed and flushed their memory (returns at once for a normal launch).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- register reallocation between warpgroups
// Every warp of the warpgroup executes these (.sync.aligned).  dec hands registers back to the CTA's pool, inc blocks until the
// pool holds enough: the counts of all warpgroups must fit the registers the kernel was launched with.
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------- proxy fences
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *m)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1, int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// L2 eviction-priority policies (createpolicy) and the hinted form of the 4-D tensor load
__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1, int c2, int c3, uint64_t pol)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol)
        : "memory");
}
// 4-D tensor stores shared -> global (bulk groups): plain store, and reduce-add performed at L2 (element type of the tensor
// map).  The shared tile is written by the generic proxy, so the writers run fence_proxy_async() before the issuing thread
// is released to issue.  Box elements past the tensor's extent are not written.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *m, const void *src, int c0, int c1, int c2, int c3)
{
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *m, const void *src, int c0, int c1, int c2, int c3, uint64_t pol)
{
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4, %5}], [%1], %6;"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap *m, const void *src, int c0, int c1, int c2, int c3)
{
    asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap *m, const void *src, int c0, int c1, int c2, int c3, uint64_t pol)
{
    asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group.L2::cache_hint [%0, {%2, %3, %4, %5}], [%1], %6;"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol) : "memory");
}
// bulk groups of the issuing thread: commit the stores issued since the last commit; wait until at most N groups are
// pending (wait: their writes are complete; wait_read: they have finished reading shared memory, which may then be reused)
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// orders this thread's generic-proxy accesses of global memory (e.g. an acquire of a counter) with its async-proxy ones
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// publish a counter: everything this thread's completed bulk stores wrote (bulk_wait<0> first) happens-before the bump
__device__ __forceinline__ void publish_count(unsigned int *cnt)
{
    fence_proxy_async_global();
    __threadfence();
    atomicAdd(cnt, 1u);
}

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor of wgmma (start >> 4 [0,14), lbo >> 4 [16,30), sbo >> 4 [32,46), layout [62,64)).
//   layout 0 (no swizzle, core matrices of 8 rows x 16 B):
//     K-major operand : next 16 B of K at lbo, next 8 M/N rows at sbo
//     MN-major operand: next 16 B of M/N at sbo, next 8 K rows at lbo
//   layout kSw128 (a TMA tile of 128-byte rows, SWIZZLE_128B, 1024-byte aligned atoms of 8 rows):
//     K-major operand : rows = M/N, next 8 rows at sbo (1024); a k-step of 16 elements advances the start by 32 B
//     MN-major operand: rows = K, 64 bf16 of M/N per row, next 8 K rows at sbo (1024); a k-step advances the start by 2048 B
constexpr uint32_t kSw128 = 1;
__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout_type = 0)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)(layout_type & 3) << 62;
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads above a wg_wait
template <int R> __device__ __forceinline__ void wg_acc_fence(float *d)
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[16 x N], 16-bit inputs (F16 = false: bf16, true: f16), fp32 accumulators in registers (d: N/2
// floats per thread; thread (warp w of the warpgroup, lane l) holds rows 16w + l/4 and +8, columns 8j + 2(l%4) + {0,1}:
// d[4j + {0,1}] and d[4j + {2,3}]).
// ss: both operands from shared memory (ta / tb: 1 = MN-major); rs: A from registers (four packed pairs in the accumulator
// layout of a 16-column slice: rows r, r+8 x columns 2(l%4), +8), B MN-major.
// The operand type is part of the instruction text: AB is "bf16.bf16" or "f16.f16"; ta / tb are immediates.
#define CCA_WGMMA_SS_N64(AB, TA, TB) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n" \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32." AB " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, " #TA ", " #TB ";\n}" \
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) : "l"(a), "l"(b), "r"(scale_d))
#define CCA_WGMMA_SS_N80(AB, TA, TB) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n" \
    "wgmma.mma_async.sync.aligned.m64n80k16.f32." AB " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, " #TA ", " #TB ";\n}" \
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]) : "l"(a), "l"(b), "r"(scale_d))
#define CCA_WGMMA_SS_N112(AB, TA, TB) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %58, 0;\n" \
    "wgmma.mma_async.sync.aligned.m64n112k16.f32." AB " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, " #TA ", " #TB ";\n}" \
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]) : "l"(a), "l"(b), "r"(scale_d))
// the four transpose forms of one ss instruction, selected by the (inlined, constant) ta / tb
#define CCA_WGMMA_SS_T(OP, AB) \
    if (ta == 0 && tb == 0) OP(AB, 0, 0); \
    else if (ta == 0) OP(AB, 0, 1); \
    else if (tb == 0) OP(AB, 1, 0); \
    else OP(AB, 1, 1)
template <bool F16 = false> __device__ __forceinline__ void wgmma_ss_n64(float *d, uint64_t a, uint64_t b, int scale_d, int ta, int tb)
{
    if constexpr (F16) { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N64, "f16.f16"); }
    else { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N64, "bf16.bf16"); }
}
// m64n32k16 (the 32-channel dV chunks of the fp32 backward); ta / tb are compile-time here
template <int TA, int TB> __device__ __forceinline__ void wgmma_ss_n32(float *d, uint64_t a, uint64_t b, int scale_d)
{
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <bool F16 = false> __device__ __forceinline__ void wgmma_ss_n80(float *d, uint64_t a, uint64_t b, int scale_d, int ta, int tb)
{
    if constexpr (F16) { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N80, "f16.f16"); }
    else { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N80, "bf16.bf16"); }
}
template <bool F16 = false> __device__ __forceinline__ void wgmma_ss_n112(float *d, uint64_t a, uint64_t b, int scale_d, int ta, int tb)
{
    if constexpr (F16) { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N112, "f16.f16"); }
    else { CCA_WGMMA_SS_T(CCA_WGMMA_SS_N112, "bf16.bf16"); }
}
#define CCA_WGMMA_RS_N64(AB) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n" \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32." AB " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}" \
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d))
template <bool F16 = false> __device__ __forceinline__ void wgmma_rs_n64_tb(float *d, const uint32_t *a, uint64_t b, int scale_d)
{
    if constexpr (F16) CCA_WGMMA_RS_N64("f16.f16");
    else CCA_WGMMA_RS_N64("bf16.bf16");
}

// dispatch on N for the S / dP products (N = key pixels of a tile)
template <int N, bool F16 = false> __device__ __forceinline__ void wgmma_ss(float *d, uint64_t a, uint64_t b, int scale_d, int ta, int tb)
{
    static_assert(N == 64 || N == 80 || N == 112, "wgmma width");
    if constexpr (N == 64) wgmma_ss_n64<F16>(d, a, b, scale_d, ta, tb);
    else if constexpr (N == 80) wgmma_ss_n80<F16>(d, a, b, scale_d, ta, tb);
    else wgmma_ss_n112<F16>(d, a, b, scale_d, ta, tb);
}

}  // namespace sm90
