// C ABI of the operator (include/cca_b200.h): argument validation, kernel-family dispatch,
// host-buffer variants.  No torch types anywhere in this library.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "cca_common.cuh"
#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace {
thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};

int fail(int code, const char *fmt, const char *a = "", const char *b = "")
{
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}
int cuda_fail(cudaError_t e, const char *where)
{
    return fail(CCA_ERR_CUDA, "CUDA error in %s: %s", where, cudaGetErrorString(e));
}

int check_dims(int B, int Cq, int C, int H, int W, int dtype)
{
    if (B <= 0 || Cq <= 0 || C <= 0 || H <= 0 || W <= 0)
        return fail(CCA_ERR_INVALID, "non-positive dimension%s%s");
    if (dtype != CCA_F32 && dtype != CCA_BF16) return fail(CCA_ERR_INVALID, "dtype must be CCA_F32 or CCA_BF16%s%s");
    if ((long long)B * C * H * W >= (1ll << 40)) return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");
    return CCA_OK;
}
size_t esize(int dtype) { return dtype == CCA_F32 ? 4 : 2; }
}  // namespace

void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

namespace {
int env_int(const char *name, int dflt, int lo, int hi)
{
    const char *e = getenv(name);
    if (!e) return dflt;
    const int v = atoi(e);
    return v < lo || v > hi ? dflt : v;
}
constexpr int kUnset = -1000;
std::atomic<int> g_pdl{kUnset}, g_zero_ahead{kUnset}, g_delta{kUnset}, g_lag{kUnset}, g_hints{kUnset};
int knob(std::atomic<int> &g, const char *name, int dflt, int lo, int hi)
{
    int v = g.load(std::memory_order_relaxed);
    if (v == kUnset) {
        v = env_int(name, dflt, lo, hi);
        g.store(v, std::memory_order_relaxed);      // racing first calls compute the same value
    }
    return v;
}
}  // namespace
int tc_pdl() { return knob(g_pdl, "CCA_B200_PDL", 1, 0, 1); }
int tc_zero_ahead() { return knob(g_zero_ahead, "CCA_B200_ZERO_AHEAD", 1, 1, 4); }
int tc_delta_mode() { return knob(g_delta, "CCA_B200_DELTA", -1, -1, 1); }
int tc_lag() { return knob(g_lag, "CCA_B200_LAG", -1, -1, 1); }
int tc_l2_hints() { return knob(g_hints, "CCA_B200_L2HINT", 1, 0, 2); }
#ifdef CCA_DEBUG_HOOKS
void set_tc_pdl(int on) { g_pdl.store(on ? 1 : 0); }
void set_tc_zero_ahead(int n) { g_zero_ahead.store(n < 1 ? 1 : (n > 4 ? 4 : n)); }
void set_tc_delta_mode(int m) { g_delta.store(m < -1 || m > 1 ? -1 : m); }
void set_tc_lag(int v) { g_lag.store(v < -1 || v > 1 ? -1 : v); }
void set_tc_l2_hints(int v) { g_hints.store(v < 0 || v > 2 ? 1 : v); }
#endif
}  // namespace cca

using namespace cca;

extern "C" {

int cca_b200_version(void) { return CCA_B200_VERSION; }
#ifdef CCA_DEBUG_HOOKS
// A/B aids of debug builds (`python -m ccnet_b200.build --debug`); not part of the ABI, absent from release builds
CCA_API void cca_b200__set_pdl(int on) { set_tc_pdl(on); }
CCA_API void cca_b200__set_zero_ahead(int n) { set_tc_zero_ahead(n); }
CCA_API void cca_b200__set_delta_mode(int m) { set_tc_delta_mode(m); }
CCA_API void cca_b200__set_lag(int v) { set_tc_lag(v); }
CCA_API void cca_b200__set_l2_hints(int v) { set_tc_l2_hints(v); }
#endif
const char *cca_b200_last_error(void) { return g_err; }
const char *cca_b200_strerror(int s)
{
    switch (s) {
        case CCA_OK: return "ok";
        case CCA_ERR_INVALID: return "invalid argument";
        case CCA_ERR_UNSUPPORTED: return "unsupported shape";
        case CCA_ERR_WORKSPACE: return "workspace too small";
        case CCA_ERR_CUDA: return "CUDA error";
        case CCA_ERR_DEVICE: return "device is not sm_90";
        default: return "unknown status";
    }
}
unsigned long long cca_b200_launch_count(void) { return g_launches.load(); }

namespace {
// compute capability major of the current device, cached per device id (0 on failure)
int device_major()
{
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (dev < 0 || dev >= 64) dev = 0;
    int v = cache[dev].load(std::memory_order_relaxed);
    if (v == 0) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
        v = major;
        cache[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}
int check_device()
{
    const int major = device_major();
    if (major == 0) return fail(CCA_ERR_CUDA, "cannot query the current CUDA device%s%s");
    if (major != 9) return fail(CCA_ERR_DEVICE, "the current device is not sm_90 (H100); this library has no other code path%s%s");
    return CCA_OK;
}
}  // namespace

int cca_b200_device_ok(void)
{
    int dev = 0, major = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceGetAttribute");
    return major == 9 ? 1 : 0;
}

int cca_b200_tc_supported(int which, int B, int Cq, int C, int H, int W, int dtype)
{
    if (check_dims(B, Cq, C, H, W, dtype)) return 0;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0 && device_major() != 9) return 0;   // (no device at all: shape answer only)
    const Dims d{B, Cq, C, H, W};
    return (which == CCA_WS_BACKWARD ? tc_backward_supported(d, dtype) : tc_forward_supported(d, dtype)) ? 1 : 0;
}

size_t cca_b200_workspace_bytes(int which, int B, int Cq, int C, int H, int W, int dtype)
{
    (void)dtype;
    if (B <= 0 || Cq <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
    const Dims d{B, Cq, C, H, W};
    const size_t pix = (size_t)B * H * W;
    // generic kernels: per-pixel (m,l) of the column pass (forward) / delta (backward); tensor-core kernels: partial lse
    // planes + zero-ahead counters (forward) / delta + counters (backward).  One size that covers whichever family runs.
    const size_t simt = (which == CCA_WS_FORWARD ? pix * sizeof(float2) : pix * sizeof(float)) + 16;
    const size_t tcb = which == CCA_WS_FORWARD ? tc_forward_workspace(d) : tc_backward_workspace(d);
    return simt > tcb ? simt : tcb;
}

void cca_b200_item_space(int B, int H, int W, int *out8)
{
    const tc::ItemSpace s = tc::make_space(B, H, W);
    out8[0] = s.total; out8[1] = s.per_sample; out8[2] = s.seg0; out8[3] = s.seg1; out8[4] = s.seg2;
    out8[5] = s.col.nt; out8[6] = s.row.nt; out8[7] = tc::lk_for(tc::max_tile(s));
}
void cca_b200_decode_item(int B, int H, int W, int index, int lagged, int *out10)
{
    const tc::ItemSpace s = tc::make_space(B, H, W);
    const tc::Item it = tc::decode_item_order(s, index, lagged);
    out10[0] = it.col; out10[1] = it.b; out10[2] = it.line; out10[3] = it.iq; out10[4] = it.ik;
    out10[5] = it.q0; out10[6] = it.lq; out10[7] = it.k0; out10[8] = it.lk; out10[9] = it.j;
}

int cca_b200_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, size_t ws_bytes,
                     int B, int Cq, int C, int H, int W, int dtype, unsigned flags, void *stream)
{
    int rc = check_dims(B, Cq, C, H, W, dtype);
    if (rc) return rc;
    if (!q || !k || !v || !out || !lse || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes(CCA_WS_FORWARD, B, Cq, C, H, W, dtype))
        return fail(CCA_ERR_WORKSPACE, "forward workspace too small%s%s");
    if ((flags & CCA_FLAG_FORCE_SIMT) && (flags & CCA_FLAG_FORCE_TC))
        return fail(CCA_ERR_INVALID, "FORCE_SIMT and FORCE_TC are exclusive%s%s");
    if ((rc = check_device())) return rc;
    const Dims d{B, Cq, C, H, W};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const char *why = "";
    const bool nhwc = (flags & CCA_FLAG_NHWC) != 0;
    const bool tc_ok = nhwc && tc_forward_supported(d, dtype);
    if ((flags & CCA_FLAG_FORCE_TC) && !tc_ok)
        return fail(CCA_ERR_UNSUPPORTED, "tensor-core forward needs CCA_FLAG_NHWC and a covered shape%s%s");
    if (nhwc && (!tc_ok || (flags & CCA_FLAG_FORCE_SIMT)))
        return fail(CCA_ERR_UNSUPPORTED, "channels-last tensors are only handled by the tensor-core kernels; pass NCHW%s%s");
    cudaError_t e;
    if (tc_ok) {
        if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
             reinterpret_cast<uintptr_t>(out)) & 15)
            return fail(CCA_ERR_INVALID, "tensor-core path needs 16-byte aligned tensors%s%s");
        e = tc_forward(q, k, v, out, lse, ws, d, dtype, st, &why);
        if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "tc_forward");
        return CCA_OK;
    }
    if (!simt_supported(d, false)) return fail(CCA_ERR_UNSUPPORTED, "H or W too large for the generic kernels%s%s");
    e = simt_forward(q, k, v, out, lse, ws, d, dtype, st, &why);
    if (e != cudaSuccess) return cuda_fail(e, "simt_forward");
    return CCA_OK;
}

int cca_b200_backward(const void *dout, const void *q, const void *k, const void *v, const void *out,
                      const float *lse, void *dq, void *dk, void *dv, void *ws, size_t ws_bytes,
                      int B, int Cq, int C, int H, int W, int dtype, unsigned flags, void *stream)
{
    int rc = check_dims(B, Cq, C, H, W, dtype);
    if (rc) return rc;
    if (!dout || !q || !k || !v || !out || !lse || !dq || !dk || !dv || !ws)
        return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes(CCA_WS_BACKWARD, B, Cq, C, H, W, dtype))
        return fail(CCA_ERR_WORKSPACE, "backward workspace too small%s%s");
    if ((flags & CCA_FLAG_FORCE_SIMT) && (flags & CCA_FLAG_FORCE_TC))
        return fail(CCA_ERR_INVALID, "FORCE_SIMT and FORCE_TC are exclusive%s%s");
    if ((rc = check_device())) return rc;
    const Dims d{B, Cq, C, H, W};
    const char *why = "";
    const bool nhwc = (flags & CCA_FLAG_NHWC) != 0;
    const bool tc_ok = nhwc && tc_backward_supported(d, dtype);
    if ((flags & CCA_FLAG_FORCE_TC) && !tc_ok)
        return fail(CCA_ERR_UNSUPPORTED, "tensor-core backward needs CCA_FLAG_NHWC and a covered shape%s%s");
    if (nhwc && (!tc_ok || (flags & CCA_FLAG_FORCE_SIMT)))
        return fail(CCA_ERR_UNSUPPORTED, "channels-last tensors are only handled by the tensor-core kernels; pass NCHW%s%s");
    if (tc_ok) {
        if ((reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) |
             reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(dq) |
             reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv)) & 15)
            return fail(CCA_ERR_INVALID, "tensor-core path needs 16-byte aligned tensors%s%s");
        cudaError_t e = tc_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d, dtype,
                                    reinterpret_cast<cudaStream_t>(stream), &why);
        if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "tc_backward");
        return CCA_OK;
    }
    if (!simt_supported(d, true)) return fail(CCA_ERR_UNSUPPORTED, "H or W too large for the generic kernels%s%s");
    cudaError_t e = simt_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d, dtype,
                                  reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, "simt_backward");
    return CCA_OK;
}

// ---------------------------------------------------------------------------------------
// 1x1 Q/K/V projections (functions.py:29,32,35) as tensor-core GEMMs on the channels-last view
// ---------------------------------------------------------------------------------------
int cca_b200_qkv_supported(int C, int Cq)
{
    if (C <= 0 || Cq <= 0) return 0;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0 && device_major() != 9) return 0;
    return qkv_gemm_supported(C, Cq) ? 1 : 0;
}
size_t cca_b200_qkv_workspace_bytes(int C, int Cq) { return C > 0 && Cq > 0 ? qkv_gemm_workspace(C, Cq) : 0; }

int cca_b200_qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk, const float *wv,
                         const float *bv, float *q, float *k, float *v, void *ws, size_t ws_bytes, long long pixels, int C, int Cq,
                         void *stream)
{
    if (!x || !wq || !bq || !wk || !bk || !wv || !bv || !q || !k || !v || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (pixels <= 0 || pixels >= (1ll << 31) || C <= 0 || Cq <= 0) return fail(CCA_ERR_INVALID, "bad dimension%s%s");
    if (ws_bytes < qkv_gemm_workspace(C, Cq)) return fail(CCA_ERR_WORKSPACE, "projection workspace too small%s%s");
    int rc = check_device();
    if (rc) return rc;
    if (!qkv_gemm_supported(C, Cq)) return fail(CCA_ERR_UNSUPPORTED, "projection GEMM needs C %% 64 == 0 and Cq %% 64 == 0%s%s");
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
         reinterpret_cast<uintptr_t>(ws)) & 15)
        return fail(CCA_ERR_INVALID, "projection GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project(x, wq, bq, wk, bk, wv, bv, q, k, v, ws, (long)pixels, C, Cq, reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project");
    return CCA_OK;
}

int cca_b200_qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk, const float *wv,
                               const float *scale, float *dx, void *ws, size_t ws_bytes, long long pixels, int C, int Cq,
                               int accumulate, void *stream)
{
    if (!dq || !dk || !dv || !wq || !wk || !wv || !dx || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (pixels <= 0 || pixels >= (1ll << 31) || C <= 0 || Cq <= 0) return fail(CCA_ERR_INVALID, "bad dimension%s%s");
    if (ws_bytes < qkv_gemm_workspace(C, Cq)) return fail(CCA_ERR_WORKSPACE, "projection workspace too small%s%s");
    int rc = check_device();
    if (rc) return rc;
    if (!qkv_gemm_supported(C, Cq)) return fail(CCA_ERR_UNSUPPORTED, "projection GEMM needs C %% 64 == 0 and Cq %% 64 == 0%s%s");
    if ((reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(dq) | reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv) |
         reinterpret_cast<uintptr_t>(ws)) & 15)
        return fail(CCA_ERR_INVALID, "projection GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project_dgrad(dq, dk, dv, wq, wk, wv, scale, dx, ws, (long)pixels, C, Cq, accumulate,
                                      reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project_dgrad");
    return CCA_OK;
}

int cca_b200_qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                               float *dwk, float *dwv, float *db, long long pixels, int C, int Cq, void *stream)
{
    if (!x || !dq || !dk || !dv || !dwq || !dwk || !dwv) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (pixels <= 0 || pixels >= (1ll << 31) || C <= 0 || Cq <= 0) return fail(CCA_ERR_INVALID, "bad dimension%s%s");
    int rc = check_device();
    if (rc) return rc;
    if (!qkv_wgrad_supported(C, Cq)) return fail(CCA_ERR_UNSUPPORTED, "weight-gradient GEMM needs C %% 256 == 0 and Cq %% 64 == 0%s%s");
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dq) | reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv) |
         reinterpret_cast<uintptr_t>(dwq) | reinterpret_cast<uintptr_t>(dwk) | reinterpret_cast<uintptr_t>(dwv)) & 15)
        return fail(CCA_ERR_INVALID, "weight-gradient GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project_wgrad(x, dq, dk, dv, scale, dwq, dwk, dwv, db, (long)pixels, C, Cq, reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project_wgrad");
    return CCA_OK;
}
int cca_b200_qkv_wgrad_supported(int C, int Cq)
{
    if (C <= 0 || Cq <= 0) return 0;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0 && device_major() != 9) return 0;
    return qkv_wgrad_supported(C, Cq) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------
// host-buffer variants
// ---------------------------------------------------------------------------------------
namespace {
struct DevBufs {
    static constexpr int kMax = 12;
    void *p[kMax] = {};
    int n = 0;
    cudaStream_t st = nullptr;
    ~DevBufs()
    {
        for (int i = 0; i < n; ++i) cudaFree(p[i]);
        if (st) cudaStreamDestroy(st);
    }
    void *alloc(size_t bytes, cudaError_t &e)
    {
        void *r = nullptr;
        if (e == cudaSuccess) e = cudaMalloc(&r, bytes ? bytes : 1);
        if (e == cudaSuccess) p[n++] = r;
        return r;
    }
};
}  // namespace

int cca_b200_forward_host(const void *q, const void *k, const void *v, void *out, float *lse,
                          int B, int Cq, int C, int H, int W, int dtype, unsigned flags)
{
    int rc = check_dims(B, Cq, C, H, W, dtype);
    if (rc) return rc;
    if (!q || !k || !v || !out || !lse) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    const size_t px = (size_t)B * H * W, es = esize(dtype);
    const size_t nq = px * Cq * es, nv = px * C * es, nl = px * sizeof(float);
    const size_t nws = cca_b200_workspace_bytes(CCA_WS_FORWARD, B, Cq, C, H, W, dtype);
    DevBufs d;
    cudaError_t e = cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking);
    void *dq = d.alloc(nq, e), *dk = d.alloc(nq, e), *dv = d.alloc(nv, e), *dout = d.alloc(nv, e);
    void *dl = d.alloc(nl, e), *dws = d.alloc(nws, e);
    if (e != cudaSuccess) return cuda_fail(e, "forward_host alloc");
    if ((e = cudaMemcpyAsync(dq, q, nq, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(dk, k, nq, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(dv, v, nv, cudaMemcpyHostToDevice, d.st)) != cudaSuccess)
        return cuda_fail(e, "forward_host H2D");
    rc = cca_b200_forward(dq, dk, dv, dout, (float *)dl, dws, nws, B, Cq, C, H, W, dtype, flags, d.st);
    if (rc) return rc;
    if ((e = cudaMemcpyAsync(out, dout, nv, cudaMemcpyDeviceToHost, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(lse, dl, nl, cudaMemcpyDeviceToHost, d.st)) != cudaSuccess ||
        (e = cudaStreamSynchronize(d.st)) != cudaSuccess)
        return cuda_fail(e, "forward_host D2H");
    return CCA_OK;
}

int cca_b200_backward_host(const void *dout, const void *q, const void *k, const void *v, const void *out,
                           const float *lse, void *dq, void *dk, void *dv,
                           int B, int Cq, int C, int H, int W, int dtype, unsigned flags)
{
    int rc = check_dims(B, Cq, C, H, W, dtype);
    if (rc) return rc;
    if (!dout || !q || !k || !v || !out || !lse || !dq || !dk || !dv) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    const size_t px = (size_t)B * H * W, es = esize(dtype);
    const size_t nq = px * Cq * es, nv = px * C * es, nl = px * sizeof(float);
    const size_t nws = cca_b200_workspace_bytes(CCA_WS_BACKWARD, B, Cq, C, H, W, dtype);
    DevBufs d;
    cudaError_t e = cudaStreamCreateWithFlags(&d.st, cudaStreamNonBlocking);
    void *g = d.alloc(nv, e), *tq = d.alloc(nq, e), *tk = d.alloc(nq, e), *tv = d.alloc(nv, e), *to = d.alloc(nv, e);
    void *tl = d.alloc(nl, e), *gq = d.alloc(nq, e), *gk = d.alloc(nq, e), *gv = d.alloc(nv, e), *ws = d.alloc(nws, e);
    if (e != cudaSuccess) return cuda_fail(e, "backward_host alloc");
    if ((e = cudaMemcpyAsync(g, dout, nv, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(tq, q, nq, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(tk, k, nq, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(tv, v, nv, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(to, out, nv, cudaMemcpyHostToDevice, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(tl, lse, nl, cudaMemcpyHostToDevice, d.st)) != cudaSuccess)
        return cuda_fail(e, "backward_host H2D");
    rc = cca_b200_backward(g, tq, tk, tv, to, (const float *)tl, gq, gk, gv, ws, nws, B, Cq, C, H, W, dtype, flags, d.st);
    if (rc) return rc;
    if ((e = cudaMemcpyAsync(dq, gq, nq, cudaMemcpyDeviceToHost, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(dk, gk, nq, cudaMemcpyDeviceToHost, d.st)) != cudaSuccess ||
        (e = cudaMemcpyAsync(dv, gv, nv, cudaMemcpyDeviceToHost, d.st)) != cudaSuccess ||
        (e = cudaStreamSynchronize(d.st)) != cudaSuccess)
        return cuda_fail(e, "backward_host D2H");
    return CCA_OK;
}

}  // extern "C"
