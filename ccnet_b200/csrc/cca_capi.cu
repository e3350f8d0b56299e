// C ABI of the operator (include/cca_b200.h): argument validation, kernel-family dispatch,
// host-buffer variants.  No torch types anywhere in this library.
#include <atomic>
#include <cstdio>
#include <initializer_list>
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
    if (dtype != CCA_F32 && dtype != CCA_BF16 && dtype != CCA_F16)
        return fail(CCA_ERR_INVALID, "dtype must be CCA_F32, CCA_BF16 or CCA_F16%s%s");
    if ((long long)B * C * H * W >= (1ll << 40)) return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");
    return CCA_OK;
}
size_t esize(int dtype) { return dtype == CCA_F32 ? 4 : 2; }    // (CCA_BF16, CCA_F16: 2)
constexpr const char *kDetHalfMsg =
    "CCA_FLAG_DETERMINISTIC with 16-bit I/O on lines longer than 112 pixels: call CCA_F32 on upcast tensors%s%s";
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
std::atomic<int> g_pdl{kUnset}, g_delta{kUnset}, g_lag{kUnset}, g_hints{kUnset};
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
int tc_delta_mode() { return knob(g_delta, "CCA_B200_DELTA", -1, -1, 1); }
int tc_lag() { return knob(g_lag, "CCA_B200_LAG", -1, -1, 1); }
int tc_l2_hints() { return knob(g_hints, "CCA_B200_L2HINT", 1, 0, 2); }
#ifdef CCA_DEBUG_HOOKS
void set_tc_pdl(int on) { g_pdl.store(on ? 1 : 0); }
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
// the *_supported queries: 0 on a device that is not sm_90; with no device at all they answer from the shape alone
bool other_device()
{
    int ndev = 0;
    return cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0 && device_major() != 9;
}
bool aligned16(std::initializer_list<const void *> ptrs)
{
    uintptr_t a = 0;
    for (const void *p : ptrs) a |= reinterpret_cast<uintptr_t>(p);
    return (a & 15) == 0;
}
constexpr const char *kAlignMsg = "tensor-core path needs 16-byte aligned tensors%s%s";
// Which kernel family runs a call that passed its dimension, pointer and workspace checks: 1 tensor cores, 0 generic
// kernels, < 0 an error status.  tc_covered: the tensor-core kernels cover the shape; det_16bit: CCA_FLAG_DETERMINISTIC with
// 16-bit I/O on tiled lines, which only the fp32 kernels have a planes mode for.  op and layout name the call and the
// generic kernels' layout in messages.  The generic kernels' own limits are the caller's.
int kernel_family(unsigned flags, bool tc_covered, bool det_16bit, const char *op, const char *layout)
{
    if ((flags & CCA_FLAG_FORCE_SIMT) && (flags & CCA_FLAG_FORCE_TC))
        return fail(CCA_ERR_INVALID, "FORCE_SIMT and FORCE_TC are exclusive%s%s");
    int rc = check_device();
    if (rc) return rc;
    const bool nhwc = (flags & CCA_FLAG_NHWC) != 0;
    const bool tc_ok = nhwc && tc_covered;
    if ((flags & CCA_FLAG_FORCE_TC) && !tc_ok)
        return fail(CCA_ERR_UNSUPPORTED, "tensor-core %s needs CCA_FLAG_NHWC and a covered shape%s", op);
    if (nhwc && (!tc_ok || (flags & CCA_FLAG_FORCE_SIMT)))
        return fail(CCA_ERR_UNSUPPORTED, "channels-last tensors are only handled by the tensor-core kernels; pass %s%s", layout);
    if (tc_ok && det_16bit) return fail(CCA_ERR_UNSUPPORTED, kDetHalfMsg);
    return tc_ok ? 1 : 0;
}
bool det_16bit_tiled(unsigned flags, Dims d, int dtype) { return (flags & CCA_FLAG_DETERMINISTIC) && dtype != CCA_F32 && tc_tiled(d); }
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
    if (check_dims(B, Cq, C, H, W, dtype) || other_device()) return 0;
    const Dims d{B, Cq, C, H, W};
    return (which == CCA_WS_BACKWARD ? tc_backward_supported(d, dtype) : tc_forward_supported(d, dtype)) ? 1 : 0;
}

// CCA_FLAG_DETERMINISTIC on a tiled fp32 channels-last problem the tensor-core kernels cover: the partial planes follow the
// tensor-core workspace (tc_forward / tc_backward)
size_t cca_b200_workspace_bytes_ex(int which, int B, int Cq, int C, int H, int W, int dtype, unsigned flags)
{
    const size_t base = cca_b200_workspace_bytes(which, B, Cq, C, H, W, dtype);
    if (!base || !(flags & CCA_FLAG_DETERMINISTIC) || !(flags & CCA_FLAG_NHWC) || dtype != CCA_F32) return base;
    const Dims d{B, Cq, C, H, W};
    if (!tc::shape_fits(d, dtype)) return base;
    const size_t need = (which == CCA_WS_FORWARD ? tc_forward_workspace(d) : tc_backward_workspace(d)) + tc_planes_bytes(which, d);
    return need > base ? need : base;
}

size_t cca_b200_workspace_bytes(int which, int B, int Cq, int C, int H, int W, int dtype)
{
    (void)dtype;
    if (B <= 0 || Cq <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
    const Dims d{B, Cq, C, H, W};
    // one size that covers whichever family runs
    const size_t simt = simt_workspace(which, d);
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

void cca_b200_item_planes(int B, int H, int W, int index, int lagged, int *out2)
{
    const tc::ItemSpace s = tc::make_space(B, H, W);
    const tc::Item it = tc::decode_item_order(s, index, lagged);
    out2[0] = tc::part_index(s, it); out2[1] = tc::qtile_part_index(s, it);
}

int cca_b200_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, size_t ws_bytes,
                     int B, int Cq, int C, int H, int W, int dtype, unsigned flags, void *stream)
{
    int rc = check_dims(B, Cq, C, H, W, dtype);
    if (rc) return rc;
    if (!q || !k || !v || !out || !lse || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes_ex(CCA_WS_FORWARD, B, Cq, C, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "forward workspace too small%s%s");
    const Dims d{B, Cq, C, H, W};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc_forward_supported(d, dtype), det_16bit_tiled(flags, d, dtype),
                                  "forward", "NCHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const char *why = "";
    cudaError_t e;
    if (fam == 1) {
        if (!aligned16({q, k, v, out})) return fail(CCA_ERR_INVALID, kAlignMsg);
        const bool det = (flags & CCA_FLAG_DETERMINISTIC) && tc_tiled(d);
        e = tc_forward(q, k, v, out, lse, ws, d, dtype, st, &why, det);
        if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "tc_forward");
        return CCA_OK;
    }
    if (!simt_supported(d, false)) return fail(CCA_ERR_UNSUPPORTED, "H or W too large for the generic kernels%s%s");
    e = simt_forward(q, k, v, out, lse, ws, d, dtype, st);
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
    if (ws_bytes < cca_b200_workspace_bytes_ex(CCA_WS_BACKWARD, B, Cq, C, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "backward workspace too small%s%s");
    const Dims d{B, Cq, C, H, W};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc_backward_supported(d, dtype), det_16bit_tiled(flags, d, dtype),
                                  "backward", "NCHW");
    if (fam < 0) return fam;
    const char *why = "";
    if (fam == 1) {
        if (!aligned16({dout, q, k, v, out, dq, dk, dv})) return fail(CCA_ERR_INVALID, kAlignMsg);
        const bool det = (flags & CCA_FLAG_DETERMINISTIC) && tc_tiled(d);
        cudaError_t e = tc_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d, dtype,
                                    reinterpret_cast<cudaStream_t>(stream), &why, det);
        if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "tc_backward");
        return CCA_OK;
    }
    if (!simt_supported(d, true)) return fail(CCA_ERR_UNSUPPORTED, "H or W too large for the generic kernels%s%s");
    cudaError_t e = simt_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d, dtype, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return cuda_fail(e, "simt_backward");
    return CCA_OK;
}

// ---------------------------------------------------------------------------------------
// attention map (functions.py:40 `concate`) and its gradient w.r.t. q, k
// ---------------------------------------------------------------------------------------
namespace {
int check_attention_dims(int B, int Cq, int H, int W, int dtype)
{
    int rc = check_dims(B, Cq, 1, H, W, dtype);
    if (rc) return rc;
    if ((long long)B * Cq * H * W >= (1ll << 40) || (long long)B * H * W * (H + W) >= (1ll << 40))
        return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");
    return CCA_OK;
}
bool attention_det_planes(Dims d, int dtype, unsigned flags)
{
    return (flags & CCA_FLAG_DETERMINISTIC) && (flags & CCA_FLAG_NHWC) && dtype == CCA_F32 && tc::shape_fits(Dims{d.B, d.Cq, tc::kNC, d.H, d.W}, dtype);
}
}  // namespace

int cca_b200_attention_tc_supported(int B, int Cq, int H, int W, int dtype)
{
    if (check_attention_dims(B, Cq, H, W, dtype) || other_device()) return 0;
    return tc_attention_supported(Dims{B, Cq, 0, H, W}, dtype) ? 1 : 0;
}

size_t cca_b200_attention_workspace_bytes(int backward, int B, int Cq, int H, int W, int dtype, unsigned flags)
{
    if (B <= 0 || Cq <= 0 || H <= 0 || W <= 0) return 0;
    const Dims d{B, Cq, 0, H, W};
    const size_t simt = simt_attention_workspace(backward, d);
    const size_t tcb = tc_attention_workspace(backward, d, attention_det_planes(d, dtype, flags));
    return simt > tcb ? simt : tcb;
}

int cca_b200_attention_forward(const void *q, const void *k, float *attn, void *ws, size_t ws_bytes, int B, int Cq, int H, int W,
                               int dtype, unsigned flags, void *stream)
{
    int rc = check_attention_dims(B, Cq, H, W, dtype);
    if (rc) return rc;
    if (!q || !k || !attn || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (reinterpret_cast<uintptr_t>(attn) & 3) return fail(CCA_ERR_INVALID, "attn must be 4-byte aligned%s%s");
    if (ws_bytes < cca_b200_attention_workspace_bytes(0, B, Cq, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "attention map workspace too small%s%s");
    const Dims d{B, Cq, 0, H, W};
    // (the forward writes every map element once: deterministic in every mode)
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc_attention_supported(d, dtype), false, "attention map", "NCHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const char *why = "";
    if (fam == 1) {
        if (!aligned16({q, k, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
        cudaError_t e = tc_attention_forward(q, k, attn, ws, d, dtype, st, &why);
        return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_attention_forward") : CCA_OK;
    }
    cudaError_t e = simt_attention_forward(q, k, attn, d, dtype, st);
    return e != cudaSuccess ? cuda_fail(e, "simt_attention_forward") : CCA_OK;
}

int cca_b200_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                size_t ws_bytes, int B, int Cq, int H, int W, int dtype, unsigned flags, void *stream)
{
    int rc = check_attention_dims(B, Cq, H, W, dtype);
    if (rc) return rc;
    if (!dattn || !attn || !q || !k || !dq || !dk || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if ((reinterpret_cast<uintptr_t>(attn) | reinterpret_cast<uintptr_t>(dattn)) & 3)
        return fail(CCA_ERR_INVALID, "attn and dattn must be 4-byte aligned%s%s");
    if (ws_bytes < cca_b200_attention_workspace_bytes(1, B, Cq, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "attention map backward workspace too small%s%s");
    const Dims d{B, Cq, 0, H, W};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc_attention_supported(d, dtype), det_16bit_tiled(flags, d, dtype),
                                  "attention map", "NCHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const char *why = "";
    if (fam == 1) {
        if (!aligned16({q, k, dq, dk, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
        cudaError_t e = tc_attention_backward(dattn, attn, q, k, dq, dk, ws, d, dtype, st, &why,
                                              (flags & CCA_FLAG_DETERMINISTIC) != 0);
        return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_attention_backward") : CCA_OK;
    }
    cudaError_t e = simt_attention_backward(dattn, attn, q, k, dq, dk, ws, d, dtype, st);
    return e != cudaSuccess ? cuda_fail(e, "simt_attention_backward") : CCA_OK;
}

// ---------------------------------------------------------------------------------------
// criss-cross attention over clips (the 3D op): tensor-core path (cca_tc_time.cu) or generic kernels (cca_simt_3d.cu)
// ---------------------------------------------------------------------------------------
namespace {
constexpr const char *kSimt3dKeysMsg = "H + W - 1 + time keys (T - 1, or the window) above 2048 for the generic 3D kernels%s%s";
int check_dims3d(int B, int Cq, int C, int T, int H, int W, int dtype)
{
    if (T <= 0) return fail(CCA_ERR_INVALID, "non-positive dimension%s%s");
    if ((long long)B * T >= (1ll << 31)) return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");
    return check_dims(B * T, Cq, C, H, W, dtype);
}
// a time window (window > 0) is a causal-mode parameter
int check_window(int window, unsigned flags)
{
    if (window < 0) return fail(CCA_ERR_INVALID, "negative time window%s%s");
    if (window > 0 && !(flags & CCA_FLAG_CAUSAL)) return fail(CCA_ERR_INVALID, "a time window needs CCA_FLAG_CAUSAL%s%s");
    return CCA_OK;
}
bool det3d_planes(Dims3 d, int dtype, unsigned flags)
{
    return (flags & CCA_FLAG_DETERMINISTIC) && (flags & CCA_FLAG_NHWC) && dtype == CCA_F32 && tc::shape_fits(d.frames(), dtype);
}
}  // namespace

int cca_b200_tc3d_supported(int which, int B, int Cq, int C, int T, int H, int W, int dtype)
{
    (void)which;                              // (forward and backward cover the same shapes)
    if (B <= 0 || T <= 0 || check_dims3d(B, Cq, C, T, H, W, dtype) || other_device()) return 0;
    return tc3d_supported(Dims3{B, Cq, C, T, H, W}, dtype) ? 1 : 0;
}

// one size that covers whichever family runs (as cca_b200_workspace_bytes_ex does in 2D)
size_t cca_b200_workspace_bytes3d(int which, int B, int Cq, int C, int T, int H, int W, int dtype, unsigned flags)
{
    if (B <= 0 || Cq <= 0 || C <= 0 || T <= 0 || H <= 0 || W <= 0 || (long long)B * T >= (1ll << 31)) return 0;
    const Dims3 d{B, Cq, C, T, H, W};
    const size_t tcb = (which == CCA_WS_FORWARD ? tc_forward3d_workspace(d) : tc_backward3d_workspace(d)) +
                       (det3d_planes(d, dtype, flags) ? tc_planes_bytes(which, d.frames()) : 0);
    const size_t simt = simt3d_workspace(which, d);
    return tcb > simt ? tcb : simt;
}

int cca_b200_forward3d(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, size_t ws_bytes,
                       int B, int Cq, int C, int T, int H, int W, int dtype, unsigned flags, void *stream)
{
    return cca_b200_forward3d_window(q, k, v, out, lse, ws, ws_bytes, B, Cq, C, T, H, W, 0, dtype, flags, stream);
}

int cca_b200_forward3d_window(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, size_t ws_bytes,
                              int B, int Cq, int C, int T, int H, int W, int window, int dtype, unsigned flags, void *stream)
{
    int rc = check_dims3d(B, Cq, C, T, H, W, dtype);
    if (rc || (rc = check_window(window, flags))) return rc;
    if (!q || !k || !v || !out || !lse || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes3d(CCA_WS_FORWARD, B, Cq, C, T, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "forward workspace too small%s%s");
    const Dims3 d{B, Cq, C, T, H, W, window};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc3d_supported(d, dtype), det_16bit_tiled(flags, d.frames(), dtype),
                                  "3D op", "NCDHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (fam == 0) {
        if (!simt3d_supported(d)) return fail(CCA_ERR_UNSUPPORTED, kSimt3dKeysMsg);
        cudaError_t e = (flags & CCA_FLAG_CAUSAL) ? simt_forward3d_causal(q, k, v, out, lse, d, dtype, st)
                                                  : simt_forward3d(q, k, v, out, lse, d, dtype, st);
        return e != cudaSuccess ? cuda_fail(e, "simt_forward3d") : CCA_OK;
    }
    if (!aligned16({q, k, v, out, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
    const char *why = "";
    const bool det = (flags & CCA_FLAG_DETERMINISTIC) && tc_tiled(d.frames());
    cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? tc_forward3d_causal : tc_forward3d)(q, k, v, out, lse, ws, d, dtype, st, &why, det);
    return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_forward3d") : CCA_OK;
}

int cca_b200_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, size_t ws_bytes, int B, int Cq, int C, int T, int H, int W,
                        int dtype, unsigned flags, void *stream)
{
    return cca_b200_backward3d_window(dout, q, k, v, out, lse, dq, dk, dv, ws, ws_bytes, B, Cq, C, T, H, W, 0, dtype, flags, stream);
}

int cca_b200_backward3d_window(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                               void *dq, void *dk, void *dv, void *ws, size_t ws_bytes, int B, int Cq, int C, int T, int H, int W,
                               int window, int dtype, unsigned flags, void *stream)
{
    int rc = check_dims3d(B, Cq, C, T, H, W, dtype);
    if (rc || (rc = check_window(window, flags))) return rc;
    if (!dout || !q || !k || !v || !out || !lse || !dq || !dk || !dv || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes3d(CCA_WS_BACKWARD, B, Cq, C, T, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "backward workspace too small%s%s");
    const Dims3 d{B, Cq, C, T, H, W, window};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc3d_supported(d, dtype), det_16bit_tiled(flags, d.frames(), dtype),
                                  "3D op", "NCDHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (fam == 0) {
        if (!simt3d_supported(d)) return fail(CCA_ERR_UNSUPPORTED, kSimt3dKeysMsg);
        if (reinterpret_cast<uintptr_t>(ws) & 3) return fail(CCA_ERR_INVALID, "workspace must be 4-byte aligned%s%s");
        cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? simt_backward3d_causal : simt_backward3d)(dout, q, k, v, out, lse, dq, dk, dv, ws, d,
                                                                                             dtype, st);
        return e != cudaSuccess ? cuda_fail(e, "simt_backward3d") : CCA_OK;
    }
    if (!aligned16({dout, q, k, v, out, dq, dk, dv, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
    const char *why = "";
    const bool det = (flags & CCA_FLAG_DETERMINISTIC) && tc_tiled(d.frames());
    cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? tc_backward3d_causal : tc_backward3d)(dout, q, k, v, out, lse, dq, dk, dv, ws, d, dtype,
                                                                                       st, &why, det);
    return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_backward3d") : CCA_OK;
}

// ---------------------------------------------------------------------------------------
// streaming step of the causal 3D op: tensor-core path (cca_tc_causal.cu) or generic kernel (cca_simt_causal.cu)
// ---------------------------------------------------------------------------------------
size_t cca_b200_workspace_bytes3d_step(int B, int Cq, int C, int S, int H, int W, int dtype, unsigned flags)
{
    // the forward workspace of a one-frame clip: the frame's lse planes and the time plane
    if (S < 0) return 0;
    return cca_b200_workspace_bytes3d(CCA_WS_FORWARD, B, Cq, C, 1, H, W, dtype, flags);
}

int cca_b200_forward3d_step(const void *q, const void *k, const void *v, const void *k_cache, const void *v_cache, void *out, float *lse,
                            void *ws, size_t ws_bytes, int B, int Cq, int C, int S, int H, int W, int dtype, unsigned flags,
                            void *stream)
{
    return cca_b200_forward3d_step_ring(q, k, v, k_cache, v_cache, out, lse, ws, ws_bytes, B, Cq, C, S, S, 0, H, W, dtype, flags, stream);
}

int cca_b200_forward3d_step_ring(const void *q, const void *k, const void *v, const void *k_ring, const void *v_ring, void *out,
                                 float *lse, void *ws, size_t ws_bytes, int B, int Cq, int C, int N, int S, int head, int H, int W,
                                 int dtype, unsigned flags, void *stream)
{
    if (S < 0) return fail(CCA_ERR_INVALID, "negative number of cached frames%s%s");
    if (S > N) return fail(CCA_ERR_INVALID, "more cached frames than ring slots%s%s");
    if (N > 0 && (head < 0 || head >= N)) return fail(CCA_ERR_INVALID, "ring head outside [0, N)%s%s");
    int rc = check_dims3d(B, Cq, C, S + 1, H, W, dtype);
    if (rc) return rc;
    if ((long long)N * H * W >= (1ll << 31) || (long long)B * N * H * W * (Cq > C ? Cq : C) >= (1ll << 40))
        return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");           // (the rings)
    if (!q || !k || !v || !out || !lse || !ws || (S > 0 && (!k_ring || !v_ring))) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (ws_bytes < cca_b200_workspace_bytes3d_step(B, Cq, C, S, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "step workspace too small%s%s");
    const Dims3 d3{B, Cq, C, S + 1, H, W};
    const Dims d{B, Cq, C, H, W};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc3d_supported(d3, dtype), det_16bit_tiled(flags, d, dtype),
                                  "3D step", "NCHW q, k, v and NCDHW caches");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (fam == 0) {
        if ((long)H + W + S - 1 > kMaxKeys3d || !simt3d_supported(d3))
            return fail(CCA_ERR_UNSUPPORTED, "H + W + S - 1 above 2048 for the generic step kernel%s%s");
        cudaError_t e = simt_forward3d_step(q, k, v, k_ring, v_ring, out, lse, d, N, S, head, dtype, st);
        return e != cudaSuccess ? cuda_fail(e, "simt_forward3d_step") : CCA_OK;
    }
    if (!aligned16({q, k, v, out, ws}) || (S > 0 && !aligned16({k_ring, v_ring}))) return fail(CCA_ERR_INVALID, kAlignMsg);
    const char *why = "";
    const bool det = (flags & CCA_FLAG_DETERMINISTIC) && tc_tiled(d);
    cudaError_t e = tc_forward3d_step(q, k, v, k_ring, v_ring, out, lse, ws, d, N, S, head, dtype, st, &why, det);
    return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_forward3d_step") : CCA_OK;
}

// ---------------------------------------------------------------------------------------
// attention map of the 3D op: tensor-core path (cca_tc_attn3d.cu) or generic kernels (cca_simt_attn3d.cu)
// ---------------------------------------------------------------------------------------
namespace {
int check_attention_dims3d(int B, int Cq, int T, int H, int W, int dtype)
{
    int rc = check_dims3d(B, Cq, 1, T, H, W, dtype);
    if (rc) return rc;
    const long long npix = (long long)B * T * H * W;
    if (npix * Cq >= (1ll << 40) || npix * ((long long)H + W + T) >= (1ll << 40)) return fail(CCA_ERR_UNSUPPORTED, "tensor too large%s%s");
    return CCA_OK;
}
}  // namespace

int cca_b200_attention_tc3d_supported(int B, int Cq, int T, int H, int W, int dtype)
{
    if (B <= 0 || T <= 0 || check_attention_dims3d(B, Cq, T, H, W, dtype) || other_device()) return 0;
    return tc3d_attention_supported(Dims3{B, Cq, 0, T, H, W}, dtype) ? 1 : 0;
}

size_t cca_b200_attention_workspace_bytes3d(int backward, int B, int Cq, int T, int H, int W, int dtype, unsigned flags)
{
    if (B <= 0 || Cq <= 0 || T <= 0 || H <= 0 || W <= 0 || (long long)B * T >= (1ll << 31)) return 0;
    const Dims3 d{B, Cq, 0, T, H, W};
    const size_t simt = simt_attention3d_workspace(backward, d);
    const size_t tcb = tc_attention3d_workspace(backward, d, attention_det_planes(d.frames(), dtype, flags));
    return simt > tcb ? simt : tcb;
}

int cca_b200_attention_forward3d(const void *q, const void *k, float *attn, void *ws, size_t ws_bytes, int B, int Cq, int T, int H,
                                 int W, int dtype, unsigned flags, void *stream)
{
    return cca_b200_attention_forward3d_window(q, k, attn, ws, ws_bytes, B, Cq, T, H, W, 0, dtype, flags, stream);
}

int cca_b200_attention_forward3d_window(const void *q, const void *k, float *attn, void *ws, size_t ws_bytes, int B, int Cq, int T,
                                        int H, int W, int window, int dtype, unsigned flags, void *stream)
{
    int rc = check_attention_dims3d(B, Cq, T, H, W, dtype);
    if (rc || (rc = check_window(window, flags))) return rc;
    if (!q || !k || !attn || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (reinterpret_cast<uintptr_t>(attn) & 3) return fail(CCA_ERR_INVALID, "attn must be 4-byte aligned%s%s");
    if (ws_bytes < cca_b200_attention_workspace_bytes3d(0, B, Cq, T, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "attention map workspace too small%s%s");
    const Dims3 d{B, Cq, 0, T, H, W, window};
    // (the forward writes every map element once: deterministic in every mode)
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc3d_attention_supported(d, dtype), false, "3D attention map",
                                  "NCDHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (fam == 1) {
        if (!aligned16({q, k, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
        const char *why = "";
        cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? tc_attention_forward3d_causal : tc_attention_forward3d)(q, k, attn, ws, d, dtype, st,
                                                                                                         &why);
        return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_attention_forward3d") : CCA_OK;
    }
    cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? simt_attention_forward3d_causal : simt_attention_forward3d)(q, k, attn, d, dtype, st);
    return e != cudaSuccess ? cuda_fail(e, "simt_attention_forward3d") : CCA_OK;
}

int cca_b200_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                  size_t ws_bytes, int B, int Cq, int T, int H, int W, int dtype, unsigned flags, void *stream)
{
    return cca_b200_attention_backward3d_window(dattn, attn, q, k, dq, dk, ws, ws_bytes, B, Cq, T, H, W, 0, dtype, flags, stream);
}

int cca_b200_attention_backward3d_window(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                         void *ws, size_t ws_bytes, int B, int Cq, int T, int H, int W, int window, int dtype,
                                         unsigned flags, void *stream)
{
    int rc = check_attention_dims3d(B, Cq, T, H, W, dtype);
    if (rc || (rc = check_window(window, flags))) return rc;
    if (!dattn || !attn || !q || !k || !dq || !dk || !ws) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if ((reinterpret_cast<uintptr_t>(attn) | reinterpret_cast<uintptr_t>(dattn)) & 3)
        return fail(CCA_ERR_INVALID, "attn and dattn must be 4-byte aligned%s%s");
    if (ws_bytes < cca_b200_attention_workspace_bytes3d(1, B, Cq, T, H, W, dtype, flags))
        return fail(CCA_ERR_WORKSPACE, "attention map backward workspace too small%s%s");
    const Dims3 d{B, Cq, 0, T, H, W, window};
    const int fam = kernel_family(flags, (flags & CCA_FLAG_NHWC) && tc3d_attention_supported(d, dtype),
                                  det_16bit_tiled(flags, d.frames(), dtype), "3D attention map", "NCDHW");
    if (fam < 0) return fam;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (fam == 1) {
        if (!aligned16({q, k, dq, dk, ws})) return fail(CCA_ERR_INVALID, kAlignMsg);
        const char *why = "";
        cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? tc_attention_backward3d_causal : tc_attention_backward3d)(
            dattn, attn, q, k, dq, dk, ws, d, dtype, st, &why, (flags & CCA_FLAG_DETERMINISTIC) != 0);
        return e != cudaSuccess ? cuda_fail(e, why && *why ? why : "tc_attention_backward3d") : CCA_OK;
    }
    if (reinterpret_cast<uintptr_t>(ws) & 3) return fail(CCA_ERR_INVALID, "workspace must be 4-byte aligned%s%s");
    cudaError_t e = ((flags & CCA_FLAG_CAUSAL) ? simt_attention_backward3d_causal : simt_attention_backward3d)(dattn, attn, q, k, dq, dk,
                                                                                                              ws, d, dtype, st);
    return e != cudaSuccess ? cuda_fail(e, "simt_attention_backward3d") : CCA_OK;
}

// ---------------------------------------------------------------------------------------
// 1x1 Q/K/V projections (functions.py:29,32,35) as tensor-core GEMMs on the channels-last view
// ---------------------------------------------------------------------------------------
namespace {
// the projection GEMMs' checks before their alignment, in this order: null pointers, dimensions, the workspace (not for the
// weight gradient: its size follows the device's SM count), the device, the shapes the GEMM covers
int check_gemm(bool null_ptr, long long pixels, int C, int Cq, bool wgrad, size_t ws_bytes)
{
    if (null_ptr) return fail(CCA_ERR_INVALID, "null pointer%s%s");
    if (pixels <= 0 || pixels >= (1ll << 31) || C <= 0 || Cq <= 0) return fail(CCA_ERR_INVALID, "bad dimension%s%s");
    if (!wgrad && ws_bytes < qkv_gemm_workspace(C, Cq)) return fail(CCA_ERR_WORKSPACE, "projection workspace too small%s%s");
    int rc = check_device();
    if (rc) return rc;
    if (wgrad && !qkv_wgrad_supported(C, Cq))
        return fail(CCA_ERR_UNSUPPORTED, "weight-gradient GEMM needs C %% 256 == 0 and Cq %% 64 == 0%s%s");
    if (!wgrad && !qkv_gemm_supported(C, Cq)) return fail(CCA_ERR_UNSUPPORTED, "projection GEMM needs C %% 64 == 0 and Cq %% 64 == 0%s%s");
    return CCA_OK;
}
}  // namespace

int cca_b200_qkv_supported(int C, int Cq)
{
    if (C <= 0 || Cq <= 0 || other_device()) return 0;
    return qkv_gemm_supported(C, Cq) ? 1 : 0;
}
size_t cca_b200_qkv_workspace_bytes(int C, int Cq) { return C > 0 && Cq > 0 ? qkv_gemm_workspace(C, Cq) : 0; }

int cca_b200_qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk, const float *wv,
                         const float *bv, float *q, float *k, float *v, void *ws, size_t ws_bytes, long long pixels, int C, int Cq,
                         void *stream)
{
    int rc = check_gemm(!x || !wq || !bq || !wk || !bk || !wv || !bv || !q || !k || !v || !ws, pixels, C, Cq, false, ws_bytes);
    if (rc) return rc;
    if (!aligned16({x, q, k, v, ws})) return fail(CCA_ERR_INVALID, "projection GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project(x, wq, bq, wk, bk, wv, bv, q, k, v, ws, (long)pixels, C, Cq, reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project");
    return CCA_OK;
}

int cca_b200_qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk, const float *wv,
                               const float *scale, float *dx, void *ws, size_t ws_bytes, long long pixels, int C, int Cq,
                               int accumulate, void *stream)
{
    int rc = check_gemm(!dq || !dk || !dv || !wq || !wk || !wv || !dx || !ws, pixels, C, Cq, false, ws_bytes);
    if (rc) return rc;
    if (!aligned16({dx, dq, dk, dv, ws})) return fail(CCA_ERR_INVALID, "projection GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project_dgrad(dq, dk, dv, wq, wk, wv, scale, dx, ws, (long)pixels, C, Cq, accumulate,
                                      reinterpret_cast<cudaStream_t>(stream), &why);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project_dgrad");
    return CCA_OK;
}

int cca_b200_qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                               float *dwk, float *dwv, float *db, long long pixels, int C, int Cq, void *stream)
{
    return cca_b200_qkv_project_wgrad_ex(x, dq, dk, dv, scale, dwq, dwk, dwv, db, pixels, C, Cq, nullptr, 0, 0, stream);
}
size_t cca_b200_qkv_wgrad_workspace_bytes(int C, int Cq)
{
    return C > 0 && Cq > 0 && qkv_wgrad_supported(C, Cq) ? qkv_wgrad_workspace(C, Cq) : 0;
}
int cca_b200_qkv_project_wgrad_ex(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                                  float *dwk, float *dwv, float *db, long long pixels, int C, int Cq, void *ws, size_t ws_bytes,
                                  unsigned flags, void *stream)
{
    const bool det = (flags & CCA_FLAG_DETERMINISTIC) != 0;
    int rc = check_gemm(!x || !dq || !dk || !dv || !dwq || !dwk || !dwv || (det && !ws), pixels, C, Cq, true, 0);
    if (rc) return rc;
    if (det && ws_bytes < qkv_wgrad_workspace(C, Cq)) return fail(CCA_ERR_WORKSPACE, "weight-gradient workspace too small%s%s");
    if (!(det ? aligned16({x, dq, dk, dv, ws}) : aligned16({x, dq, dk, dv, dwq, dwk, dwv})))
        return fail(CCA_ERR_INVALID, "weight-gradient GEMM needs 16-byte aligned tensors%s%s");
    const char *why = "";
    cudaError_t e = qkv_project_wgrad(x, dq, dk, dv, scale, dwq, dwk, dwv, db, (long)pixels, C, Cq, reinterpret_cast<cudaStream_t>(stream),
                                      &why, det ? ws : nullptr);
    if (e != cudaSuccess) return cuda_fail(e, why && *why ? why : "qkv_project_wgrad");
    return CCA_OK;
}
int cca_b200_qkv_wgrad_supported(int C, int Cq)
{
    if (C <= 0 || Cq <= 0 || other_device()) return 0;
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
    const size_t nws = cca_b200_workspace_bytes_ex(CCA_WS_FORWARD, B, Cq, C, H, W, dtype, flags);
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
    const size_t nws = cca_b200_workspace_bytes_ex(CCA_WS_BACKWARD, B, Cq, C, H, W, dtype, flags);
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
