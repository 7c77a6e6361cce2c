// extern "C" boundary of fastecc_b200 (include/fastecc_b200.h): context, planning, launches, host<->device staging.
#include "../../include/fastecc_b200.h"
#include "plan.h"
#include "ntt_pass.h"
#include "small_dft.h"
#include "byte_recode.h"
#include "elementwise.h"
#include "mixed_radix.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <cstdlib>
#include <mutex>
#include <vector>
#include <atomic>
#include <map>

using namespace fecc;

namespace {

struct DevBuf {
    void* p = nullptr; size_t bytes = 0;
    cudaError_t reserve(size_t need) {
        if (need <= bytes) return cudaSuccess;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        cudaError_t e = cudaMalloc(&p, need);
        if (e == cudaSuccess) bytes = need;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
};

// Stage tables of one plan: built once, on the stream of the first call that needs them.  `ready` is recorded behind the
// build; a call on any other stream waits for it (a no-op once the build has finished).
struct TableSet {
    struct Slot { DevBuf buf; cudaEvent_t ready = nullptr; cudaStream_t built_on = nullptr; };
    std::vector<Slot> slots;             // one block per pass (plan.h table_bytes)
};
// A buffer shared by calls that may come in on different streams (the Y buffer of the two-pass NTT, the repack buffer):
// `done` is recorded behind its last use and the next user on another stream waits for it, so that two transforms in
// flight on two streams are serialised on the buffer instead of racing on it.
struct SharedBuf {
    DevBuf buf;
    cudaEvent_t done = nullptr;
    cudaStream_t last = nullptr;
    bool used = false;
    cudaError_t acquire(size_t need, cudaStream_t st) {
        if (need > buf.bytes && used) { cudaError_t e = cudaEventSynchronize(done); if (e != cudaSuccess) return e; }     // about to be reallocated
        cudaError_t e = buf.reserve(need);
        if (e != cudaSuccess) return e;
        if (!done) { e = cudaEventCreateWithFlags(&done, cudaEventDisableTiming); if (e != cudaSuccess) return e; }
        if (used && last != st) e = cudaStreamWaitEvent(st, done, 0);
        return e;
    }
    cudaError_t release_to(cudaStream_t st) { used = true; last = st; return cudaEventRecord(done, st); }
    void destroy() { buf.release(); if (done) cudaEventDestroy(done); done = nullptr; used = false; }
};

struct Context {
    int device = -1;
    int num_sms = 0;
    uint4* d_tw = nullptr;
    SharedBuf scratch;   // Y buffer of the two-pass NTT and of the asymmetric encode
    SharedBuf packed;    // repacked copy for unaligned device layouts
    SharedBuf mixed;     // destination of the order-3 / order-9 step of the N = 3 * 2^k, 9 * 2^k transforms
    DevBuf staging;      // device copy for the host (T**) entry points (serialised by g_mu)
    std::map<uint32_t, TableSet> tables;              // per (mode, log2 N, ...)
    bool pin_caller = false;                          // fastecc_b200_pin_host_buffers()
    std::vector<std::pair<char*, size_t>> registered; // caller buffers we page-locked in place (cudaHostRegister)
    cudaStream_t stream = nullptr;       // compute
    cudaStream_t h2d = nullptr, d2h = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_done;
};

Context* g_ctx = nullptr;
std::mutex g_mu;          // guards g_ctx, the table cache and the shared buffers' bookkeeping (short critical sections)
std::mutex g_host_mu;     // held by the host (T**) entry points for their whole duration: they share the staging buffer, three streams and the chunk events
std::atomic<unsigned long long> g_launches{0};
thread_local char g_err[512] = "no error";

int fail(int code, const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
#define CUDA_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
    return fail(e_ == cudaErrorMemoryAllocation ? FASTECC_B200_ENOMEM : FASTECC_B200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); } while (0)

// N = r * 2^k with r = 3 or 9: the orders served by mixed_radix.cu on top of the power-of-two kernels (transforms only)
uint32_t odd_factor(size_t N)
{
    if (!N) return 0;
    while (!(N & 1)) N >>= 1;
    return (uint32_t)(N <= 9 ? N : 0);
}
int check_shape(size_t N, size_t size, size_t max_log, const char* who, bool allow_mixed = false)
{
    if (size == 0) return fail(FASTECC_B200_EINVAL, "%s: SIZE must be >= 1 word", who);
    const uint32_t r = odd_factor(N);
    if (allow_mixed && (r == 3 || r == 9) && is_pow2(N / r) && N / r <= ((size_t)1 << max_log)) {
        if (size > 0xFFFFFFF0u) return fail(FASTECC_B200_EINVAL, "%s: SIZE too large", who);
        return 0;
    }
    if (!is_pow2(N) || N > ((size_t)1 << max_log))
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu must be a power of two in [1, 2^%zu]%s (P-1 = 2^20*4095)", who, N, max_log, allow_mixed ? ", or 3 or 9 times one" : "");
    if (size > 0xFFFFFFF0u) return fail(FASTECC_B200_EINVAL, "%s: SIZE too large", who);
    return 0;
}

// Host (T**) entry points on a large contiguous PAGEABLE array: cudaMemcpy2DAsync would be staged through the driver's bounce
// buffers, synchronously, and nothing would overlap.  When the caller has opted in (fastecc_b200_pin_host_buffers: it keeps
// the array alive and calls again on it, like the reference's drivers, RS.cpp:31 / main.cpp:244), the array is page-locked in
// place once -- about 0.2 s per GiB -- and every later call runs the pinned, pipelined path.  Failure is not an error.
void pin_caller_array(Context* c, void* base, size_t bytes)
{
    if (!c->pin_caller || bytes < ((size_t)32 << 20)) return;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, base) != cudaSuccess) { cudaGetLastError(); return; }
    if (at.type != cudaMemoryTypeUnregistered) return;                      // already pinned (by us earlier, or by the caller)
    char* b = (char*)base;
    for (size_t i = 0; i < c->registered.size();) {                         // a stale, overlapping registration (the caller re-allocated): drop it
        auto& r = c->registered[i];
        if (b < r.first + r.second && r.first < b + bytes) { cudaHostUnregister(r.first); cudaGetLastError(); r = c->registered.back(); c->registered.pop_back(); }
        else ++i;
    }
    if (cudaHostRegister(base, bytes, cudaHostRegisterDefault) == cudaSuccess) c->registered.emplace_back(b, bytes);
    else cudaGetLastError();
}

// Stage tables of `plan` under cache key `key`: built on first use (into a local set that enters the cache only when every
// block is allocated and its build launched), then attached to the passes.  which >= 0: only that pass of a 3-pass plan.
int attach_tables(Context* c, uint32_t key, std::vector<PassParams>& plan, cudaStream_t st, int which = -1, size_t slots = 0)
{
    std::lock_guard<std::mutex> lk(g_mu);
    TableSet& ts = c->tables[key];
    const size_t n = slots ? slots : plan.size();
    if (ts.slots.size() != n) ts.slots.resize(n);
    for (size_t i = 0; i < plan.size(); ++i) {
        TableSet::Slot& sl = ts.slots[which >= 0 ? (size_t)which : i];
        if (!sl.buf.p) {
            DevBuf nb;
            cudaEvent_t ev = nullptr;
            cudaError_t e = nb.reserve(table_bytes(plan[i]));
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
            if (e == cudaSuccess) e = launch_build_tables(plan[i], (uint4*)nb.p, st);
            if (e == cudaSuccess) e = cudaEventRecord(ev, st);
            if (e != cudaSuccess) { nb.release(); if (ev) cudaEventDestroy(ev); CUDA_TRY(e); }
            g_launches++;
            sl.buf = nb; sl.ready = ev; sl.built_on = st;
        } else if (sl.built_on != st) {
            CUDA_TRY(cudaStreamWaitEvent(st, sl.ready, 0));
        }
        plan[i].tables = (const uint4*)sl.buf.p;
        plan[i].table_set_stride = table_sets(plan[i]) > 1 ? (plan[i].nxf << plan[i].log_r) : 0u;
    }
    return 0;
}

struct PassTimer {                       // optional per-pass timing (fastecc_b200_rs_encode_dev_timed)
    std::vector<cudaEvent_t> ev;
    std::vector<const char*> names;
};

int launch_plan(Context* c, std::vector<PassParams>& plan, cudaStream_t st, PassTimer* timer = nullptr)
{
    for (size_t i = 0; i < plan.size(); ++i) {
        const char* name = nullptr;
        if (timer && i == 0) { cudaEvent_t e; CUDA_TRY(cudaEventCreate(&e)); CUDA_TRY(cudaEventRecord(e, st)); timer->ev.push_back(e); }
        CUDA_TRY(launch_pass(plan[i], c->num_sms, st, &name)); g_launches++;
        if (timer) { cudaEvent_t e; CUDA_TRY(cudaEventCreate(&e)); CUDA_TRY(cudaEventRecord(e, st)); timer->ev.push_back(e); timer->names.push_back(name); }
    }
    return 0;
}

// Run the planned passes on an aligned, padded device buffer.
int run_aligned(Context* c, uint32_t* x, size_t N, size_t size, size_t pitch, int mode /*0 fwd,1 inv,2 encode*/, cudaStream_t st, PassTimer* timer = nullptr)
{
    const uint32_t pitch4 = (uint32_t)(pitch / 4), s4 = (uint32_t)((size + 3) / 4);
    if (!is_pow2(N)) {                                    // N = r * M, r = 3 or 9 (mixed_radix.cu); transforms only
        const uint32_t r = odd_factor(N);
        const size_t M = N / r;
        if (mode == 2 || (r != 3 && r != 9) || (unsigned long long)r * pitch > 0xFFFFFFF0ull) return fail(FASTECC_B200_EINVAL, "unsupported order N=%zu", N);
        if (M > 1)                                        // step 1: r transforms of order M, each on every r-th row (row pitch r times larger), in place
            for (uint32_t n1 = 0; n1 < r; ++n1)
                if (int rc = run_aligned(c, x + (size_t)n1 * pitch, M, size, (size_t)r * pitch, mode, st)) return rc;
        { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->mixed.acquire(N * pitch * sizeof(uint32_t), st)); }
        uint32_t* y = (uint32_t*)c->mixed.buf.p;          // step 2: twiddles + order-r transform, into natural order (out of place), then back
        CUDA_TRY(launch_radix_pass(x, y, pitch4, s4, r, (uint32_t)M, mode == 1, c->d_tw, c->num_sms, st)); g_launches++;
        CUDA_TRY(cudaMemcpy2DAsync(x, pitch * 4, y, pitch * 4, (size_t)s4 * 16 < pitch * 4 ? (size_t)s4 * 16 : pitch * 4, N, cudaMemcpyDeviceToDevice, st));
        { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->mixed.release_to(st)); }
        return 0;
    }
    if (N < ((size_t)1 << kMinLogR)) {
        const uint32_t z = (uint32_t)(gf::M / N) * (mode == 1 ? (uint32_t)-1 : 1u) & (gf::M - 1);
        const uint32_t q = mode == 2 ? (uint32_t)(gf::M / (2 * N)) : 0;
        const gf::Tw in = gf::make_tw(gf::inv((uint32_t)N));
        CUDA_TRY(launch_small_dft(x, pitch4, s4, (uint32_t)N, z, mode == 2, q, make_uint4(in.w, in.whi, in.wlo, 0), c->d_tw, st));
        g_launches++;
        return 0;
    }
    Buffers b{x, nullptr, c->d_tw, (uint32_t)pitch, (uint32_t)size};
    const bool need_y = mode != 2 && !single_pass(ilog2(N));               // the two-pass NTT ping-pongs through Y
    if (need_y) {
        std::lock_guard<std::mutex> lk(g_mu);
        CUDA_TRY(c->scratch.acquire(N * pitch * sizeof(uint32_t), st));
        b.y = (uint32_t*)c->scratch.buf.p;
    }
    std::vector<PassParams> plan = (mode == 2) ? plan_encode(b, N) : plan_ntt(b, N, mode == 1);
    if (int rc = attach_tables(c, (uint32_t)mode << 8 | ilog2(N), plan, st)) return rc;
    if (int rc = launch_plan(c, plan, st, timer)) return rc;
    if (need_y) { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->scratch.release_to(st)); }
    return 0;
}

// N data blocks -> M = N / 2^k parity blocks in rows [0, M) of x (rows [M, N) are left undefined).
int run_aligned_asym(Context* c, uint32_t* x, size_t N, size_t M, size_t size, size_t pitch, cudaStream_t st)
{
    if (M == N) return run_aligned(c, x, N, size, pitch, 2, st);
    size_t M0 = N;                                        // what the passes produce; M0 >= M
    const bool native = N > ((size_t)1 << kMaxLogR);
    if (!native) { if (int rc = run_aligned(c, x, N, size, pitch, 2, st)) return rc; }
    { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->scratch.acquire(N * pitch * sizeof(uint32_t), st)); }
    uint32_t* y = (uint32_t*)c->scratch.buf.p;
    if (native) {
        M0 = M;
        while (!asym_native(N, M0)) M0 *= 2;              // M0 = max(M, N1)
        Buffers b{x, y, c->d_tw, (uint32_t)pitch, (uint32_t)size};
        std::vector<PassParams> plan = plan_encode_asym(b, N, M0);
        if (int rc = attach_tables(c, 0x40000000u | ilog2(N / M0) << 8 | ilog2(N), plan, st)) return rc;
        if (int rc = launch_plan(c, plan, st)) return rc;
    }
    if (M0 != M) {                                        // keep every (M0/M)-th parity block: gather through the scratch buffer
        CUDA_TRY(cudaMemcpy2DAsync(y, pitch * 4, x, (M0 / M) * pitch * 4, size * 4, M, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpy2DAsync(x, pitch * 4, y, pitch * 4, size * 4, M, cudaMemcpyDeviceToDevice, st));
    }
    { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->scratch.release_to(st)); }
    return 0;
}

int run_dev(uint32_t* d, size_t N, size_t size, size_t pitch, int mode, void* stream, const char* who, PassTimer* timer = nullptr)
{
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (int rc = check_shape(N, size, mode == 2 ? FASTECC_B200_MAX_LOG_N_ENCODE : FASTECC_B200_MAX_LOG_N, who, mode != 2)) return rc;
    if (pitch < size || pitch > 0xFFFFFFF0u) return fail(FASTECC_B200_EINVAL, "%s: pitch_words (%zu) must be in [SIZE_words (%zu), 2^32 - 16]", who, pitch, size);
    if ((unsigned long long)N * ((pitch + 3) / 4) >= (1ull << 32))
        return fail(FASTECC_B200_EINVAL, "%s: buffer of %zu x %zu words is 64 GiB or more (32-bit chunk indexing)", who, N, pitch);
    cudaStream_t st = (cudaStream_t)stream;
    const bool aligned = (pitch % 4 == 0) && (((uintptr_t)d) % 16 == 0);
    if (aligned) return run_aligned(c, d, N, size, pitch, mode, st, timer);
    // unaligned layout: repack into a padded copy, transform, copy the SIZE data words back
    const size_t ppitch = (size + 3) / 4 * 4;
    { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->packed.acquire(N * ppitch * sizeof(uint32_t), st)); }
    uint32_t* pk = (uint32_t*)c->packed.buf.p;
    CUDA_TRY(launch_pack(d, pitch, pk, ppitch, N, (uint32_t)size, st)); g_launches++;
    if (int rc = run_aligned(c, pk, N, size, ppitch, mode, st, timer)) return rc;
    CUDA_TRY(launch_unpack(pk, ppitch, d, pitch, N, (uint32_t)size, st)); g_launches++;
    { std::lock_guard<std::mutex> lk(g_mu); CUDA_TRY(c->packed.release_to(st)); }
    return 0;
}

int run_host(uint32_t** data, size_t N, size_t size, int mode, const char* who)
{
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!data) return fail(FASTECC_B200_EINVAL, "%s: null block table", who);
    if (int rc = check_shape(N, size, mode == 2 ? FASTECC_B200_MAX_LOG_N_ENCODE : FASTECC_B200_MAX_LOG_N, who, mode != 2)) return rc;
    for (size_t i = 0; i < N; i++) if (!data[i]) return fail(FASTECC_B200_EINVAL, "%s: data[%zu] is null", who, i);
    std::lock_guard<std::mutex> host_lock(g_host_mu);
    const size_t pitch = (size + 3) / 4 * 4;
    CUDA_TRY(c->staging.reserve(N * pitch * sizeof(uint32_t)));
    uint32_t* dv = (uint32_t*)c->staging.p;
    cudaStream_t st = c->stream;
    bool contiguous = true;
    for (size_t i = 1; i < N; i++) if (data[i] != data[0] + i * size) { contiguous = false; break; }
    if (pitch != size) CUDA_TRY(cudaMemsetAsync(dv, 0, N * pitch * sizeof(uint32_t), st));
    // Large contiguous arrays: the word columns are independent codewords, so the array is cut into column chunks and
    // H2D(chunk c+1), the transform of chunk c and D2H(chunk c-1) run concurrently on three streams (PCIe is full duplex).
    static const size_t chunk_env = getenv("FASTECC_B200_CHUNK_WORDS") ? (size_t)atol(getenv("FASTECC_B200_CHUNK_WORDS")) : 0;
    size_t cw = chunk_env ? (chunk_env + 15) / 16 * 16 : 128;
    const bool pipelined = contiguous && pitch == size && size >= 2 * cw && N * size * 4 >= ((size_t)32 << 20);
    if (pipelined) {
        pin_caller_array(c, data[0], N * size * sizeof(uint32_t));
        const size_t nchunks = (size + cw - 1) / cw;
        while (c->ev_in.size() < nchunks) { cudaEvent_t e; CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->ev_in.push_back(e); }
        while (c->ev_done.size() < nchunks) { cudaEvent_t e; CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->ev_done.push_back(e); }
        for (size_t k = 0; k < nchunks; ++k) {
            const size_t c0 = k * cw, w = (c0 + cw <= size) ? cw : size - c0;
            CUDA_TRY(cudaMemcpy2DAsync(dv + c0, pitch * 4, data[0] + c0, size * 4, w * 4, N, cudaMemcpyHostToDevice, c->h2d));
            CUDA_TRY(cudaEventRecord(c->ev_in[k], c->h2d));
            CUDA_TRY(cudaStreamWaitEvent(st, c->ev_in[k], 0));
            if (int rc = run_aligned(c, dv + c0, N, w, pitch, mode, st)) return rc;
            CUDA_TRY(cudaEventRecord(c->ev_done[k], st));
            CUDA_TRY(cudaStreamWaitEvent(c->d2h, c->ev_done[k], 0));
            CUDA_TRY(cudaMemcpy2DAsync(data[0] + c0, size * 4, dv + c0, pitch * 4, w * 4, N, cudaMemcpyDeviceToHost, c->d2h));
        }
        CUDA_TRY(cudaStreamSynchronize(c->d2h));
        CUDA_TRY(cudaStreamSynchronize(st));
        return 0;
    }
    if (contiguous) {
        CUDA_TRY(cudaMemcpy2DAsync(dv, pitch * 4, data[0], size * 4, size * 4, N, cudaMemcpyHostToDevice, st));
    } else {
        for (size_t i = 0; i < N; i++) CUDA_TRY(cudaMemcpyAsync(dv + i * pitch, data[i], size * 4, cudaMemcpyHostToDevice, st));
    }
    if (int rc = run_aligned(c, dv, N, size, pitch, mode, st)) return rc;
    if (contiguous) {
        CUDA_TRY(cudaMemcpy2DAsync(data[0], size * 4, dv, pitch * 4, size * 4, N, cudaMemcpyDeviceToHost, st));
    } else {
        for (size_t i = 0; i < N; i++) CUDA_TRY(cudaMemcpyAsync(data[i], dv + i * pitch, size * 4, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

} // namespace

// internal accessors for the other translation units of the library (decode.cu)
namespace fecc {
const uint4* context_power_table() { return g_ctx ? g_ctx->d_tw : nullptr; }
int context_num_sms() { return g_ctx ? g_ctx->num_sms : 0; }
int api_fail(int code, const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
}

extern "C" {

int fastecc_b200_init(int device)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_ctx && g_ctx->device == device) return 0;
    if (g_ctx) return fail(FASTECC_B200_EINVAL, "fastecc_b200_init: already initialised on device %d (one process per GPU)", g_ctx->device);
    int count = 0;
    CUDA_TRY(cudaGetDeviceCount(&count));
    if (device < 0 || device >= count) return fail(FASTECC_B200_EINVAL, "fastecc_b200_init: device %d out of range (%d visible)", device, count);
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(FASTECC_B200_ECUDA, "fastecc_b200_init: device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
    Context* c = new Context;
    c->device = device; c->num_sms = prop.multiProcessorCount;
    std::vector<gf::Tw> tw(gf::M);
    fill_power_table(tw.data());
    CUDA_TRY(cudaMalloc((void**)&c->d_tw, sizeof(gf::Tw) * gf::M));
    CUDA_TRY(cudaMemcpy(c->d_tw, tw.data(), sizeof(gf::Tw) * gf::M, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->h2d, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->d2h, cudaStreamNonBlocking));
    g_ctx = c;
    return 0;
}

void fastecc_b200_shutdown(void)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_ctx) return;
    cudaSetDevice(g_ctx->device);
    cudaDeviceSynchronize();
    g_ctx->scratch.destroy(); g_ctx->packed.destroy(); g_ctx->mixed.destroy(); g_ctx->staging.release();
    for (auto& r : g_ctx->registered) cudaHostUnregister(r.first);
    for (auto& kv : g_ctx->tables) for (auto& sl : kv.second.slots) { sl.buf.release(); if (sl.ready) cudaEventDestroy(sl.ready); }
    if (g_ctx->d_tw) cudaFree(g_ctx->d_tw);
    if (g_ctx->stream) cudaStreamDestroy(g_ctx->stream);
    if (g_ctx->h2d) cudaStreamDestroy(g_ctx->h2d);
    if (g_ctx->d2h) cudaStreamDestroy(g_ctx->d2h);
    for (auto e : g_ctx->ev_in) cudaEventDestroy(e);
    for (auto e : g_ctx->ev_done) cudaEventDestroy(e);
    delete g_ctx; g_ctx = nullptr;
}

const char* fastecc_b200_last_error(void) { return g_err; }
int fastecc_b200_device(void)  { return g_ctx ? g_ctx->device : -1; }
int fastecc_b200_num_sms(void) { return g_ctx ? g_ctx->num_sms : 0; }
unsigned long long fastecc_b200_kernel_launches(void) { return g_launches.load(); }

int fastecc_b200_ntt_u32_dev(uint32_t* d, size_t N, size_t size, size_t pitch, int inverse, void* stream)
{ return run_dev(d, N, size, pitch, inverse ? 1 : 0, stream, "fastecc_b200_ntt_u32_dev"); }

int fastecc_b200_rs_encode_dev(uint32_t* d, size_t N, size_t size, size_t pitch, void* stream)
{ return run_dev(d, N, size, pitch, 2, stream, "fastecc_b200_rs_encode_dev"); }

int fastecc_b200_rs_encode_dev_timed(uint32_t* d, size_t N, size_t size, size_t pitch, void* stream, float* pass_ms, const char** pass_kernel, int* n_passes)
{
    const char* who = "fastecc_b200_rs_encode_dev_timed";
    if (!pass_ms || !n_passes || *n_passes < 1) return fail(FASTECC_B200_EINVAL, "%s: pass_ms / n_passes missing", who);
    PassTimer t;
    int rc = run_dev(d, N, size, pitch, 2, stream, who, &t);
    if (rc == 0 && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) rc = fail(FASTECC_B200_ECUDA, "%s: %s", who, cudaGetErrorString(cudaGetLastError()));
    int n = 0;
    for (size_t i = 0; rc == 0 && i + 1 < t.ev.size() && n < *n_passes; ++i, ++n) {
        if (cudaEventElapsedTime(&pass_ms[n], t.ev[i], t.ev[i + 1]) != cudaSuccess) rc = fail(FASTECC_B200_ECUDA, "%s: cudaEventElapsedTime failed", who);
        if (pass_kernel) pass_kernel[n] = t.names[i];
    }
    for (cudaEvent_t e : t.ev) cudaEventDestroy(e);
    *n_passes = n;
    return rc;
}

int fastecc_b200_shard_geometry(size_t N, int n_ranks, size_t* N1, size_t* N2, int* fused_exchange_ok)
{
    if (!is_pow2(N) || N < 2) return fail(FASTECC_B200_EINVAL, "fastecc_b200_shard_geometry: N must be a power of two");
    const uint32_t LN = ilog2(N), L1 = LN <= (uint32_t)kMaxLogR ? LN : split_l1(LN);
    if (N1) *N1 = (size_t)1 << L1;
    if (N2) *N2 = (size_t)1 << (LN - L1);
    if (fused_exchange_ok) *fused_exchange_ok = n_ranks >= 2 ? (shard_p2p_supported(N, (uint32_t)n_ranks) ? 1 : 0) | (ntt_shard_p2p_supported(N, (uint32_t)n_ranks) ? 2 : 0) : 0;
    return n_ranks < 2 || shard_supported(N, (uint32_t)n_ranks) || ntt_shard_p2p_supported(N, (uint32_t)n_ranks) ? 0 : fail(FASTECC_B200_EINVAL, "fastecc_b200_shard_geometry: N=%zu cannot be sharded over %d ranks", N, n_ranks);
}

int fastecc_b200_copy2d_async(void* dst, size_t dst_pitch_bytes, const void* src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, int to_device, void* stream)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_copy2d_async: call fastecc_b200_init() first");
    CUDA_TRY(cudaMemcpy2DAsync(dst, dst_pitch_bytes, src, src_pitch_bytes, width_bytes, rows, to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return 0;
}

int fastecc_b200_gf_mul_dev(const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n, void* stream)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_gf_mul_dev: call fastecc_b200_init() first");
    if (n && (!a || !b || !out)) return fail(FASTECC_B200_EINVAL, "fastecc_b200_gf_mul_dev: null device pointer");
    CUDA_TRY(launch_gf_mul(a, b, out, n, (cudaStream_t)stream)); g_launches++;
    return 0;
}
int fastecc_b200_gf_inv_dev(const uint32_t* a, uint32_t* out, size_t n, void* stream)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_gf_inv_dev: call fastecc_b200_init() first");
    if (n && (!a || !out)) return fail(FASTECC_B200_EINVAL, "fastecc_b200_gf_inv_dev: null device pointer");
    CUDA_TRY(launch_gf_inv(a, out, n, (cudaStream_t)stream)); g_launches++;
    return 0;
}
int fastecc_b200_row_scale_dev(uint32_t* d, size_t n_rows, size_t size, size_t pitch, const uint32_t* d_consts, void* stream)
{
    const char* who = "fastecc_b200_row_scale_dev";
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d || !d_consts) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (size == 0 || pitch < size || pitch > 0xFFFFFFF0u || pitch % 4 || ((uintptr_t)d) % 16) return fail(FASTECC_B200_EINVAL, "%s: needs SIZE >= 1, SIZE <= pitch_words <= 2^32 - 16, pitch %% 4 == 0 and a 16-byte aligned buffer (pad words of a row are scaled too)", who);
    CUDA_TRY(launch_row_scale(d, n_rows, (uint32_t)((size + 3) / 4), (uint32_t)(pitch / 4), d_consts, g_ctx->num_sms, (cudaStream_t)stream)); g_launches++;
    return 0;
}

static int recode_args(const void* a, const void* b, size_t n_blocks, size_t W, size_t pitch, const char* who)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!a || !b) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (W == 0 || W > 1024 || W % 4) return fail(FASTECC_B200_EINVAL, "%s: words_per_block=%zu must be a multiple of 4 in [4, 1024] (10-bit positions, GF.md:84)", who, W);
    if (pitch < W + 1 || pitch % 4) return fail(FASTECC_B200_EINVAL, "%s: pitch_words must be >= words_per_block + 1 and a multiple of 4", who);
    if (((uintptr_t)a) % 16 || ((uintptr_t)b) % 16) return fail(FASTECC_B200_EINVAL, "%s: buffers must be 16-byte aligned", who);
    if (n_blocks >= (1ull << 31)) return fail(FASTECC_B200_EINVAL, "%s: too many blocks", who);
    return 0;
}
int fastecc_b200_bytes_to_gfp_dev(const void* d_bytes, uint32_t* d_words, size_t n_blocks, size_t W, size_t pitch, void* stream)
{
    if (int rc = recode_args(d_bytes, d_words, n_blocks, W, pitch, "fastecc_b200_bytes_to_gfp_dev")) return rc;
    CUDA_TRY(launch_bytes_to_gfp(d_bytes, d_words, n_blocks, (uint32_t)W, pitch, (cudaStream_t)stream)); g_launches++;
    return 0;
}
int fastecc_b200_gfp_to_bytes_dev(const uint32_t* d_words, void* d_bytes, size_t n_blocks, size_t W, size_t pitch, void* stream)
{
    if (int rc = recode_args(d_words, d_bytes, n_blocks, W, pitch, "fastecc_b200_gfp_to_bytes_dev")) return rc;
    CUDA_TRY(launch_gfp_to_bytes(d_words, d_bytes, n_blocks, (uint32_t)W, pitch, (cudaStream_t)stream)); g_launches++;
    return 0;
}

int fastecc_b200_rs_encode_asym_dev(uint32_t* d, size_t N, size_t M, size_t size, size_t pitch, void* stream)
{
    const char* who = "fastecc_b200_rs_encode_asym_dev";
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (int rc = check_shape(N, size, FASTECC_B200_MAX_LOG_N_ENCODE, who)) return rc;
    if (!is_pow2(M) || M > N) return fail(FASTECC_B200_EINVAL, "%s: M=%zu must be a power of two in [1, N]", who, M);
    if (pitch < size || pitch > 0xFFFFFFF0u || pitch % 4 || ((uintptr_t)d) % 16) return fail(FASTECC_B200_EINVAL, "%s: needs SIZE_words <= pitch_words <= 2^32 - 16, pitch %% 4 == 0 and a 16-byte aligned buffer", who);
    if ((unsigned long long)N * (pitch / 4) >= (1ull << 32)) return fail(FASTECC_B200_EINVAL, "%s: buffer too large (32-bit chunk indexing)", who);
    return run_aligned_asym(c, d, N, M, size, pitch, (cudaStream_t)stream);
}

int fastecc_b200_rs_encode_asym(uint32_t** data, size_t N, size_t M, size_t size)
{
    const char* who = "fastecc_b200_rs_encode_asym";
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!data) return fail(FASTECC_B200_EINVAL, "%s: null block table", who);
    if (int rc = check_shape(N, size, FASTECC_B200_MAX_LOG_N_ENCODE, who)) return rc;
    if (!is_pow2(M) || M > N) return fail(FASTECC_B200_EINVAL, "%s: M=%zu must be a power of two in [1, N]", who, M);
    for (size_t i = 0; i < N; i++) if (!data[i]) return fail(FASTECC_B200_EINVAL, "%s: data[%zu] is null", who, i);
    std::lock_guard<std::mutex> host_lock(g_host_mu);
    const size_t pitch = (size + 3) / 4 * 4;
    CUDA_TRY(c->staging.reserve(N * pitch * sizeof(uint32_t)));
    uint32_t* dv = (uint32_t*)c->staging.p;
    cudaStream_t st = c->stream;
    bool contiguous = true;
    for (size_t i = 1; i < N; i++) if (data[i] != data[0] + i * size) { contiguous = false; break; }
    if (pitch != size) CUDA_TRY(cudaMemsetAsync(dv, 0, N * pitch * sizeof(uint32_t), st));
    if (contiguous) CUDA_TRY(cudaMemcpy2DAsync(dv, pitch * 4, data[0], size * 4, size * 4, N, cudaMemcpyHostToDevice, st));
    else for (size_t i = 0; i < N; i++) CUDA_TRY(cudaMemcpyAsync(dv + i * pitch, data[i], size * 4, cudaMemcpyHostToDevice, st));
    if (int rc = run_aligned_asym(c, dv, N, M, size, pitch, st)) return rc;
    if (contiguous) CUDA_TRY(cudaMemcpy2DAsync(data[0], size * 4, dv, pitch * 4, size * 4, M, cudaMemcpyDeviceToHost, st));
    else for (size_t i = 0; i < M; i++) CUDA_TRY(cudaMemcpyAsync(data[i], dv + i * pitch, size * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

int fastecc_b200_rs_encode_shard_pass(uint32_t* d_local, size_t N, int n_ranks, int rank, size_t size, size_t pitch, int which, void* stream)
{
    const char* who = "fastecc_b200_rs_encode_shard_pass";
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d_local || which < 0 || which > 2 || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    if (!shard_supported(N, (uint32_t)n_ranks)) return fail(FASTECC_B200_EINVAL, "%s: N=%zu cannot be sharded over %d ranks (need a power of two 2^11..2^19 with N2 %% ranks == 0)", who, N, n_ranks);
    if (size == 0 || pitch < size || pitch > 0xFFFFFFF0u || pitch % 4 || ((uintptr_t)d_local) % 16) return fail(FASTECC_B200_EINVAL, "%s: needs SIZE >= 1, a 16-byte aligned buffer and pitch %% 4 == 0", who);
    if ((unsigned long long)(N / n_ranks) * (pitch / 4) >= (1ull << 32)) return fail(FASTECC_B200_EINVAL, "%s: local buffer too large", who);
    cudaStream_t st = (cudaStream_t)stream;
    Buffers b{d_local, nullptr, c->d_tw, (uint32_t)pitch, (uint32_t)size};
    PassParams p = plan_encode_shard(b, N, (uint32_t)n_ranks, (uint32_t)rank, which);
    std::vector<PassParams> one{p};
    if (int rc = attach_tables(c, 0x80000000u | (uint32_t)n_ranks << 16 | (uint32_t)rank << 8 | ilog2(N), one, st, which, 3)) return rc;
    CUDA_TRY(launch_pass(one[0], c->num_sms, st)); g_launches++;
    return 0;
}

int fastecc_b200_rs_encode_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank, size_t size, size_t pitch,
                                          int which, void* stream)
{
    const char* who = "fastecc_b200_rs_encode_shard_pass_p2p";
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d_src || !d_peers || which < 0 || which > 2 || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    if (!shard_p2p_supported(N, (uint32_t)n_ranks))
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu cannot be sharded over %d ranks with fused exchange (need 2^11..2^19, ranks <= 8 and <= both tile heights / 32)", who, N, n_ranks);
    if (size == 0 || pitch < size || pitch > 0xFFFFFFF0u || pitch % 4 || ((uintptr_t)d_src) % 16) return fail(FASTECC_B200_EINVAL, "%s: needs SIZE >= 1, 16-byte aligned buffers and pitch %% 4 == 0", who);
    for (int r = 0; r < n_ranks; ++r)
        if (!d_peers[r] || ((uintptr_t)d_peers[r]) % 16) return fail(FASTECC_B200_EINVAL, "%s: peer buffer %d missing or misaligned", who, r);
    if ((unsigned long long)(N / n_ranks) * (pitch / 4) >= (1ull << 32)) return fail(FASTECC_B200_EINVAL, "%s: local buffer too large", who);
    cudaStream_t st = (cudaStream_t)stream;
    PassParams p = plan_encode_shard_p2p(d_src, d_peers, c->d_tw, (uint32_t)pitch, (uint32_t)size, N, (uint32_t)n_ranks, (uint32_t)rank, which);
    std::vector<PassParams> one{p};
    if (int rc = attach_tables(c, 0xA0000000u | (uint32_t)n_ranks << 16 | (uint32_t)rank << 8 | ilog2(N), one, st, which, 3)) return rc;
    CUDA_TRY(launch_pass(one[0], c->num_sms, st)); g_launches++;
    return 0;
}

int fastecc_b200_ntt_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank, size_t size, size_t pitch,
                                    int inverse, int which, void* stream)
{
    const char* who = "fastecc_b200_ntt_shard_pass_p2p";
    Context* c = g_ctx;
    if (!c) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d_src || !d_peers || which < 0 || which > 1 || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    if (!ntt_shard_p2p_supported(N, (uint32_t)n_ranks))
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu cannot be sharded over %d ranks (need 2^11..2^20, ranks <= 8, first tile height >= 32 * ranks)", who, N, n_ranks);
    if (size == 0 || pitch < size || pitch > 0xFFFFFFF0u || pitch % 4 || ((uintptr_t)d_src) % 16) return fail(FASTECC_B200_EINVAL, "%s: needs SIZE >= 1, 16-byte aligned buffers and pitch %% 4 == 0", who);
    for (int r = 0; r < n_ranks; ++r)
        if (!d_peers[r] || ((uintptr_t)d_peers[r]) % 16) return fail(FASTECC_B200_EINVAL, "%s: peer buffer %d missing or misaligned", who, r);
    if ((unsigned long long)(N / n_ranks) * (pitch / 4) >= (1ull << 32)) return fail(FASTECC_B200_EINVAL, "%s: local buffer too large", who);
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<PassParams> one{plan_ntt_shard_p2p(d_src, d_peers, c->d_tw, (uint32_t)pitch, (uint32_t)size, N, (uint32_t)n_ranks, (uint32_t)rank, inverse != 0, which)};
    if (int rc = attach_tables(c, 0xC0000000u | (inverse ? 1u : 0u) << 28 | (uint32_t)n_ranks << 16 | (uint32_t)rank << 8 | ilog2(N), one, st, which, 2)) return rc;
    CUDA_TRY(launch_pass(one[0], c->num_sms, st)); g_launches++;
    return 0;
}

int fastecc_b200_shard_barrier(uint32_t* const* d_flag_peers, int n_ranks, int rank, uint32_t epoch, void* stream)
{
    const char* who = "fastecc_b200_shard_barrier";
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    if (!d_flag_peers || n_ranks < 1 || n_ranks > 8 || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    for (int r = 0; r < n_ranks; ++r) if (!d_flag_peers[r]) return fail(FASTECC_B200_EINVAL, "%s: flag array of rank %d missing", who, r);
    CUDA_TRY(launch_shard_barrier(d_flag_peers, (uint32_t)n_ranks, (uint32_t)rank, epoch, (cudaStream_t)stream)); g_launches++;
    return 0;
}

// The whole sharded encode / transform of one rank as ONE call: the passes and the barriers between them, enqueued on the
// stream.  *epoch is the rank's barrier counter (starts at 0, same sequence of calls on every rank).
int fastecc_b200_rs_encode_shard_p2p(uint32_t* const* d_x_peers, uint32_t* const* d_y_peers, uint32_t* const* d_flag_peers, uint32_t* epoch,
                                     size_t N, int n_ranks, int rank, size_t size, size_t pitch, void* stream)
{
    const char* who = "fastecc_b200_rs_encode_shard_p2p";
    if (!d_x_peers || !d_y_peers || !d_flag_peers || !epoch || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    if (int rc = fastecc_b200_rs_encode_shard_pass_p2p(d_x_peers[rank], d_y_peers, N, n_ranks, rank, size, pitch, 0, stream)) return rc;
    if (int rc = fastecc_b200_shard_barrier(d_flag_peers, n_ranks, rank, ++*epoch, stream)) return rc;
    if (int rc = fastecc_b200_rs_encode_shard_pass_p2p(d_y_peers[rank], d_x_peers, N, n_ranks, rank, size, pitch, 1, stream)) return rc;
    if (int rc = fastecc_b200_shard_barrier(d_flag_peers, n_ranks, rank, ++*epoch, stream)) return rc;
    return fastecc_b200_rs_encode_shard_pass_p2p(d_x_peers[rank], d_x_peers, N, n_ranks, rank, size, pitch, 2, stream);
}

int fastecc_b200_ntt_shard_p2p(uint32_t* const* d_x_peers, uint32_t* const* d_y_peers, uint32_t* const* d_flag_peers, uint32_t* epoch,
                               size_t N, int n_ranks, int rank, size_t size, size_t pitch, int inverse, void* stream)
{
    const char* who = "fastecc_b200_ntt_shard_p2p";
    if (!d_x_peers || !d_y_peers || !d_flag_peers || !epoch || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    if (int rc = fastecc_b200_ntt_shard_pass_p2p(d_x_peers[rank], d_y_peers, N, n_ranks, rank, size, pitch, inverse, 0, stream)) return rc;
    if (int rc = fastecc_b200_shard_barrier(d_flag_peers, n_ranks, rank, ++*epoch, stream)) return rc;
    if (int rc = fastecc_b200_ntt_shard_pass_p2p(d_y_peers[rank], d_x_peers, N, n_ranks, rank, size, pitch, inverse, 1, stream)) return rc;
    return fastecc_b200_shard_barrier(d_flag_peers, n_ranks, rank, ++*epoch, stream);      // nobody overwrites a Y its owner is still reading
}

// Device buffers that can be mapped into the other ranks' address spaces (cudaMalloc + CUDA IPC: torch's caching
// allocator hands out sub-blocks, which cannot be exported).
void* fastecc_b200_dev_alloc(size_t bytes)
{
    if (!g_ctx) { fail(FASTECC_B200_ENOINIT, "fastecc_b200_dev_alloc: call fastecc_b200_init() first"); return nullptr; }
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); fail(FASTECC_B200_ENOMEM, "fastecc_b200_dev_alloc: cudaMalloc(%zu) failed", bytes); return nullptr; }
    return p;
}
void fastecc_b200_dev_free(void* p) { if (p) cudaFree(p); }
int fastecc_b200_ipc_export(void* d_ptr, void* handle64)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_ipc_export: call fastecc_b200_init() first");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    CUDA_TRY(cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle64, &h, 64);
    return 0;
}
int fastecc_b200_ipc_open(const void* handle64, void** d_ptr)
{
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_ipc_open: call fastecc_b200_init() first");
    cudaIpcMemHandle_t h; memcpy(&h, handle64, 64);
    CUDA_TRY(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}
int fastecc_b200_ipc_close(void* d_ptr)
{
    CUDA_TRY(cudaIpcCloseMemHandle(d_ptr));
    return 0;
}

int fastecc_b200_ntt_u32(uint32_t** data, size_t N, size_t size, int inverse)
{ return run_host(data, N, size, inverse ? 1 : 0, "fastecc_b200_ntt_u32"); }

int fastecc_b200_rs_encode(uint32_t** data, size_t N, size_t size)
{ return run_host(data, N, size, 2, "fastecc_b200_rs_encode"); }

int fastecc_b200_pin_host_buffers(int enable)
{
    std::lock_guard<std::mutex> lk(g_host_mu);
    if (!g_ctx) return fail(FASTECC_B200_ENOINIT, "fastecc_b200_pin_host_buffers: call fastecc_b200_init() first");
    g_ctx->pin_caller = enable != 0;
    if (!enable) {                                                          // turning it off also releases what was page-locked so far
        CUDA_TRY(cudaDeviceSynchronize());
        for (auto& r : g_ctx->registered) { cudaHostUnregister(r.first); cudaGetLastError(); }
        g_ctx->registered.clear();
    }
    return 0;
}

uint32_t fastecc_b200_hash_u32(uint32_t* const* data, size_t N, size_t size)
{
    uint32_t h = 314159253u;
    for (size_t i = 0; i < N; i++) {
        const uint32_t* p = data[i];
        for (size_t k = 0; k < size; k++) h = (h + p[k]) * 123456791u + (h >> 17);
    }
    return h;
}

void* fastecc_b200_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { fail(FASTECC_B200_ENOMEM, "cudaHostAlloc(%zu) failed", bytes); return nullptr; }
    return p;
}
void fastecc_b200_host_free(void* p) { if (p) cudaFreeHost(p); }

} // extern "C"
