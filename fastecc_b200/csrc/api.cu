// extern "C" boundary of fastecc_b200 (include/fastecc_b200.h): context, planning, launches, host<->device staging.
#include "context.h"
#include "plan.h"
#include "ntt_pass.h"
#include "small_dft.h"
#include "byte_recode.h"
#include "elementwise.h"
#include "mixed_radix.h"
#include "repair.h"
#include "update.h"
#include "scrub.h"
#include "reconstruct.h"
#include "batch.h"
#include "locator.h"
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <mutex>
#include <vector>
#include <atomic>
#include <map>
#include <tuple>

using namespace fecc;

namespace {
thread_local char g_err[512] = "no error";
}

namespace fecc {
int fail(int code, const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
}

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

// Stage tables of one pass: built once, on the stream of the first call that needs them.  `ready` is recorded behind the
// build; a call on any other stream waits for it (a no-op once the build has finished).
struct TableSlot { DevBuf buf; cudaEvent_t ready = nullptr; cudaStream_t built_on = nullptr; };
enum Kind { kNtt, kEncode, kEncodeAsym, kShard, kShardP2P, kNttShardP2P, kUpdate };
struct TableKey {                        // what the stage tables of a plan depend on
    int kind, inverse, n_ranks, rank;
    int sub;                             // which pass of a sharded plan, log2(N / M) of an asymmetric encode, r of kUpdate's N = r * 2^k
    int log_n;
    bool operator<(const TableKey& o) const
    { return std::tie(kind, inverse, n_ranks, rank, sub, log_n) < std::tie(o.kind, o.inverse, o.n_ranks, o.rank, o.sub, o.log_n); }
};

// A buffer shared by calls that may come in on different threads and streams (the Y buffer of the two-pass NTT, the repack
// buffer, the destination of the order-3 / order-9 step).  Only a Lease touches it.
struct SharedBuf {
    std::mutex mu;
    DevBuf buf;
    cudaEvent_t done = nullptr;          // recorded behind the last lease's launches
    cudaStream_t last = nullptr;
    bool used = false;
    void destroy() { buf.release(); if (done) cudaEventDestroy(done); done = nullptr; used = false; }
};
// Exclusive use of a SharedBuf for the launches of one call: the buffer's mutex is held from construction to destruction,
// and the destructor records `done` on the caller's stream on every exit path, error returns included.  A user on another
// stream waits for `done` in acquire(), so two transforms that need the same buffer run one after the other on the device
// and the buffer is never reallocated under launches that still use it.
// Lock order: g_host_mu -> packed -> repair -> (scratch | mixed, never both at once) -> g_mu.
class Lease {
public:
    Lease(SharedBuf* s, cudaStream_t st) : s_(s), st_(st) { if (s_) lk_ = std::unique_lock<std::mutex>(s_->mu); }
    ~Lease() { if (s_ && s_->done) { s_->used = true; s_->last = st_; cudaEventRecord(s_->done, st_); } }
    cudaError_t acquire(size_t need)
    {
        if (need > s_->buf.bytes && s_->used) { cudaError_t e = cudaEventSynchronize(s_->done); if (e != cudaSuccess) return e; }   // about to be reallocated
        cudaError_t e = s_->buf.reserve(need);
        if (e == cudaSuccess && !s_->done) e = cudaEventCreateWithFlags(&s_->done, cudaEventDisableTiming);
        if (e == cudaSuccess && s_->used && s_->last != st_) e = cudaStreamWaitEvent(st_, s_->done, 0);
        return e;
    }
    uint32_t* ptr() const { return s_ ? (uint32_t*)s_->buf.p : nullptr; }
private:
    SharedBuf* s_;
    cudaStream_t st_;
    std::unique_lock<std::mutex> lk_;
};

struct Context {
    int device = -1;
    int num_sms = 0;
    uint4* d_tw = nullptr;
    SharedBuf scratch;   // Y buffer of the two-pass NTT and of the asymmetric encode
    SharedBuf packed;    // repacked copy for unaligned device layouts
    SharedBuf mixed;     // destination of the order-3 / order-9 step of the N = 3 * 2^k, 9 * 2^k transforms
    SharedBuf repair;    // workspace of fastecc_b200_rs_repair: N + M rows of one column chunk; and of fastecc_b200_rs_update, _scrub and _reconstruct
    struct HostList { uint32_t* p = nullptr; size_t cap = 0; cudaEvent_t copied = nullptr; };
    std::vector<HostList> lists;         // page-locked copies of host arrays for rs_update and rs_reconstruct (used under repair's lease)
    size_t next_list = 0;                // the one to wait for next once there are kMaxLists
    DevBuf staging;      // device copy for the host (T**) entry points (serialised by g_host_mu)
    std::map<TableKey, std::vector<TableSlot>> tables;   // one slot per pass of the plan
    bool pin_caller = false;                          // fastecc_b200_pin_host_buffers()
    std::vector<std::pair<char*, size_t>> registered; // caller buffers we page-locked in place (cudaHostRegister)
    cudaStream_t stream = nullptr;       // compute
    cudaStream_t h2d = nullptr, d2h = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_done;
};

Context* g_ctx = nullptr;
std::mutex g_mu;          // guards g_ctx and the table cache (short critical sections)
std::mutex g_host_mu;     // held by the host (T**) entry points for their whole duration: they share the staging buffer, three streams and the chunk events
std::atomic<unsigned long long> g_launches{0};

// The live context, or nullptr after recording the ENOINIT message.
Context* ctx(const char* who)
{
    if (!g_ctx) fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    return g_ctx;
}

constexpr size_t kMaxPitch = 0xFFFFFFF0u;
// The shape of every transform and encode, checked before anything is allocated, copied or launched: SIZE in [1, 2^32 - 16];
// N = r * 2^k with 2^k <= 2^max_log and r = 1, or r in {3, 9} if `mixed_ok` (mixed_radix.cu); M divides N (the M parity blocks
// of an encode; M = N for a transform); r * run_pitch <= 2^32 - 16, since the order-2^k steps of r > 1 run on every r-th row of
// the buffer at the row pitch `run_pitch` (the caller's for an aligned layout, ceil(SIZE / 4) * 4 for a repacked or staged one).
int check_order(size_t N, size_t M, size_t size, size_t run_pitch, size_t max_log, bool mixed_ok, const char* who)
{
    if (size == 0 || size > kMaxPitch) return fail(FASTECC_B200_EINVAL, "%s: SIZE_words=%zu must be in [1, 2^32 - 16]", who, size);
    const Order o = split_order(N);
    if (!o.r || (o.r != 1 && !mixed_ok) || o.log2_m > max_log)
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu must be a power of two in [1, 2^%zu]%s (P-1 = 2^20*4095)", who, N, max_log, mixed_ok ? ", or 3 or 9 times one" : "");
    if (M == 0 || N % M) return fail(FASTECC_B200_EINVAL, "%s: M=%zu must divide N=%zu", who, M, N);
    if ((unsigned long long)o.r * run_pitch > kMaxPitch) return fail(FASTECC_B200_EINVAL, "%s: %u * pitch_words (%zu) must be <= 2^32 - 16", who, o.r, run_pitch);
    return 0;
}
bool is_aligned(const void* d, size_t pitch) { return pitch % 4 == 0 && (uintptr_t)d % 16 == 0; }
size_t padded_pitch(size_t size) { return (size + 3) / 4 * 4; }
// A device buffer of `rows` rows of `pitch` words, the first SIZE of each meaningful: d != null, 1 <= SIZE <= pitch <= 2^32 - 16,
// fewer than 2^32 16-byte chunks (the kernels index them in 32 bits); `aligned`: pitch % 4 == 0 and d 16-byte aligned as well.
int check_rows(const void* d, size_t rows, size_t size, size_t pitch, bool aligned, const char* who)
{
    if (!d) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (size == 0 || pitch < size || pitch > kMaxPitch) return fail(FASTECC_B200_EINVAL, "%s: needs 1 <= SIZE_words (%zu) <= pitch_words (%zu) <= 2^32 - 16", who, size, pitch);
    if (aligned && (pitch % 4 || (uintptr_t)d % 16)) return fail(FASTECC_B200_EINVAL, "%s: needs pitch_words %% 4 == 0 and a 16-byte aligned buffer", who);
    if ((unsigned long long)rows * ((pitch + 3) / 4) >= (1ull << 32))
        return fail(FASTECC_B200_EINVAL, "%s: buffer of %zu x %zu words is 64 GiB or more (32-bit chunk indexing)", who, rows, pitch);
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
    if (cudaPointerGetAttributes(&at, base) != cudaSuccess) { clear_cuda_error(); return; }
    if (at.type != cudaMemoryTypeUnregistered) return;                      // already pinned (by us earlier, or by the caller)
    char* b = (char*)base;
    for (size_t i = 0; i < c->registered.size();) {                         // a stale, overlapping registration (the caller re-allocated): drop it
        auto& r = c->registered[i];
        if (b < r.first + r.second && r.first < b + bytes) { cudaHostUnregister(r.first); clear_cuda_error(); r = c->registered.back(); c->registered.pop_back(); }
        else ++i;
    }
    if (cudaHostRegister(base, bytes, cudaHostRegisterDefault) == cudaSuccess) c->registered.emplace_back(b, bytes);
    else clear_cuda_error();
}

// The table block of slot `sl` (caller holds g_mu): built on first use by the one launch `build(buffer)` on `st` (a block enters
// the cache only once it is allocated and its build launched); a call on another stream waits for the build.
template <class Build>
int use_table(TableSlot& sl, size_t bytes, cudaStream_t st, Build build)
{
    if (!sl.buf.p) {
        DevBuf nb;
        cudaEvent_t ev = nullptr;
        cudaError_t e = nb.reserve(bytes);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (e == cudaSuccess) e = build((uint4*)nb.p);
        if (e == cudaSuccess) e = cudaEventRecord(ev, st);
        if (e != cudaSuccess) { nb.release(); if (ev) cudaEventDestroy(ev); CUDA_TRY(e); }
        g_launches++;
        sl.buf = nb; sl.ready = ev; sl.built_on = st;
    } else if (sl.built_on != st) {
        CUDA_TRY(cudaStreamWaitEvent(st, sl.ready, 0));
    }
    return 0;
}

// Stage tables of `plan` under cache key `key`, attached to the passes.
int attach_tables(Context* c, const TableKey& key, std::vector<PassParams>& plan, cudaStream_t st)
{
    std::lock_guard<std::mutex> lk(g_mu);
    std::vector<TableSlot>& slots = c->tables[key];
    slots.resize(plan.size());
    for (size_t i = 0; i < plan.size(); ++i) {
        TableSlot& sl = slots[i];
        if (int rc = use_table(sl, table_bytes(plan[i]), st, [&](uint4* t) { return launch_build_tables(plan[i], t, st); })) return rc;
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

// N < 2^kMinLogR: one small-DFT launch, the transform of order N or (`encode`) the whole encode of N data blocks.
int small_dft(Context* c, uint32_t* x, size_t N, size_t size, size_t pitch, bool inverse, bool encode, cudaStream_t st)
{
    const uint32_t z = (uint32_t)(gf::M / N) * (inverse ? (uint32_t)-1 : 1u) & (gf::M - 1);
    const uint32_t q = encode ? (uint32_t)(gf::M / (2 * N)) : 0;
    const gf::Tw in = gf::make_tw(gf::inv((uint32_t)N));
    CUDA_TRY(launch_small_dft(x, (uint32_t)(pitch / 4), (uint32_t)((size + 3) / 4), (uint32_t)N, z, encode, q, make_uint4(in.w, in.whi, in.wlo, 0), c->d_tw, st));
    g_launches++;
    return 0;
}

// The transform of order N = 2^k, 3 * 2^k or 9 * 2^k, in place on an aligned, padded device buffer.
int ntt(Context* c, uint32_t* x, size_t N, size_t size, size_t pitch, bool inverse, cudaStream_t st)
{
    const Order o = split_order(N);
    if (o.r > 1) {                                        // N = r * L (mixed_radix.cu)
        const size_t L = N / o.r;
        if (L > 1)                                        // step 1: r transforms of order L, each on every r-th row (row pitch r times larger), in place
            for (uint32_t n1 = 0; n1 < o.r; ++n1)
                if (int rc = ntt(c, x + (size_t)n1 * pitch, L, size, (size_t)o.r * pitch, inverse, st)) return rc;
        const uint32_t pitch4 = (uint32_t)(pitch / 4), s4 = (uint32_t)((size + 3) / 4);
        Lease y(&c->mixed, st);                           // step 2: twiddles + order-r transform, into natural order (out of place), then back
        CUDA_TRY(y.acquire(N * pitch * sizeof(uint32_t)));
        CUDA_TRY(launch_radix_pass(x, y.ptr(), pitch4, s4, o.r, (uint32_t)L, inverse, c->d_tw, c->num_sms, st)); g_launches++;
        CUDA_TRY(cudaMemcpy2DAsync(x, pitch * 4, y.ptr(), pitch * 4, (size_t)s4 * 16 < pitch * 4 ? (size_t)s4 * 16 : pitch * 4, N, cudaMemcpyDeviceToDevice, st));
        return 0;
    }
    if (N < ((size_t)1 << kMinLogR)) return small_dft(c, x, N, size, pitch, inverse, false, st);
    const bool need_y = !single_pass(ilog2(N));                              // the two-pass NTT ping-pongs through Y
    Lease y(need_y ? &c->scratch : nullptr, st);
    if (need_y) CUDA_TRY(y.acquire(N * pitch * sizeof(uint32_t)));
    Buffers b{x, y.ptr(), c->d_tw, (uint32_t)pitch, (uint32_t)size};
    std::vector<PassParams> plan = plan_ntt(b, N, inverse);
    if (int rc = attach_tables(c, {kNtt, inverse, 0, 0, 0, (int)ilog2(N)}, plan, st)) return rc;
    return launch_plan(c, plan, st);
}

// The whole encode of a power-of-two N: one small-DFT launch or the passes of plan_encode (timed for rs_encode_dev_timed).
int encode_pow2(Context* c, uint32_t* x, size_t N, size_t size, size_t pitch, cudaStream_t st, PassTimer* timer)
{
    if (N < ((size_t)1 << kMinLogR)) return small_dft(c, x, N, size, pitch, false, true, st);
    Buffers b{x, nullptr, c->d_tw, (uint32_t)pitch, (uint32_t)size};
    std::vector<PassParams> plan = plan_encode(b, N);
    if (int rc = attach_tables(c, {kEncode, 0, 0, 0, 0, (int)ilog2(N)}, plan, st)) return rc;
    return launch_plan(c, plan, st, timer);
}

// N = 2^k, 3 * 2^k or 9 * 2^k data blocks -> M parity blocks (M | N) in rows [0, M) of an aligned, padded device buffer; rows
// [M, N) are left undefined.
int encode(Context* c, uint32_t* x, size_t N, size_t M, size_t size, size_t pitch, cudaStream_t st, PassTimer* timer = nullptr)
{
    const Order ord = split_order(N), ratio = split_order(N / M);            // N = r * L, D = N / M = s * 2^i
    if (ord.r == 1 && M == N) return encode_pow2(c, x, N, size, pitch, st, timer);
    if (ord.r == 1) {                                     // power of two, M = N / 2^i
        size_t M0 = N;                                    // what the passes produce; M0 >= M
        const bool native = N > ((size_t)1 << kMaxLogR);
        if (!native) { if (int rc = encode_pow2(c, x, N, size, pitch, st, nullptr)) return rc; }
        Lease y(&c->scratch, st);
        CUDA_TRY(y.acquire(N * pitch * sizeof(uint32_t)));
        if (native) {
            M0 = M;
            while (!asym_native(N, M0)) M0 *= 2;          // M0 = max(M, N1)
            Buffers b{x, y.ptr(), c->d_tw, (uint32_t)pitch, (uint32_t)size};
            std::vector<PassParams> plan = plan_encode_asym(b, N, M0);
            if (int rc = attach_tables(c, {kEncodeAsym, 0, 0, 0, (int)ilog2(N / M0), (int)ilog2(N)}, plan, st)) return rc;
            if (int rc = launch_plan(c, plan, st)) return rc;
        }
        if (M0 != M) {                                    // keep every (M0/M)-th parity block: gather through the scratch buffer
            CUDA_TRY(cudaMemcpy2DAsync(y.ptr(), pitch * 4, x, (M0 / M) * pitch * 4, size * 4, M, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpy2DAsync(x, pitch * 4, y.ptr(), pitch * 4, size * 4, M, cudaMemcpyDeviceToDevice, st));
        }
        return 0;
    }
    // N = r * L (DESIGN 3e, 3f): step 1, r inverse transforms of order L on every r-th row; step 2 in place, launch_radix_encode
    // for D = 1, else launch_radix_fold; step 3, the r / s forward transforms of order T = L / 2^f on rows d + r*t, of whose
    // outputs every 2^(i-f)-th is gathered into rows [0, M).
    const uint32_t r = ord.r, s = ratio.r, u = r / s, log_d2 = ratio.log2_m;
    const uint32_t pitch4 = (uint32_t)(pitch / 4), s4 = (uint32_t)((size + 3) / 4);
    const size_t L = N / r;
    uint32_t log_fold = 0;                                // fold as far as L / 2^f rows still give every SM 1024 threads
    while (log_fold < log_d2 && (L >> (log_fold + 1)) * s4 >= (size_t)c->num_sms * 1024) ++log_fold;
    const size_t T = L >> log_fold, keep = ((size_t)1 << log_d2) >> log_fold;
    if (L > 1)
        for (uint32_t n1 = 0; n1 < r; ++n1)
            if (int rc = ntt(c, x + (size_t)n1 * pitch, L, size, (size_t)r * pitch, true, st)) return rc;
    if (M == N) CUDA_TRY(launch_radix_encode(x, pitch4, s4, r, (uint32_t)L, c->d_tw, c->num_sms, st));
    else        CUDA_TRY(launch_radix_fold(x, pitch4, s4, r, (uint32_t)L, s, log_d2, log_fold, c->d_tw, c->num_sms, st));
    g_launches++;
    if (T > 1)                                            // parity d + u*j'' lands in row d + r*keep*j''
        for (uint32_t d = 0; d < u; ++d)
            if (int rc = ntt(c, x + (size_t)d * pitch, T, size, (size_t)r * pitch, false, st)) return rc;
    if (u == r && keep == 1) return 0;                    // already rows [0, M)
    Lease y(&c->scratch, st);                             // gather the groups of u rows through the scratch buffer
    CUDA_TRY(y.acquire(M * pitch * sizeof(uint32_t)));
    const size_t groups = M / u, spitch = (size_t)r * keep * pitch * 4, width = ((u - 1) * pitch + size) * 4;
    if (spitch < ((size_t)1 << 30))
        CUDA_TRY(cudaMemcpy2DAsync(y.ptr(), u * pitch * 4, x, spitch, width, groups, cudaMemcpyDeviceToDevice, st));
    else                                                  // beyond what a 2D copy's pitch may be: fewer than 64 groups then (check_rows)
        for (size_t g = 0; g < groups; ++g)
            CUDA_TRY(cudaMemcpyAsync(y.ptr() + g * u * pitch, x + g * r * keep * pitch, width, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpy2DAsync(x, pitch * 4, y.ptr(), pitch * 4, size * 4, M, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// A device entry point's buffer: run `transform(x, pitch)` on it in place if it is aligned, else on a packed copy of which
// rows [0, rows_back) are copied back.
template <class Transform>
int run_repacked(Context* c, uint32_t* d, size_t N, size_t rows_back, size_t size, size_t pitch, cudaStream_t st, Transform transform)
{
    if (is_aligned(d, pitch)) return transform(d, pitch);
    // unaligned layout: repack into a padded copy, transform, copy the SIZE data words back
    const size_t ppitch = padded_pitch(size);
    Lease pk(&c->packed, st);
    CUDA_TRY(pk.acquire(N * ppitch * sizeof(uint32_t)));
    CUDA_TRY(launch_pack(d, pitch, pk.ptr(), ppitch, N, (uint32_t)size, st)); g_launches++;
    if (int rc = transform(pk.ptr(), ppitch)) return rc;
    CUDA_TRY(launch_unpack(pk.ptr(), ppitch, d, pitch, rows_back, (uint32_t)size, st)); g_launches++;
    return 0;
}

// The device entry points, validated in full before anything is allocated or launched.  Unaligned layouts are repacked
// (run_repacked), except where `repack_ok` is false: there they are rejected.
int ntt_dev(uint32_t* d, size_t N, size_t size, size_t pitch, bool inverse, void* stream, const char* who)
{
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_rows(d, N, size, pitch, false, who)) return rc;
    if (int rc = check_order(N, N, size, is_aligned(d, pitch) ? pitch : padded_pitch(size), FASTECC_B200_MAX_LOG_N, true, who)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    return run_repacked(c, d, N, N, size, pitch, st, [&](uint32_t* x, size_t p) { return ntt(c, x, N, size, p, inverse, st); });
}

int encode_dev(uint32_t* d, size_t N, size_t M, size_t size, size_t pitch, void* stream, bool mixed_ok, bool repack_ok, const char* who,
               PassTimer* timer = nullptr)
{
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_rows(d, N, size, pitch, !repack_ok, who)) return rc;
    if (int rc = check_order(N, M, size, is_aligned(d, pitch) ? pitch : padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, mixed_ok, who)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    return run_repacked(c, d, N, M, size, pitch, st, [&](uint32_t* x, size_t p) { return encode(c, x, N, M, size, p, st, timer); });
}

// The host (T**) entry points: the N blocks are staged in a padded device copy, `transform(x, SIZE, pitch)` runs on it in place
// on the context's stream, and rows [0, rows_back) are copied back.
template <class Transform>
int run_host(Context* c, uint32_t** data, size_t N, size_t rows_back, size_t size, const char* who, Transform transform)
{
    if (!data) return fail(FASTECC_B200_EINVAL, "%s: null block table", who);
    for (size_t i = 0; i < N; i++) if (!data[i]) return fail(FASTECC_B200_EINVAL, "%s: data[%zu] is null", who, i);
    std::lock_guard<std::mutex> host_lock(g_host_mu);
    const size_t pitch = padded_pitch(size);
    CUDA_TRY(c->staging.reserve(N * pitch * sizeof(uint32_t)));
    uint32_t* dv = (uint32_t*)c->staging.p;
    cudaStream_t st = c->stream;
    bool contiguous = true;
    for (size_t i = 1; i < N; i++) if (data[i] != data[0] + i * size) { contiguous = false; break; }
    if (pitch != size) CUDA_TRY(cudaMemsetAsync(dv, 0, N * pitch * sizeof(uint32_t), st));
    // Large contiguous arrays of which every row comes back: the word columns are independent codewords, so the array is cut
    // into column chunks and H2D(chunk c+1), the transform of chunk c and D2H(chunk c-1) run concurrently on three streams
    // (PCIe is full duplex).
    constexpr size_t cw = 128;                            // words per column chunk
    if (rows_back == N && contiguous && pitch == size && size >= 2 * cw && N * size * 4 >= ((size_t)32 << 20)) {
        pin_caller_array(c, data[0], N * size * sizeof(uint32_t));
        const size_t nchunks = (size + cw - 1) / cw;
        while (c->ev_in.size() < nchunks) { cudaEvent_t e; CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->ev_in.push_back(e); }
        while (c->ev_done.size() < nchunks) { cudaEvent_t e; CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c->ev_done.push_back(e); }
        for (size_t k = 0; k < nchunks; ++k) {
            const size_t c0 = k * cw, w = (c0 + cw <= size) ? cw : size - c0;
            CUDA_TRY(cudaMemcpy2DAsync(dv + c0, pitch * 4, data[0] + c0, size * 4, w * 4, N, cudaMemcpyHostToDevice, c->h2d));
            CUDA_TRY(cudaEventRecord(c->ev_in[k], c->h2d));
            CUDA_TRY(cudaStreamWaitEvent(st, c->ev_in[k], 0));
            if (int rc = transform(dv + c0, w, pitch)) return rc;
            CUDA_TRY(cudaEventRecord(c->ev_done[k], st));
            CUDA_TRY(cudaStreamWaitEvent(c->d2h, c->ev_done[k], 0));
            CUDA_TRY(cudaMemcpy2DAsync(data[0] + c0, size * 4, dv + c0, pitch * 4, w * 4, N, cudaMemcpyDeviceToHost, c->d2h));
        }
        CUDA_TRY(cudaStreamSynchronize(c->d2h));
        CUDA_TRY(cudaStreamSynchronize(st));
        return 0;
    }
    if (contiguous) CUDA_TRY(cudaMemcpy2DAsync(dv, pitch * 4, data[0], size * 4, size * 4, N, cudaMemcpyHostToDevice, st));
    else for (size_t i = 0; i < N; i++) CUDA_TRY(cudaMemcpyAsync(dv + i * pitch, data[i], size * 4, cudaMemcpyHostToDevice, st));
    if (int rc = transform(dv, size, pitch)) return rc;
    if (contiguous) CUDA_TRY(cudaMemcpy2DAsync(data[0], size * 4, dv, pitch * 4, size * 4, rows_back, cudaMemcpyDeviceToHost, st));
    else for (size_t i = 0; i < rows_back; i++) CUDA_TRY(cudaMemcpyAsync(data[i], dv + i * pitch, size * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// The host entry points, validated as the device ones (at the pitch of the staged copy) before anything is staged.
int ntt_host(uint32_t** data, size_t N, size_t size, bool inverse, const char* who)
{
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, N, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N, true, who)) return rc;
    return run_host(c, data, N, N, size, who, [&](uint32_t* x, size_t w, size_t pitch) { return ntt(c, x, N, w, pitch, inverse, c->stream); });
}

int encode_host(uint32_t** data, size_t N, size_t M, size_t size, bool mixed_ok, const char* who)
{
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, mixed_ok, who)) return rc;
    return run_host(c, data, N, M, size, who, [&](uint32_t* x, size_t w, size_t pitch) { return encode(c, x, N, M, w, pitch, c->stream); });
}

// One pass of a sharded encode / transform (the three fastecc_b200_*_shard_pass* entry points): kShard (exchange by the
// caller, `peers` unused), kShardP2P or kNttShardP2P (exchange fused into the stores to `peers`).
int shard_pass(Kind kind, const uint32_t* src, uint32_t* const* peers, size_t N, int n_ranks, int rank, size_t size, size_t pitch,
               int inverse, int which, void* stream, const char* who)
{
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    const bool p2p = kind != kShard;
    const int passes = kind == kNttShardP2P ? 2 : 3;
    if (!src || (p2p && !peers) || which < 0 || which >= passes || rank < 0 || rank >= n_ranks) return fail(FASTECC_B200_EINVAL, "%s: bad arguments", who);
    const uint32_t G = (uint32_t)n_ranks;
    if (!(kind == kShard ? shard_supported(N, G) : kind == kShardP2P ? shard_p2p_supported(N, G) : ntt_shard_p2p_supported(N, G)))
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu cannot be sharded over %d ranks (fastecc_b200_shard_geometry tells which can)", who, N, n_ranks);
    if (int rc = check_rows(src, N / G, size, pitch, true, who)) return rc;
    for (int r = 0; p2p && r < n_ranks; ++r)
        if (!peers[r] || ((uintptr_t)peers[r]) % 16) return fail(FASTECC_B200_EINVAL, "%s: peer buffer %d missing or misaligned", who, r);
    cudaStream_t st = (cudaStream_t)stream;
    Buffers b{const_cast<uint32_t*>(src), nullptr, c->d_tw, (uint32_t)pitch, (uint32_t)size};
    std::vector<PassParams> plan{kind == kShard ? plan_encode_shard(b, N, G, (uint32_t)rank, which)
                                 : kind == kShardP2P ? plan_encode_shard_p2p(src, peers, c->d_tw, (uint32_t)pitch, (uint32_t)size, N, G, (uint32_t)rank, which)
                                 : plan_ntt_shard_p2p(src, peers, c->d_tw, (uint32_t)pitch, (uint32_t)size, N, G, (uint32_t)rank, inverse != 0, which)};
    if (int rc = attach_tables(c, {kind, inverse != 0, n_ranks, rank, which, (int)ilog2(N)}, plan, st)) return rc;
    return launch_plan(c, plan, st);
}

// Words per column chunk of a repair: the padded SIZE if the (N + M)-row workspace of it fits in kMaxRepairBytes, else the
// widest multiple of 4 that does.
constexpr size_t kMaxRepairBytes = (size_t)4 << 30;
size_t repair_chunk_words(size_t N, size_t M, size_t size)
{
    const size_t w = padded_pitch(size), cap = kMaxRepairBytes / 4 / (N + M) / 4 * 4;
    return w <= cap ? w : cap;
}

// The repair of one stripe (DESIGN 3g), once per column chunk [c0, c0 + cols) of the caller's rows: load the data with the lost
// rows zeroed, encode it, syndromes, inverse order-M transform, split, the forward order-N / order-M transforms of what was lost,
// scatter into the lost rows.  Transforms of order 1 are the identity and are skipped.
int repair(Context* c, const fastecc_b200_repair* R, uint32_t* data, size_t dpitch, uint32_t* parity, size_t ppitch, size_t size, cudaStream_t st)
{
    const size_t N = R->N, M = R->M, w = repair_chunk_words(N, M, size);
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire((N + M) * w * sizeof(uint32_t)));
    uint32_t* x = ws.ptr();
    for (size_t c0 = 0; c0 < size; c0 += w) {
        const size_t cols = size - c0 < w ? size - c0 : w;
        CUDA_TRY(launch_repair_load(N, R->d_lost, data, dpitch, c0, x, w, cols, c->num_sms, st)); g_launches++;
        if (int rc = encode(c, x, N, M, cols, w, st)) return rc;
        CUDA_TRY(launch_repair_syndrome(M, R->d_cs, parity, ppitch, c0, size, x, w, cols, c->num_sms, st)); g_launches++;
        if (M > 1) { if (int rc = ntt(c, x, M, cols, w, true, st)) return rc; }
        CUDA_TRY(launch_repair_split(R, x, w, cols, c->num_sms, st)); g_launches++;
        if (R->ned && N > 1) { if (int rc = ntt(c, x, N, cols, w, false, st)) return rc; }
        if (R->nep && M > 1) { if (int rc = ntt(c, x + N * w, M, cols, w, false, st)) return rc; }
        CUDA_TRY(launch_repair_scatter(R, data, dpitch, parity, ppitch, c0, size, x, w, cols, c->num_sms, st)); g_launches++;
    }
    return 0;
}

// Whether a device buffer of `rows` rows (the first SIZE words of each) shares a word with another.
bool rows_overlap(const void* a, size_t a_rows, size_t a_pitch, const void* b, size_t b_rows, size_t b_pitch, size_t size)
{
    const uintptr_t a0 = (uintptr_t)a, a1 = a0 + ((a_rows - 1) * a_pitch + size) * 4;
    const uintptr_t b0 = (uintptr_t)b, b1 = b0 + ((b_rows - 1) * b_pitch + size) * 4;
    return a0 < b1 && b0 < a1;
}

// The table T of fastecc_b200_rs_update at order N (update.h), built on first use and cached like the stage tables.
int update_table(Context* c, size_t N, cudaStream_t st, const uint4** T)
{
    const Order o = split_order(N);
    std::lock_guard<std::mutex> lk(g_mu);
    std::vector<TableSlot>& slots = c->tables[{kUpdate, 0, 0, 0, (int)o.r, (int)o.log2_m}];
    slots.resize(1);
    if (int rc = use_table(slots[0], N * sizeof(uint4), st, [&](uint4* t) { return launch_update_table(t, N, st); })) return rc;
    *T = (const uint4*)slots[0].buf.p;
    return 0;
}

// The caller's host array of n words (update's changed rows, the lists and the combination of a reconstruct) into d_dst without
// waiting for the stream: a pageable source could make cudaMemcpyAsync synchronise, so the array goes through one of the context's
// page-locked buffers, one whose last copy has run.
// While fewer than kMaxLists exist, a new one is added when none is free and large enough (one that is new because the array
// outgrew them all is at least twice the largest); after that the buffers are taken in turn, waiting for the copy out of the
// next one, so a caller that queues many calls behind long work holds at most kMaxLists of them.  Freeing page-locked memory
// could synchronise the device, so a buffer is only replaced when it is too small.  The caller holds repair's lease.
constexpr size_t kMaxLists = 8;
int upload_list(Context* c, const uint32_t* src, size_t n, uint32_t* d_dst, cudaStream_t st)
{
    Context::HostList* h = nullptr;
    size_t largest = 0;
    for (Context::HostList& b : c->lists) {
        largest = b.cap > largest ? b.cap : largest;
        if (h || b.cap < n) continue;
        const cudaError_t e = cudaEventQuery(b.copied);
        if (e == cudaSuccess) h = &b;
        else clear_cuda_error();                                     // cudaErrorNotReady: still in flight
    }
    size_t cap = n <= largest ? n : n > 2 * largest ? n : 2 * largest;
    if (cap < 4096) cap = 4096;
    if (!h && c->lists.size() >= kMaxLists) {
        h = &c->lists[c->next_list];
        c->next_list = (c->next_list + 1) % kMaxLists;
        CUDA_TRY(cudaEventSynchronize(h->copied));
        if (h->cap < n) {
            cudaFreeHost(h->p); h->p = nullptr; h->cap = 0;
            CUDA_TRY(cudaHostAlloc((void**)&h->p, cap * sizeof(uint32_t), cudaHostAllocDefault));
            h->cap = cap;
        }
    }
    if (!h) {
        Context::HostList b;
        b.cap = cap;
        CUDA_TRY(cudaEventCreateWithFlags(&b.copied, cudaEventDisableTiming));
        if (cudaError_t e = cudaHostAlloc((void**)&b.p, b.cap * sizeof(uint32_t), cudaHostAllocDefault)) { cudaEventDestroy(b.copied); CUDA_TRY(e); }
        c->lists.push_back(b);
        h = &c->lists.back();
    }
    memcpy(h->p, src, n * sizeof(uint32_t));
    CUDA_TRY(cudaMemcpyAsync(d_dst, h->p, n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaEventRecord(h->copied, st));
    return 0;
}

// The path of an update of k of N data blocks with M parity blocks of SIZE words (DESIGN 3h), in units of one product per
// 16-byte lane at full occupancy.  The direct path costs k times the lanes of update_parity_kernel's grid (32 parity rows x 32
// chunks per CTA, padding included: ceil32(M) * ceil32(s4)) plus kUpdateRowLanes per changed row, the part of a row's cost that
// does not shrink with the grid (a grid too small to fill the GPU runs each row at the latency of one CTA).  The re-encode costs
// about eight passes over the N data rows whatever k, kUpdateDirect * N * s4, plus kUpdateFixed for its launches and short-row
// passes.  The direct path also needs its k delta rows within repair's 4 GiB bound.  The three constants are fitted to where the
// measured curves cross on the H100 at the eleven points of tools/sweep.py --update.
size_t update_lanes(size_t M, size_t s4) { return (M + 31) / 32 * 32 * ((s4 + 31) / 32 * 32); }
#if defined(FECC_UPDATE_PATH)            // experiment switch (DESIGN 13): 1 = always direct, 2 = always re-encode (tools/sweep.py --update)
bool update_direct(size_t, size_t, size_t, size_t) { return FECC_UPDATE_PATH == 1; }
#else
constexpr size_t kUpdateDirect = 20, kUpdateRowLanes = 400000, kUpdateFixed = 50000000;
bool update_direct(size_t N, size_t M, size_t k, size_t size)
{
    const size_t s4 = (size + 3) / 4;
    if (k * s4 * 16 > kMaxRepairBytes) return false;
    return k * (update_lanes(M, s4) + kUpdateRowLanes) <= kUpdateDirect * N * s4 + kUpdateFixed;
}
#endif

// The update of one stripe (DESIGN 3h), on the repair workspace: either the k delta rows (direct) or N rows of one column chunk
// (re-encode), from the start of the buffer so that every row keeps the allocation's alignment, then the k indices.  Direct:
// delta, then the parity update.  Re-encode: the new rows in place, then per column chunk repair's load with no row lost, the
// encode of api.cu, and the store of all M parity rows.
int update(Context* c, uint32_t* data, size_t dpitch, size_t N, uint32_t* parity, size_t ppitch, size_t M, const uint32_t* changed, size_t k,
           const uint32_t* nw, size_t npitch, size_t size, cudaStream_t st)
{
    const bool direct = update_direct(N, M, k, size);
    const size_t s4 = (size + 3) / 4, w = direct ? 0 : repair_chunk_words(N, M, size), rows_words = direct ? k * s4 * 4 : N * w;
    const uint4* T = nullptr;
    if (direct) { if (int rc = update_table(c, N, st, &T)) return rc; }
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire((rows_words + k) * sizeof(uint32_t)));
    uint32_t *x = ws.ptr(), *idx = x + rows_words;
    if (int rc = upload_list(c, changed, k, idx, st)) return rc;
    CUDA_TRY(launch_update_delta(data, dpitch, nw, npitch, direct ? (uint4*)x : nullptr, idx, k, size, c->num_sms, st)); g_launches++;
    if (direct) {
        CUDA_TRY(launch_update_parity(parity, ppitch, M, (const uint4*)x, idx, k, T, N, size, st)); g_launches++;
        return 0;
    }
    for (size_t c0 = 0; c0 < size; c0 += w) {
        const size_t cols = size - c0 < w ? size - c0 : w;
        CUDA_TRY(launch_repair_load(N, nullptr, data, dpitch, c0, x, w, cols, c->num_sms, st)); g_launches++;
        if (int rc = encode(c, x, N, M, cols, w, st)) return rc;
        CUDA_TRY(launch_repair_syndrome(M, nullptr, parity, ppitch, c0, size, x, w, cols, c->num_sms, st)); g_launches++;
    }
    return 0;
}

// The scrub of one stripe (DESIGN 3i) on the repair workspace: N + M single-column rows of 4 words (the two folds in words 0
// and 1), then four flag words {syndrome nonzero, check failed, data roots, parity roots} and the two root lists of `cap` words.
// Fold, reduce, encode, syndromes, inverse order-M transform; one sync for the flag and S^_0 .. S^_(2 max_bad - 1) of fold 0;
// Berlekamp-Massey on the host; then C's order-M transform (parity roots), the product with s, the inverse transform and the
// check of [L, M), and the order-N transform of C_k rho^-k (data roots); a second sync for the flags and the lists.  The caller's
// outputs are written only once every runtime call has succeeded, so an error return leaves them as they were.
constexpr size_t kMaxScrubBad = FASTECC_B200_SCRUB_MAX_BAD;
int scrub(Context* c, const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, size_t size, size_t max_bad,
          uint64_t seed, cudaStream_t st, int* status, uint32_t* bad_data, size_t* n_bad_data, uint32_t* bad_parity, size_t* n_bad_parity)
{
    const size_t rows = N + M, cap = max_bad ? max_bad : 1;
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire((rows * 4 + 4 + 2 * cap) * sizeof(uint32_t)));
    uint32_t *x = ws.ptr(), *flags = x + rows * 4, *list_d = flags + 4, *list_p = list_d + cap;
    CUDA_TRY(cudaMemsetAsync(x, 0, (rows * 4 + 4) * sizeof(uint32_t), st));
    CUDA_TRY(launch_scrub_fold(data, dpitch, N, parity, ppitch, M, size, seed, x, c->num_sms, st)); g_launches++;
    CUDA_TRY(launch_scrub_reduce(x, rows, st)); g_launches++;
    TRY_RC(encode(c, x, N, M, 2, 4, st));
    CUDA_TRY(launch_scrub_syndrome(x, N, M, flags, st)); g_launches++;
    if (max_bad) TRY_RC(ntt(c, x, M, 2, 4, true, st));                         // max_bad >= 1: M >= 2
    uint32_t h[4];
    std::vector<uint32_t> S(2 * max_bad);
    CUDA_TRY(cudaMemcpyAsync(h, flags, sizeof h, cudaMemcpyDeviceToHost, st));
    if (max_bad) CUDA_TRY(cudaMemcpy2DAsync(S.data(), 4, x, 16, 4, S.size(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    auto result = [&](int s) { *status = s; *n_bad_data = *n_bad_parity = 0; return 0; };
    if (!h[0]) return result(FASTECC_B200_SCRUB_CLEAN);
    if (!max_bad) return result(FASTECC_B200_SCRUB_DETECTED);
    std::vector<uint32_t> C;
    const size_t L = berlekamp_massey(S, C);
    if (L > max_bad || C.size() != L + 1) return result(FASTECC_B200_SCRUB_DETECTED);
    // the parity points zeta^j: C(zeta^j), then M * (C * S^ mod z^M - 1) = INTT_M(C(zeta^j) * s_j) in both folds
    CUDA_TRY(cudaMemsetAsync(x, 0, M * 16, st));
    CUDA_TRY(cudaMemcpy2DAsync(x, 16, C.data(), 4, 4, L + 1, cudaMemcpyHostToDevice, st));
    TRY_RC(ntt(c, x, M, 2, 4, false, st));
    CUDA_TRY(launch_scrub_roots(x, M, list_p, flags + 3, cap, st)); g_launches++;
    CUDA_TRY(launch_scrub_product(x, N, M, st)); g_launches++;
    TRY_RC(ntt(c, x, M, 2, 4, true, st));
    CUDA_TRY(launch_scrub_check(x, L, M, flags + 1, st)); g_launches++;
    // the data points omega^i: C(rho^-1 omega^i) = NTT_N(C_k rho^-k)[i]
    const uint32_t rho_inv = gf::inv(gf::root((uint32_t)(2 * N)));
    std::vector<uint32_t> T(L + 1);
    for (size_t k = 0, r = 1; k <= L; ++k, r = gf::mulmod((uint32_t)r, rho_inv)) T[k] = gf::mulmod(C[k], (uint32_t)r);
    CUDA_TRY(cudaMemsetAsync(x, 0, N * 16, st));
    CUDA_TRY(cudaMemcpy2DAsync(x, 16, T.data(), 4, 4, L + 1, cudaMemcpyHostToDevice, st));
    TRY_RC(ntt(c, x, N, 2, 4, false, st));                                     // N >= M >= 2
    CUDA_TRY(launch_scrub_roots(x, N, list_d, flags + 2, cap, st)); g_launches++;
    std::vector<uint32_t> ld(cap), lp(cap);
    CUDA_TRY(cudaMemcpyAsync(h, flags, sizeof h, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ld.data(), list_d, cap * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(lp.data(), list_p, cap * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (h[1] || (size_t)h[2] + h[3] != L) return result(FASTECC_B200_SCRUB_DETECTED);   // C fails the check, or a root is no stripe point
    std::sort(ld.begin(), ld.begin() + h[2]);
    std::sort(lp.begin(), lp.begin() + h[3]);
    std::copy(ld.begin(), ld.begin() + h[2], bad_data);
    std::copy(lp.begin(), lp.begin() + h[3], bad_parity);
    *n_bad_data = h[2]; *n_bad_parity = h[3];
    *status = FASTECC_B200_SCRUB_LOCATED;
    return 0;
}

// The scrub of a stripe with the f = |E| >= 1 blocks of the pattern R known lost (DESIGN 3j), on scrub()'s workspace and with its
// two syncs: the fold of the surviving rows only, reduce, encode, u = s * cs (zero on the lost parity rows), inverse order-M
// transform and the check of [f, M) (flag 0: not clean); Berlekamp-Massey on U^_f .. U^_(f + 2 max_bad - 1) of fold 0; C's order-M
// transform, its roots at the surviving parity points, the product with u, the inverse transform and the check of [f + L, M); the
// order-N transform of C_k rho^-k and its roots at the surviving data points.  The outputs are written as scrub() writes them.
int scrub_degraded(Context* c, const fastecc_b200_repair* R, const uint32_t* data, size_t dpitch, const uint32_t* parity, size_t ppitch, size_t size,
                   size_t max_bad, uint64_t seed, cudaStream_t st, int* status, uint32_t* bad_data, size_t* n_bad_data, uint32_t* bad_parity,
                   size_t* n_bad_parity)
{
    const size_t N = R->N, M = R->M, f = R->ned + R->nep, rows = N + M, cap = max_bad ? max_bad : 1;
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire((rows * 4 + 4 + 2 * cap) * sizeof(uint32_t)));
    uint32_t *x = ws.ptr(), *flags = x + rows * 4, *list_d = flags + 4, *list_p = list_d + cap;
    CUDA_TRY(cudaMemsetAsync(x, 0, (rows * 4 + 4) * sizeof(uint32_t), st));
    CUDA_TRY(launch_degraded_fold(data, dpitch, N, parity, ppitch, M, size, seed, R->d_lost, R->d_cs, x, c->num_sms, st)); g_launches++;
    CUDA_TRY(launch_scrub_reduce(x, rows, st)); g_launches++;
    TRY_RC(encode(c, x, N, M, 2, 4, st));
    CUDA_TRY(launch_degraded_syndrome(x, N, M, R->d_cs, st)); g_launches++;
    TRY_RC(ntt(c, x, M, 2, 4, true, st));                                      // 1 <= f < M: M >= 2
    CUDA_TRY(launch_scrub_check(x, f, M, flags, st)); g_launches++;
    uint32_t h[4];
    std::vector<uint32_t> S(2 * max_bad);
    CUDA_TRY(cudaMemcpyAsync(h, flags, sizeof h, cudaMemcpyDeviceToHost, st));
    if (max_bad) CUDA_TRY(cudaMemcpy2DAsync(S.data(), 4, x + f * 4, 16, 4, S.size(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    auto result = [&](int s) { *status = s; *n_bad_data = *n_bad_parity = 0; return 0; };
    if (!h[0]) return result(FASTECC_B200_SCRUB_CLEAN);
    if (!max_bad) return result(FASTECC_B200_SCRUB_DETECTED);
    std::vector<uint32_t> C;
    const size_t L = berlekamp_massey(S, C);
    if (L > max_bad || C.size() != L + 1) return result(FASTECC_B200_SCRUB_DETECTED);
    // the parity points zeta^j: C(zeta^j), then INTT_M(C(zeta^j) * u_j) in both folds
    CUDA_TRY(cudaMemsetAsync(x, 0, M * 16, st));
    CUDA_TRY(cudaMemcpy2DAsync(x, 16, C.data(), 4, 4, L + 1, cudaMemcpyHostToDevice, st));
    TRY_RC(ntt(c, x, M, 2, 4, false, st));
    CUDA_TRY(launch_degraded_roots(x, M, nullptr, R->d_cs, list_p, flags + 3, cap, st)); g_launches++;
    CUDA_TRY(launch_scrub_product(x, N, M, st)); g_launches++;
    TRY_RC(ntt(c, x, M, 2, 4, true, st));
    CUDA_TRY(launch_scrub_check(x, f + L, M, flags + 1, st)); g_launches++;
    // the data points omega^i: C(rho^-1 omega^i) = NTT_N(C_k rho^-k)[i]
    const uint32_t rho_inv = gf::inv(gf::root((uint32_t)(2 * N)));
    std::vector<uint32_t> T(L + 1);
    for (size_t k = 0, r = 1; k <= L; ++k, r = gf::mulmod((uint32_t)r, rho_inv)) T[k] = gf::mulmod(C[k], (uint32_t)r);
    CUDA_TRY(cudaMemsetAsync(x, 0, N * 16, st));
    CUDA_TRY(cudaMemcpy2DAsync(x, 16, T.data(), 4, 4, L + 1, cudaMemcpyHostToDevice, st));
    TRY_RC(ntt(c, x, N, 2, 4, false, st));                                     // N >= M >= 2
    CUDA_TRY(launch_degraded_roots(x, N, R->d_lost, nullptr, list_d, flags + 2, cap, st)); g_launches++;
    std::vector<uint32_t> ld(cap), lp(cap);
    CUDA_TRY(cudaMemcpyAsync(h, flags, sizeof h, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ld.data(), list_d, cap * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(lp.data(), list_p, cap * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (h[1] || (size_t)h[2] + h[3] != L) return result(FASTECC_B200_SCRUB_DETECTED);   // C fails the check, or a root is no surviving point
    std::sort(ld.begin(), ld.begin() + h[2]);
    std::sort(lp.begin(), lp.begin() + h[3]);
    std::copy(ld.begin(), ld.begin() + h[2], bad_data);
    std::copy(lp.begin(), lp.begin() + h[3], bad_parity);
    *n_bad_data = h[2]; *n_bad_parity = h[3];
    *status = FASTECC_B200_SCRUB_LOCATED;
    return 0;
}

// x[i] = -2 / x[i] mod P for every i (all nonzero), by one batch inversion.
void neg2_over(std::vector<uint32_t>& x)
{
    using gf::mulmod;
    std::vector<uint32_t> pre(x.size() + 1, 1u);
    for (size_t i = 0; i < x.size(); ++i) pre[i + 1] = mulmod(pre[i], x[i]);
    uint32_t inv = gf::inv(pre[x.size()]);
    for (size_t i = x.size(); i-- > 0;) {
        const uint32_t t = mulmod(inv, pre[i]);
        inv = mulmod(inv, x[i]);
        x[i] = mulmod(gf::P - 2, t);
    }
}

// The N entries of fastecc_b200_rs_update's table as plain words: T[t] = -2 / (N (rho^(2t+1) - 1)), rho = GF_Root(2N), equal to
// update_table_kernel's canonical entries.
std::vector<uint32_t> update_entries(size_t N)
{
    const uint32_t rho = gf::root((uint32_t)(2 * N)), n = (uint32_t)(N % gf::P);
    std::vector<uint32_t> T(N);
    for (size_t t = 0; t < N; ++t) T[t] = gf::mulmod(n, gf::sub(gf::powmod(rho, 2 * t + 1), 1u));
    neg2_over(T);
    return T;
}

// J of a degraded read (DESIGN 3k): the a lowest-numbered parity blocks not in lost_p (ascending, nlp of them, a + nlp <= M).
std::vector<uint32_t> parity_rows_J(size_t a, const uint32_t* lost_p, size_t nlp)
{
    std::vector<uint32_t> J;
    for (uint32_t j = 0, q = 0; J.size() < a; ++j) {
        while (q < nlp && lost_p[q] < j) ++q;
        if (q == nlp || lost_p[q] != j) J.push_back(j);
    }
    return J;
}

// The combination of a degraded read (DESIGN 3k), n_out x a plain words, row q for output q.  pos = J (a parity blocks) then the
// wanted parity blocks; E = the a lost data blocks.  T(j, e) = T[(D j - e) mod N] = -2 / (N (y_j z_e - 1)), y_j = rho^(2 D j + 1),
// z_e = rho^-2e, rho = GF_Root(2N), equals update_table_kernel's canonical entry (one batch inversion for all of them).  A = T(J, E)
// is a Cauchy matrix up to diagonal scalings (the points y_j and z_e^-1 are distinct), so Gauss-Jordan always finds a pivot.
// Wanted data block E[k]: row k of A^-1.  Wanted parity block j: T(j, E) A^-1.
std::vector<uint32_t> reconstruct_combination(size_t N, size_t D, const std::vector<uint32_t>& pos, const uint32_t* E, size_t a,
                                              const uint32_t* want_d, size_t nwd, size_t nwp)
{
    using gf::mulmod;
    const size_t nk = pos.size();
    const uint32_t rho = gf::root((uint32_t)(2 * N)), n = (uint32_t)(N % gf::P);
    std::vector<uint32_t> z(a), Tv(nk * a);
    for (size_t e = 0; e < a; ++e) z[e] = gf::powmod(rho, (2 * N - 2 * (uint64_t)E[e]) % (2 * N));
    for (size_t k = 0; k < nk; ++k) {
        const uint32_t y = gf::powmod(rho, 2 * D * (uint64_t)pos[k] + 1);
        for (size_t e = 0; e < a; ++e) Tv[k * a + e] = mulmod(n, gf::sub(mulmod(y, z[e]), 1u));
    }
    neg2_over(Tv);
    std::vector<uint32_t> A(Tv.begin(), Tv.begin() + a * a), X(a * a, 0u);  // [A | X], X from I to A^-1
    for (size_t i = 0; i < a; ++i) X[i * a + i] = 1;
    for (size_t col = 0; col < a; ++col) {
        size_t p = col;
        while (!A[p * a + col]) ++p;
        for (size_t j = 0; j < a; ++j) { std::swap(A[p * a + j], A[col * a + j]); std::swap(X[p * a + j], X[col * a + j]); }
        const uint32_t f = gf::inv(A[col * a + col]);
        for (size_t j = 0; j < a; ++j) { A[col * a + j] = mulmod(A[col * a + j], f); X[col * a + j] = mulmod(X[col * a + j], f); }
        for (size_t r = 0; r < a; ++r) {
            const uint32_t m = A[r * a + col];
            if (r == col || !m) continue;
            for (size_t j = 0; j < a; ++j) {
                A[r * a + j] = gf::sub(A[r * a + j], mulmod(m, A[col * a + j]));
                X[r * a + j] = gf::sub(X[r * a + j], mulmod(m, X[col * a + j]));
            }
        }
    }
    std::vector<uint32_t> B((nwd + nwp) * a);
    for (size_t q = 0, k = 0; q < nwd; ++q) {
        while (E[k] != want_d[q]) ++k;
        for (size_t j = 0; j < a; ++j) B[q * a + j] = X[k * a + j];
    }
    for (size_t m = 0; m < nwp; ++m)
        for (size_t j = 0; j < a; ++j) {
            uint64_t s = 0;
            for (size_t k = 0; k < a; ++k) s += mulmod(Tv[(a + m) * a + k], X[k * a + j]);
            B[(nwd + m) * a + j] = (uint32_t)(s % gf::P);
        }
    return B;
}

// Plain words as the Barrett triples {w, whi, wlo, 0} that gf::mul takes.
std::vector<uint32_t> barrett_triples(const std::vector<uint32_t>& w)
{
    std::vector<uint32_t> t(w.size() * 4);
    for (size_t i = 0; i < w.size(); ++i) {
        const gf::Tw x = gf::make_tw(w[i]);
        t[4 * i] = x.w; t[4 * i + 1] = x.whi; t[4 * i + 2] = x.wlo; t[4 * i + 3] = 0;
    }
    return t;
}

// The degraded read of one stripe (DESIGN 3k) on the repair workspace: K = a + nwp rows of 64-bit sums of one column chunk, then
// the uploaded words {B, pos, lost data}.  Per chunk: zero the sums, the pass over the surviving data rows, the combination.
int reconstruct(Context* c, const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, const uint32_t* lost_d,
                size_t a, const uint32_t* lost_p, size_t nlp, const uint32_t* want_d, size_t nwd, const uint32_t* want_p, size_t nwp, uint32_t* out,
                size_t opitch, size_t size, cudaStream_t st)
{
    std::vector<uint32_t> pos = parity_rows_J(a, lost_p, nlp);       // J, then the wanted parity blocks
    pos.insert(pos.end(), want_p, want_p + nwp);
    const size_t nk = pos.size(), n_out = nwd + nwp, D = N / M;
    std::vector<uint32_t> up = barrett_triples(reconstruct_combination(N, D, pos, lost_d, a, want_d, nwd, nwp));
    const size_t nb = up.size();
    up.insert(up.end(), pos.begin(), pos.end());
    up.insert(up.end(), lost_d, lost_d + a);
    const size_t cap = kMaxRepairBytes / 8 / nk / 4 * 4, w = padded_pitch(size) <= cap ? padded_pitch(size) : cap;
    const uint4* T = nullptr;
    TRY_RC(update_table(c, N, st, &T));
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire(nk * w * 8 + up.size() * sizeof(uint32_t)));
    unsigned long long* sums = (unsigned long long*)ws.ptr();
    uint32_t* d_up = (uint32_t*)(sums + nk * w);
    const uint4* B = (const uint4*)d_up;
    const uint32_t *d_pos = d_up + nb, *d_lost = d_pos + nk;
    TRY_RC(upload_list(c, up.data(), up.size(), d_up, st));
    for (size_t c0 = 0; c0 < size; c0 += w) {
        const size_t cols = size - c0 < w ? size - c0 : w;
        CUDA_TRY(cudaMemsetAsync(sums, 0, nk * ((cols + 3) / 4 * 4) * 8, st));
        CUDA_TRY(launch_reconstruct_sum(data + c0, dpitch, N, D, T, d_pos, nk, d_lost, a, cols, sums, c->num_sms, st)); g_launches++;
        CUDA_TRY(launch_reconstruct_combine(sums, parity + c0, ppitch, d_pos, a, B, n_out, nwd, out + c0, opitch, cols, c->num_sms, st)); g_launches++;
    }
    return 0;
}

// The block lists of a degraded read, host arrays: non-null where not empty; lost and wanted blocks ascending, distinct and below N
// or M; the wanted ones among the lost ones; at most M lost blocks in all.
int check_reconstruct_lists(size_t N, size_t M, const uint32_t* lost_data, size_t n_lost_data, const uint32_t* lost_parity, size_t n_lost_parity,
                            const uint32_t* want_data, size_t n_want_data, const uint32_t* want_parity, size_t n_want_parity, const char* who)
{
    if ((n_lost_data && !lost_data) || (n_lost_parity && !lost_parity) || (n_want_data && !want_data) || (n_want_parity && !want_parity))
        return fail(FASTECC_B200_EINVAL, "%s: null block list", who);
    if (!ascending_below(lost_data, n_lost_data, N) || !ascending_below(want_data, n_want_data, N))
        return fail(FASTECC_B200_EINVAL, "%s: lost and wanted data blocks must be ascending, distinct and below N=%zu", who, N);
    if (!ascending_below(lost_parity, n_lost_parity, M) || !ascending_below(want_parity, n_want_parity, M))
        return fail(FASTECC_B200_EINVAL, "%s: lost and wanted parity blocks must be ascending, distinct and below M=%zu", who, M);
    if (!std::includes(lost_data, lost_data + n_lost_data, want_data, want_data + n_want_data) ||
        !std::includes(lost_parity, lost_parity + n_lost_parity, want_parity, want_parity + n_want_parity))
        return fail(FASTECC_B200_EINVAL, "%s: every wanted block must be a lost one", who);
    if (n_lost_data + n_lost_parity > M)
        return fail(FASTECC_B200_EINVAL, "%s: %zu + %zu lost blocks exceed M=%zu", who, n_lost_data, n_lost_parity, M);
    return 0;
}

// The degraded read of a batch of stripes with one loss pattern (DESIGN 3m).  The combination B of 3k folded into C, n_out x N over
// the sources (the N - a surviving data rows ascending, then J): on surviving data row i, [q is parity block w] T(w, i) -
// sum_j B[q][j] T(J_j, i); on parity row J_j, B[q][j]; T(j, i) = T[(D j - i) mod N].  C as triples, then the N source rows,
// uploaded under repair's lease; one launch.
int reconstruct_batch(Context* c, const uint32_t* data, size_t dpitch, size_t dstride, size_t N, const uint32_t* parity, size_t ppitch, size_t pstride,
                      size_t M, const uint32_t* lost_d, size_t a, const uint32_t* lost_p, size_t nlp, const uint32_t* want_d, size_t nwd,
                      const uint32_t* want_p, size_t nwp, uint32_t* out, size_t opitch, size_t ostride, size_t n_stripes, size_t size, cudaStream_t st)
{
    const size_t D = N / M, n_out = nwd + nwp, nd = N - a;
    std::vector<uint32_t> pos = parity_rows_J(a, lost_p, nlp);       // J, then the wanted parity blocks
    pos.insert(pos.end(), want_p, want_p + nwp);
    const std::vector<uint32_t> B = reconstruct_combination(N, D, pos, lost_d, a, want_d, nwd, nwp), T = update_entries(N);
    std::vector<uint32_t> src;
    for (uint32_t i = 0, k = 0; i < N; ++i) {
        if (k < a && lost_d[k] == i) ++k;
        else src.push_back(i);
    }
    src.insert(src.end(), pos.begin(), pos.begin() + a);
    const auto Tji = [&](size_t j, size_t i) { return T[(D * j + N - i) % N]; };
    std::vector<uint32_t> C(n_out * N);
    for (size_t q = 0; q < n_out; ++q) {
        for (size_t s = 0; s < nd; ++s) {
            uint64_t v = q >= nwd ? Tji(want_p[q - nwd], src[s]) : 0;
            for (size_t j = 0; j < a; ++j) v += gf::P - gf::mulmod(B[q * a + j], Tji(pos[j], src[s]));
            C[q * N + s] = (uint32_t)(v % gf::P);
        }
        for (size_t j = 0; j < a; ++j) C[q * N + nd + j] = B[q * a + j];
    }
    std::vector<uint32_t> up = barrett_triples(C);
    const size_t nc = up.size();
    up.insert(up.end(), src.begin(), src.end());
    Lease ws(&c->repair, st);
    CUDA_TRY(ws.acquire(up.size() * sizeof(uint32_t)));
    uint32_t* d_up = ws.ptr();
    TRY_RC(upload_list(c, up.data(), up.size(), d_up, st));
    CUDA_TRY(launch_batch_reconstruct(data, dpitch, dstride, parity, ppitch, pstride, N, nd, (const uint4*)d_up, d_up + nc, n_out, out, opitch, ostride,
                                      n_stripes, size, c->num_sms, st)); g_launches++;
    return 0;
}

} // namespace

namespace fecc {
const uint4* context_power_table() { return g_ctx ? g_ctx->d_tw : nullptr; }
int context_num_sms() { return g_ctx ? g_ctx->num_sms : 0; }
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
    g_ctx->scratch.destroy(); g_ctx->packed.destroy(); g_ctx->mixed.destroy(); g_ctx->repair.destroy(); g_ctx->staging.release();
    for (auto& r : g_ctx->registered) cudaHostUnregister(r.first);
    for (auto& l : g_ctx->lists) { cudaFreeHost(l.p); cudaEventDestroy(l.copied); }
    for (auto& kv : g_ctx->tables) for (auto& sl : kv.second) { sl.buf.release(); if (sl.ready) cudaEventDestroy(sl.ready); }
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
{ return ntt_dev(d, N, size, pitch, inverse != 0, stream, "fastecc_b200_ntt_u32_dev"); }

int fastecc_b200_rs_encode_dev(uint32_t* d, size_t N, size_t size, size_t pitch, void* stream)
{ return encode_dev(d, N, N, size, pitch, stream, false, true, "fastecc_b200_rs_encode_dev"); }

int fastecc_b200_rs_encode_dev_timed(uint32_t* d, size_t N, size_t size, size_t pitch, void* stream, float* pass_ms, const char** pass_kernel, int* n_passes)
{
    const char* who = "fastecc_b200_rs_encode_dev_timed";
    if (!pass_ms || !n_passes || *n_passes < 1) return fail(FASTECC_B200_EINVAL, "%s: pass_ms / n_passes missing", who);
    PassTimer t;
    int rc = encode_dev(d, N, N, size, pitch, stream, false, true, who, &t);
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
    const uint32_t LN = ilog2(N), L1 = LN <= (uint32_t)kMaxLogR ? LN : split_l1(LN, true);
    if (N1) *N1 = (size_t)1 << L1;
    if (N2) *N2 = (size_t)1 << (LN - L1);
    if (fused_exchange_ok) *fused_exchange_ok = n_ranks >= 2 ? (shard_p2p_supported(N, (uint32_t)n_ranks) ? 1 : 0) | (ntt_shard_p2p_supported(N, (uint32_t)n_ranks) ? 2 : 0) : 0;
    return n_ranks < 2 || shard_supported(N, (uint32_t)n_ranks) || ntt_shard_p2p_supported(N, (uint32_t)n_ranks) ? 0 : fail(FASTECC_B200_EINVAL, "fastecc_b200_shard_geometry: N=%zu cannot be sharded over %d ranks", N, n_ranks);
}

int fastecc_b200_copy2d_async(void* dst, size_t dst_pitch_bytes, const void* src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, int to_device, void* stream)
{
    if (!ctx("fastecc_b200_copy2d_async")) return FASTECC_B200_ENOINIT;
    CUDA_TRY(cudaMemcpy2DAsync(dst, dst_pitch_bytes, src, src_pitch_bytes, width_bytes, rows, to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return 0;
}

int fastecc_b200_gf_mul_dev(const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n, void* stream)
{
    if (!ctx("fastecc_b200_gf_mul_dev")) return FASTECC_B200_ENOINIT;
    if (n && (!a || !b || !out)) return fail(FASTECC_B200_EINVAL, "fastecc_b200_gf_mul_dev: null device pointer");
    CUDA_TRY(launch_gf_mul(a, b, out, n, (cudaStream_t)stream)); g_launches++;
    return 0;
}
int fastecc_b200_gf_inv_dev(const uint32_t* a, uint32_t* out, size_t n, void* stream)
{
    if (!ctx("fastecc_b200_gf_inv_dev")) return FASTECC_B200_ENOINIT;
    if (n && (!a || !out)) return fail(FASTECC_B200_EINVAL, "fastecc_b200_gf_inv_dev: null device pointer");
    CUDA_TRY(launch_gf_inv(a, out, n, (cudaStream_t)stream)); g_launches++;
    return 0;
}
int fastecc_b200_row_scale_dev(uint32_t* d, size_t n_rows, size_t size, size_t pitch, const uint32_t* d_consts, void* stream)
{
    const char* who = "fastecc_b200_row_scale_dev";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (!d_consts) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if (int rc = check_rows(d, 1, size, pitch, true, who)) return rc;      // one row: the kernel's 32-bit chunk index runs within a row
    CUDA_TRY(launch_row_scale(d, n_rows, (uint32_t)((size + 3) / 4), (uint32_t)(pitch / 4), d_consts, c->num_sms, (cudaStream_t)stream)); g_launches++;
    return 0;
}

static int recode_args(const void* a, const void* b, size_t n_blocks, size_t W, size_t pitch, const char* who)
{
    if (!ctx(who)) return FASTECC_B200_ENOINIT;
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
{ return encode_dev(d, N, M, size, pitch, stream, false, false, "fastecc_b200_rs_encode_asym_dev"); }

int fastecc_b200_rs_encode_asym(uint32_t** data, size_t N, size_t M, size_t size)
{ return encode_host(data, N, M, size, false, "fastecc_b200_rs_encode_asym"); }

int fastecc_b200_rs_encode_shard_pass(uint32_t* d_local, size_t N, int n_ranks, int rank, size_t size, size_t pitch, int which, void* stream)
{ return shard_pass(kShard, d_local, nullptr, N, n_ranks, rank, size, pitch, 0, which, stream, "fastecc_b200_rs_encode_shard_pass"); }

int fastecc_b200_rs_encode_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank, size_t size, size_t pitch,
                                          int which, void* stream)
{ return shard_pass(kShardP2P, d_src, d_peers, N, n_ranks, rank, size, pitch, 0, which, stream, "fastecc_b200_rs_encode_shard_pass_p2p"); }

int fastecc_b200_ntt_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank, size_t size, size_t pitch,
                                    int inverse, int which, void* stream)
{ return shard_pass(kNttShardP2P, d_src, d_peers, N, n_ranks, rank, size, pitch, inverse, which, stream, "fastecc_b200_ntt_shard_pass_p2p"); }

int fastecc_b200_shard_barrier(uint32_t* const* d_flag_peers, int n_ranks, int rank, uint32_t epoch, void* stream)
{
    const char* who = "fastecc_b200_shard_barrier";
    if (!ctx(who)) return FASTECC_B200_ENOINIT;
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
    if (!ctx("fastecc_b200_dev_alloc")) return nullptr;
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { clear_cuda_error(); fail(FASTECC_B200_ENOMEM, "fastecc_b200_dev_alloc: cudaMalloc(%zu) failed", bytes); return nullptr; }
    return p;
}
void fastecc_b200_dev_free(void* p) { if (p) cudaFree(p); }
int fastecc_b200_ipc_export(void* d_ptr, void* handle64)
{
    if (!ctx("fastecc_b200_ipc_export")) return FASTECC_B200_ENOINIT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    CUDA_TRY(cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle64, &h, 64);
    return 0;
}
int fastecc_b200_ipc_open(const void* handle64, void** d_ptr)
{
    if (!ctx("fastecc_b200_ipc_open")) return FASTECC_B200_ENOINIT;
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
{ return ntt_host(data, N, size, inverse != 0, "fastecc_b200_ntt_u32"); }

int fastecc_b200_rs_encode(uint32_t** data, size_t N, size_t size)
{ return encode_host(data, N, N, size, false, "fastecc_b200_rs_encode"); }

int fastecc_b200_rs_encode_mixed(uint32_t** data, size_t N, size_t size)
{ return encode_host(data, N, N, size, true, "fastecc_b200_rs_encode_mixed"); }

int fastecc_b200_rs_encode_mixed_dev(uint32_t* d, size_t N, size_t size, size_t pitch, void* stream)
{ return encode_dev(d, N, N, size, pitch, stream, true, true, "fastecc_b200_rs_encode_mixed_dev"); }

int fastecc_b200_rs_encode_asym_mixed_dev(uint32_t* d, size_t N, size_t M, size_t size, size_t pitch, void* stream)
{ return encode_dev(d, N, M, size, pitch, stream, true, true, "fastecc_b200_rs_encode_asym_mixed_dev"); }

int fastecc_b200_rs_encode_asym_mixed(uint32_t** data, size_t N, size_t M, size_t size)
{ return encode_host(data, N, M, size, true, "fastecc_b200_rs_encode_asym_mixed"); }

int fastecc_b200_rs_repair(const fastecc_b200_repair* R, uint32_t* d_data, size_t data_pitch, uint32_t* d_parity, size_t parity_pitch, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_repair";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (!R) return fail(FASTECC_B200_EINVAL, "%s: null pattern", who);
    if (int rc = check_rows(d_data, R->N, size, data_pitch, true, who)) return rc;
    if (int rc = check_rows(d_parity, R->M, size, parity_pitch, true, who)) return rc;
    if (rows_overlap(d_data, R->N, data_pitch, d_parity, R->M, parity_pitch, size)) return fail(FASTECC_B200_EINVAL, "%s: the data and parity buffers overlap", who);
    if (R->ned + R->nep == 0) return 0;
    return repair(c, R, d_data, data_pitch, d_parity, parity_pitch, size, (cudaStream_t)stream);
}

int fastecc_b200_rs_update(uint32_t* d_data, size_t data_pitch, size_t N, uint32_t* d_parity, size_t parity_pitch, size_t M,
                           const uint32_t* changed, size_t n_changed, const uint32_t* d_new, size_t new_pitch, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_update";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (int rc = check_rows(d_data, N, size, data_pitch, true, who)) return rc;
    if (int rc = check_rows(d_parity, M, size, parity_pitch, true, who)) return rc;
    if (n_changed && !changed) return fail(FASTECC_B200_EINVAL, "%s: null list of changed blocks", who);
    if (!ascending_below(changed, n_changed, N)) return fail(FASTECC_B200_EINVAL, "%s: changed data blocks must be ascending, distinct and below N=%zu", who, N);
    if (rows_overlap(d_data, N, data_pitch, d_parity, M, parity_pitch, size)) return fail(FASTECC_B200_EINVAL, "%s: the data and parity buffers overlap", who);
    if (!n_changed) return 0;
    if (int rc = check_rows(d_new, n_changed, size, new_pitch, true, who)) return rc;
    if (rows_overlap(d_new, n_changed, new_pitch, d_data, N, data_pitch, size) || rows_overlap(d_new, n_changed, new_pitch, d_parity, M, parity_pitch, size))
        return fail(FASTECC_B200_EINVAL, "%s: the new blocks overlap the data or the parity buffer", who);
    return update(c, d_data, data_pitch, N, d_parity, parity_pitch, M, changed, n_changed, d_new, new_pitch, size, (cudaStream_t)stream);
}

int fastecc_b200_rs_scrub(const uint32_t* d_data, size_t data_pitch, size_t N, const uint32_t* d_parity, size_t parity_pitch, size_t M, size_t size,
                          size_t max_bad, uint64_t seed, void* stream, int* status, uint32_t* bad_data, size_t* n_bad_data, uint32_t* bad_parity,
                          size_t* n_bad_parity)
{
    const char* who = "fastecc_b200_rs_scrub";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (!status || !n_bad_data || !n_bad_parity) return fail(FASTECC_B200_EINVAL, "%s: null status or count output", who);
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (int rc = check_rows(d_data, N, size, data_pitch, true, who)) return rc;
    if (int rc = check_rows(d_parity, M, size, parity_pitch, true, who)) return rc;
    if (max_bad > M / 2 || max_bad > kMaxScrubBad)
        return fail(FASTECC_B200_EINVAL, "%s: max_bad=%zu must be at most min(M / 2, %zu) = %zu", who, max_bad, kMaxScrubBad, M / 2 < kMaxScrubBad ? M / 2 : kMaxScrubBad);
    if (max_bad && (!bad_data || !bad_parity)) return fail(FASTECC_B200_EINVAL, "%s: null list of bad blocks", who);
    return scrub(c, d_data, data_pitch, N, d_parity, parity_pitch, M, size, max_bad, seed, (cudaStream_t)stream, status, bad_data, n_bad_data, bad_parity,
                 n_bad_parity);
}

int fastecc_b200_rs_scrub_degraded(const fastecc_b200_repair* R, const uint32_t* d_data, size_t data_pitch, const uint32_t* d_parity, size_t parity_pitch,
                                   size_t size, size_t max_bad, uint64_t seed, void* stream, int* status, uint32_t* bad_data, size_t* n_bad_data,
                                   uint32_t* bad_parity, size_t* n_bad_parity)
{
    const char* who = "fastecc_b200_rs_scrub_degraded";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (!R) return fail(FASTECC_B200_EINVAL, "%s: null pattern", who);
    if (!status || !n_bad_data || !n_bad_parity) return fail(FASTECC_B200_EINVAL, "%s: null status or count output", who);
    const size_t N = R->N, M = R->M, f = R->ned + R->nep;
    if (f == M) return fail(FASTECC_B200_EINVAL, "%s: the pattern loses f = M = %zu blocks; no check symbol is left", who, M);
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (int rc = check_rows(d_data, N, size, data_pitch, true, who)) return rc;
    if (int rc = check_rows(d_parity, M, size, parity_pitch, true, who)) return rc;
    const size_t top = (M - f) / 2 < kMaxScrubBad ? (M - f) / 2 : kMaxScrubBad;
    if (max_bad > top) return fail(FASTECC_B200_EINVAL, "%s: max_bad=%zu must be at most min((M - f) / 2, %zu) = %zu (M=%zu, f=%zu lost)", who, max_bad, kMaxScrubBad, top, M, f);
    if (max_bad && (!bad_data || !bad_parity)) return fail(FASTECC_B200_EINVAL, "%s: null list of bad blocks", who);
    if (!f)
        return scrub(c, d_data, data_pitch, N, d_parity, parity_pitch, M, size, max_bad, seed, (cudaStream_t)stream, status, bad_data, n_bad_data, bad_parity,
                     n_bad_parity);
    return scrub_degraded(c, R, d_data, data_pitch, d_parity, parity_pitch, size, max_bad, seed, (cudaStream_t)stream, status, bad_data, n_bad_data,
                          bad_parity, n_bad_parity);
}

int fastecc_b200_rs_reconstruct(const uint32_t* d_data, size_t data_pitch, size_t N, const uint32_t* d_parity, size_t parity_pitch, size_t M,
                                const uint32_t* lost_data, size_t n_lost_data, const uint32_t* lost_parity, size_t n_lost_parity,
                                const uint32_t* want_data, size_t n_want_data, const uint32_t* want_parity, size_t n_want_parity,
                                uint32_t* d_out, size_t out_pitch, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_reconstruct";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (int rc = check_rows(d_data, N, size, data_pitch, true, who)) return rc;
    if (int rc = check_rows(d_parity, M, size, parity_pitch, true, who)) return rc;
    if (int rc = check_reconstruct_lists(N, M, lost_data, n_lost_data, lost_parity, n_lost_parity, want_data, n_want_data, want_parity, n_want_parity,
                                         who))
        return rc;
    if (n_lost_data + n_want_parity > FASTECC_B200_RECONSTRUCT_MAX)
        return fail(FASTECC_B200_EINVAL, "%s: n_lost_data + n_want_parity = %zu exceeds FASTECC_B200_RECONSTRUCT_MAX = %d; fastecc_b200_rs_repair rebuilds up "
                    "to M lost blocks", who, n_lost_data + n_want_parity, FASTECC_B200_RECONSTRUCT_MAX);
    const size_t n_out = n_want_data + n_want_parity;
    if (!n_out) return 0;
    if (int rc = check_rows(d_out, n_out, size, out_pitch, true, who)) return rc;
    if (rows_overlap(d_out, n_out, out_pitch, d_data, N, data_pitch, size) || rows_overlap(d_out, n_out, out_pitch, d_parity, M, parity_pitch, size))
        return fail(FASTECC_B200_EINVAL, "%s: the output overlaps the data or the parity buffer", who);
    return reconstruct(c, d_data, data_pitch, N, d_parity, parity_pitch, M, lost_data, n_lost_data, lost_parity, n_lost_parity, want_data, n_want_data,
                       want_parity, n_want_parity, d_out, out_pitch, size, (cudaStream_t)stream);
}

int fastecc_b200_rs_encode_batch(const uint32_t* d_data, size_t data_pitch, size_t data_stride, size_t N, uint32_t* d_parity, size_t parity_pitch,
                                 size_t parity_stride, size_t M, size_t n_stripes, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_encode_batch";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (N > FASTECC_B200_BATCH_MAX_N)
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu exceeds FASTECC_B200_BATCH_MAX_N = %d; encode larger stripes one at a time with "
                    "fastecc_b200_rs_encode_asym_mixed_dev", who, N, FASTECC_B200_BATCH_MAX_N);
    if (data_pitch < size || parity_pitch < size)
        return fail(FASTECC_B200_EINVAL, "%s: needs SIZE_words (%zu) <= data_pitch_words (%zu) and parity_pitch_words (%zu)", who, size, data_pitch, parity_pitch);
    if ((uintptr_t)d_data % 16 || (uintptr_t)d_parity % 16 || data_pitch % 4 || parity_pitch % 4 || data_stride % 4 || parity_stride % 4)
        return fail(FASTECC_B200_EINVAL, "%s: needs 16-byte aligned buffers and pitches and stripe strides that are multiples of 4 words", who);
    if (!n_stripes) return 0;                                              // an empty batch reads and writes nothing: any pointers do
    if (!d_data || !d_parity) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if ((unsigned long long)n_stripes * ((size + 3) / 4) >= (1ull << 36))
        return fail(FASTECC_B200_EINVAL, "%s: %zu stripes of %zu words exceed 2^36 16-byte chunks", who, n_stripes, size);
    const BatchRows d{(uintptr_t)d_data / 4, data_pitch, data_stride, N}, p{(uintptr_t)d_parity / 4, parity_pitch, parity_stride, M};
    if (!batch_layout_disjoint(d, p, n_stripes, size))
        return fail(FASTECC_B200_EINVAL, "%s: parity rows may overlap each other or the data; accepted layouts: separate data and parity spans, each "
                    "stripe-major or block-major, or one common stripe stride holding each stripe's N + M disjoint rows", who);
    const cudaStream_t st = (cudaStream_t)stream;
    const uint4* T = nullptr;
    TRY_RC(update_table(c, N, st, &T));
    CUDA_TRY(launch_batch_encode(d_data, data_pitch, data_stride, N, d_parity, parity_pitch, parity_stride, M, n_stripes, size, T, st)); g_launches++;
    return 0;
}

int fastecc_b200_rs_reconstruct_batch(const uint32_t* d_data, size_t data_pitch, size_t data_stride, size_t N, const uint32_t* d_parity,
                                      size_t parity_pitch, size_t parity_stride, size_t M, const uint32_t* lost_data, size_t n_lost_data,
                                      const uint32_t* lost_parity, size_t n_lost_parity, const uint32_t* want_data, size_t n_want_data,
                                      const uint32_t* want_parity, size_t n_want_parity, uint32_t* d_out, size_t out_pitch, size_t out_stride,
                                      size_t n_stripes, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_reconstruct_batch";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (N > FASTECC_B200_BATCH_MAX_N)
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu exceeds FASTECC_B200_BATCH_MAX_N = %d; read larger stripes one at a time with "
                    "fastecc_b200_rs_reconstruct", who, N, FASTECC_B200_BATCH_MAX_N);
    if (data_pitch < size || parity_pitch < size || out_pitch < size)
        return fail(FASTECC_B200_EINVAL, "%s: needs SIZE_words (%zu) <= data_pitch_words (%zu), parity_pitch_words (%zu) and out_pitch_words (%zu)", who, size,
                    data_pitch, parity_pitch, out_pitch);
    if ((uintptr_t)d_data % 16 || (uintptr_t)d_parity % 16 || (uintptr_t)d_out % 16 || data_pitch % 4 || parity_pitch % 4 || out_pitch % 4 ||
        data_stride % 4 || parity_stride % 4 || out_stride % 4)
        return fail(FASTECC_B200_EINVAL, "%s: needs 16-byte aligned buffers and pitches and stripe strides that are multiples of 4 words", who);
    if (int rc = check_reconstruct_lists(N, M, lost_data, n_lost_data, lost_parity, n_lost_parity, want_data, n_want_data, want_parity, n_want_parity,
                                         who))
        return rc;
    const size_t n_out = n_want_data + n_want_parity;
    if (!n_stripes || !n_out) return 0;                                   // nothing to read or write: any pointers do
    if (!d_data || !d_parity || !d_out) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if ((unsigned long long)n_stripes * ((size + 3) / 4) >= (1ull << 36))
        return fail(FASTECC_B200_EINVAL, "%s: %zu stripes of %zu words exceed 2^36 16-byte chunks", who, n_stripes, size);
    const BatchRows d{(uintptr_t)d_data / 4, data_pitch, data_stride, N}, p{(uintptr_t)d_parity / 4, parity_pitch, parity_stride, M};
    const BatchRows o{(uintptr_t)d_out / 4, out_pitch, out_stride, n_out};
    if (!batch_layout_disjoint(d, o, n_stripes, size) || !batch_layout_disjoint(p, o, n_stripes, size))
        return fail(FASTECC_B200_EINVAL, "%s: output rows may overlap each other, the data or the parity; accepted layouts: an output span apart from "
                    "each side's span, stripe-major or block-major, or one common stripe stride holding each stripe's rows disjoint", who);
    return reconstruct_batch(c, d_data, data_pitch, data_stride, N, d_parity, parity_pitch, parity_stride, M, lost_data, n_lost_data, lost_parity,
                             n_lost_parity, want_data, n_want_data, want_parity, n_want_parity, d_out, out_pitch, out_stride, n_stripes, size,
                             (cudaStream_t)stream);
}

int fastecc_b200_rs_update_batch(uint32_t* d_data, size_t data_pitch, size_t data_stride, size_t N, uint32_t* d_parity, size_t parity_pitch,
                                 size_t parity_stride, size_t M, const uint32_t* changed, size_t n_changed, const uint32_t* d_new, size_t new_pitch,
                                 size_t new_stride, size_t n_stripes, size_t size, void* stream)
{
    const char* who = "fastecc_b200_rs_update_batch";
    Context* c = ctx(who);
    if (!c) return FASTECC_B200_ENOINIT;
    if (int rc = check_order(N, M, size, padded_pitch(size), FASTECC_B200_MAX_LOG_N_ENCODE, true, who)) return rc;
    if (N > FASTECC_B200_BATCH_MAX_N)
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu exceeds FASTECC_B200_BATCH_MAX_N = %d; update larger stripes one at a time with "
                    "fastecc_b200_rs_update", who, N, FASTECC_B200_BATCH_MAX_N);
    if (data_pitch < size || parity_pitch < size || new_pitch < size)
        return fail(FASTECC_B200_EINVAL, "%s: needs SIZE_words (%zu) <= data_pitch_words (%zu), parity_pitch_words (%zu) and new_pitch_words (%zu)", who, size,
                    data_pitch, parity_pitch, new_pitch);
    if ((uintptr_t)d_data % 16 || (uintptr_t)d_parity % 16 || (uintptr_t)d_new % 16 || data_pitch % 4 || parity_pitch % 4 || new_pitch % 4 ||
        data_stride % 4 || parity_stride % 4 || new_stride % 4)
        return fail(FASTECC_B200_EINVAL, "%s: needs 16-byte aligned buffers and pitches and stripe strides that are multiples of 4 words", who);
    if (n_changed && !changed) return fail(FASTECC_B200_EINVAL, "%s: null list of changed blocks", who);
    if (!ascending_below(changed, n_changed, N)) return fail(FASTECC_B200_EINVAL, "%s: changed data blocks must be ascending, distinct and below N=%zu", who, N);
    if (!n_stripes || !n_changed) return 0;                                // nothing to read or write: any pointers do
    if (!d_data || !d_parity || !d_new) return fail(FASTECC_B200_EINVAL, "%s: null device pointer", who);
    if ((unsigned long long)n_stripes * ((size + 3) / 4) >= (1ull << 36))
        return fail(FASTECC_B200_EINVAL, "%s: %zu stripes of %zu words exceed 2^36 16-byte chunks", who, n_stripes, size);
    const BatchRows d{(uintptr_t)d_data / 4, data_pitch, data_stride, N}, p{(uintptr_t)d_parity / 4, parity_pitch, parity_stride, M};
    const BatchRows n{(uintptr_t)d_new / 4, new_pitch, new_stride, n_changed};
    if (!batch_update_layout_disjoint(d, p, n, n_stripes, size))
        return fail(FASTECC_B200_EINVAL, "%s: the data and parity rows of all stripes must be pairwise disjoint and apart from the new rows; accepted "
                    "layouts: separate spans, each stripe-major or block-major, or one common stripe stride holding each stripe's rows disjoint", who);
    const cudaStream_t st = (cudaStream_t)stream;
    const uint4* T = nullptr;
    TRY_RC(update_table(c, N, st, &T));
    CUDA_TRY(launch_batch_update(d_data, data_pitch, data_stride, N, d_parity, parity_pitch, parity_stride, M, changed, n_changed, d_new, new_pitch,
                                 new_stride, n_stripes, size, T, c->num_sms, st)); g_launches++;
    return 0;
}

int fastecc_b200_pin_host_buffers(int enable)
{
    std::lock_guard<std::mutex> lk(g_host_mu);
    if (!ctx("fastecc_b200_pin_host_buffers")) return FASTECC_B200_ENOINIT;
    g_ctx->pin_caller = enable != 0;
    if (!enable) {                                                          // turning it off also releases what was page-locked so far
        CUDA_TRY(cudaDeviceSynchronize());
        for (auto& r : g_ctx->registered) { cudaHostUnregister(r.first); clear_cuda_error(); }
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
