// garage_ec.cu -- C ABI (include/garage_ec.h) over the sm_90a kernels in rs_kernels.cuh.
//
// Product code: no CPU fallback, nothing from oracle/.  Every entry point returns a status
// code and never throws/aborts across the boundary, mirroring the reference's
// Result<_, Error> convention (src/util/error.rs:14-82; SURVEY.md section 8(b)).
#include "../../include/garage_ec.h"

#if defined(__x86_64__)
#include <emmintrin.h>
#include <immintrin.h>
#endif
#include <cuda_runtime.h>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "rs_kernels.cuh"
#include "clay_kernels.cuh"
#include "sse_kernels.cuh"

using namespace garage_ec;

static_assert(GARAGE_EC_MAX_K == kMaxK && GARAGE_EC_MAX_M == kMaxM, "header/kernels limits differ");
static_assert(GARAGE_EC_MAX_K == GARAGE_EC_MAX_K_HOST && GARAGE_EC_MAX_M == GARAGE_EC_MAX_M_HOST,
              "header/gf256 limits differ");

namespace {

constexpr int kHostLanes = 3;  // H2D / kernel / D2H overlap across chunks

struct HostLane {
    cudaStream_t stream = nullptr;
    uint8_t *d_buf = nullptr;  // chunk of shards (sources + outputs)
    size_t d_cap = 0;
    uint8_t *d_small = nullptr;  // shard_len / present / want / status / mismatch / plan
    size_t small_cap = 0;
    cudaEvent_t done = nullptr;  // blocking-sync event (garage_ec_set_wait_mode)
    uint8_t *h_key = nullptr;    // pinned staging of SSE-C keys and nonces (zeroed once their upload completed)
    size_t h_key_cap = 0;
};
// One HOST-mode call owns one set of lanes for its duration; concurrent callers (tokio
// spawn_blocking threads, src/block/block.rs:86) get different sets, up to kMaxLaneSets.
struct LaneSet {
    HostLane lanes[kHostLanes];
};
constexpr int kMaxLaneSets = 4;

}  // namespace

struct garage_ec_ctx {
    int device = 0, k = 0, m = 0;
    int l = 0;  // LRC local groups (garage_ec_create_lrc); 0 = RS (MDS: any k shards decode)
    bool pb = false;  // piggybacked RS PB(k, m) (garage_ec_create_piggyback, DESIGN.md section 2.2)
    bool clay = false;  // Clay(k, m) (garage_ec_create_clay, DESIGN.md section 2.4): P is then the m x (k+s) base rows
    ClayGeo cg{};
    uint32_t quantum = 1;  // code_shard_len rounding: 1 (RS, LRC), 128 (PB), 16*alpha (Clay)
    uint8_t P[kMaxM * kMaxK] = {0};
    int sm_count = 0;
    size_t smem_optin = 0;
    std::mutex pool_mu;  // lane-set pool of the HOST-mode calls
    std::condition_variable pool_cv;
    std::vector<LaneSet *> free_sets;
    int n_sets = 0;
    // NUMA placement of the GPU (from sysfs): host memory for DMA should live on this node
    // stream-ordered scratch (decode plans of DEVICE-mode calls) comes from a pool of our own that KEEPS freed memory:
    // the default pool hands memory back to the driver at every synchronisation, and re-mapping it on the next call
    // cost 10-40 ms of host time at random whenever the GPU work ahead of it was short (config-5 sweep with adler8 tags)
    cudaMemPool_t pool = nullptr;
    std::atomic<int> sum_kind{GARAGE_EC_SUM_BLAKE2};  // per-shard integrity tag (garage_ec_set_sum_kind)
    int numa_node = -1;
    bool have_node_cpus = false;
    cpu_set_t node_cpus;
    int last_alloc_node = -1;                 // node the last garage_ec_host_alloc landed on (-1 unknown)
    std::atomic<long> fault_countdown{-1};
    // how a HOST-mode call waits for its lanes: 0 = cudaStreamSynchronize (the driver spins: lowest latency, one CPU
    // per waiting caller), 1 = block on an event (garage_ec_set_wait_mode)
    std::atomic<int> wait_blocking{0};
    // test hook: fail the n-th staged operation (see garage_ec_debug_fail_after)
    std::mutex misc_mu;  // timing list, last_error
    bool timing = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
    std::vector<cudaEvent_t> free_events;
    std::atomic<uint64_t> launches{0};
    std::atomic<int> batch_copy_ok{1};  // cudaMemcpyBatchAsync usable (cleared on first failure)
    char last_error[256] = {0};
};

namespace {

int set_cuda_error(garage_ec_ctx *ctx, cudaError_t e, const char *what)
{
    if (ctx) {
        std::lock_guard<std::mutex> g(ctx->misc_mu);
        snprintf(ctx->last_error, sizeof(ctx->last_error), "%s: %s", what, cudaGetErrorString(e));
    }
    (void)cudaGetLastError();  // clear sticky-less errors
    return e == cudaErrorMemoryAllocation ? GARAGE_EC_E_NOMEM : GARAGE_EC_E_CUDA;
}

// test hook (garage_ec_debug_fail_after): the n-th checked runtime call from now fails
inline bool fault_hit(garage_ec_ctx *ctx)
{
    if (!ctx || ctx->fault_countdown.load(std::memory_order_relaxed) < 0) return false;
    return ctx->fault_countdown.fetch_sub(1, std::memory_order_relaxed) == 0;
}

#define CU_TRY(ctx, expr)                                                                          \
    do {                                                                                           \
        if (fault_hit(ctx)) return set_cuda_error(ctx, cudaErrorUnknown, "injected fault at " #expr); \
        cudaError_t e__ = (expr);                                                                  \
        if (e__ != cudaSuccess) return set_cuda_error(ctx, e__, #expr);                            \
    } while (0)

// wait for everything queued on a lane (see garage_ec_ctx::wait_blocking)
inline cudaError_t lane_wait(garage_ec_ctx *ctx, HostLane &L)
{
    if (!ctx->wait_blocking.load(std::memory_order_relaxed)) return cudaStreamSynchronize(L.stream);
    cudaError_t e = cudaSuccess;
    if (!L.done) e = cudaEventCreateWithFlags(&L.done, cudaEventBlockingSync | cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(L.done, L.stream);
    if (e == cudaSuccess) e = cudaEventSynchronize(L.done);
    return e;
}

// Stream-ordered device scratch of `bytes` for the work f(scratch) queues on st, freed on st after it: from the context's
// pool (the default pool if it has none), so that DEVICE-mode calls stay capturable in a CUDA graph.  f's error first.
template <class F>
int with_stream_scratch(garage_ec_ctx *ctx, size_t bytes, cudaStream_t st, F &&f)
{
    void *scratch = nullptr;
    CU_TRY(ctx, ctx->pool ? cudaMallocFromPoolAsync(&scratch, bytes, ctx->pool, st) : cudaMallocAsync(&scratch, bytes, st));
    const int rc = f(static_cast<uint8_t *>(scratch));
    const cudaError_t e = cudaFreeAsync(scratch, st);
    if (rc) return rc;
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaFreeAsync");
    return GARAGE_EC_OK;
}

// ---- NUMA placement of the GPU ------------------------------------------------------------
// 8-GPU hosts hang 4 GPUs off each socket; pinned buffers that land on the other socket cross
// the inter-socket link on every DMA (round 1: e2e weak scaling 0.65 at 8 GPUs with unplaced
// buffers).  The node comes from sysfs, the CPU list of the node likewise; no libnuma.
#ifndef MPOL_PREFERRED
#define MPOL_DEFAULT 0
#define MPOL_PREFERRED 1
#endif
bool read_small_file(const char *path, char *buf, size_t cap)
{
    FILE *f = fopen(path, "r");
    if (!f) return false;
    const size_t n = fread(buf, 1, cap - 1, f);
    fclose(f);
    buf[n] = 0;
    return n > 0;
}
bool parse_cpulist(const char *s, cpu_set_t *out)
{
    CPU_ZERO(out);
    bool any = false;
    while (*s) {
        while (*s == ',' || isspace((unsigned char)*s)) s++;
        if (!isdigit((unsigned char)*s)) break;
        char *e;
        long a = strtol(s, &e, 10), b = a;
        if (*e == '-') b = strtol(e + 1, &e, 10);
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) {
            CPU_SET((int)c, out);
            any = true;
        }
        s = e;
    }
    return any;
}
void probe_numa(garage_ec_ctx *ctx)
{
    char busid[64] = {0}, path[160], buf[4096];
    if (cudaDeviceGetPCIBusId(busid, sizeof(busid), ctx->device) != cudaSuccess) {
        (void)cudaGetLastError();
        return;
    }
    for (char *c = busid; *c; c++) *c = (char)tolower((unsigned char)*c);
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", busid);
    if (!read_small_file(path, buf, sizeof(buf))) return;
    const int node = atoi(buf);
    if (node < 0) return;
    ctx->numa_node = node;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    if (read_small_file(path, buf, sizeof(buf))) ctx->have_node_cpus = parse_cpulist(buf, &ctx->node_cpus);
}
// node a page lives on (move_pages with nodes == NULL only queries), -1 if unknown
int node_of_page(void *p)
{
    int status = -1;
    void *pages[1] = {p};
    if (syscall(SYS_move_pages, 0, 1ul, pages, nullptr, &status, 0) != 0) return -1;
    return status;
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_geometry(const garage_ec_ctx *ctx, size_t stride, size_t n, int shards_per_stripe)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (stride == 0 || (stride & 15)) return GARAGE_EC_E_ALIGN;
    if ((unsigned long long)stride * (unsigned long long)shards_per_stripe >= (1ull << 32))
        return GARAGE_EC_E_INVALID;
    if (n > 0xffffffffull) return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

// ---- timing ---------------------------------------------------------------------------
struct TimedLaunch {
    garage_ec_ctx *ctx;
    cudaStream_t st;
    cudaEvent_t a = nullptr, b = nullptr;
    TimedLaunch(garage_ec_ctx *c, cudaStream_t s) : ctx(c), st(s)
    {
        if (!ctx->timing) return;
        std::lock_guard<std::mutex> g(ctx->misc_mu);
        for (cudaEvent_t *e : {&a, &b}) {
            if (!ctx->free_events.empty()) {
                *e = ctx->free_events.back();
                ctx->free_events.pop_back();
            } else if (cudaEventCreate(e) != cudaSuccess) {
                *e = nullptr;
            }
        }
        if (a && b) cudaEventRecord(a, st);
    }
    ~TimedLaunch()
    {
        if (!a || !b) return;
        cudaEventRecord(b, st);
        std::lock_guard<std::mutex> g(ctx->misc_mu);
        ctx->pending.emplace_back(a, b);
    }
};

// ---- kernel dispatch --------------------------------------------------------------------
// Launch shape, table layout and shared-memory carve-up are compile-time functions of (k, mode):
// StreamCfg in rs_kernels.cuh.
template <int K, int MODE>
cudaError_t launch_apply_t(const garage_ec_ctx *ctx, const ApplyParams &p, cudaStream_t st)
{
    static std::atomic<int> configured_for_device{-1};  // per instantiation
    using CFG = StreamCfg<K, cfg_mode(MODE)>;
    auto kern = rs_apply_kernel<K, MODE>;
    if ((size_t)CFG::kSmem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    // opt-in shared memory size is a per-function, per-device attribute; setting it is cheap
    // but not free, so remember the last device it was set for.
    if (configured_for_device.load(std::memory_order_acquire) != ctx->device) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CFG::kSmem);
        if (e != cudaSuccess) return e;
        configured_for_device.store(ctx->device, std::memory_order_release);
    }
    kern<<<ctx->sm_count, CFG::kThreads, CFG::kSmem, st>>>(p);
    return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_apply(garage_ec_ctx *ctx, const ApplyParams &p, cudaStream_t st)
{
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    switch (p.k) {
#define GEC_CASE(KK) case KK: return launch_apply_t<KK, MODE>(ctx, p, st);
#ifndef GEC_FAST_BUILD
        GEC_CASE(1) GEC_CASE(2) GEC_CASE(3) GEC_CASE(4) GEC_CASE(5) GEC_CASE(6) GEC_CASE(7) GEC_CASE(8)
        GEC_CASE(9) GEC_CASE(11) GEC_CASE(12) GEC_CASE(13) GEC_CASE(14) GEC_CASE(15) GEC_CASE(16)
        GEC_CASE(17) GEC_CASE(18) GEC_CASE(19) GEC_CASE(20) GEC_CASE(21) GEC_CASE(22) GEC_CASE(23) GEC_CASE(24)
        GEC_CASE(25) GEC_CASE(26) GEC_CASE(27) GEC_CASE(28) GEC_CASE(29) GEC_CASE(30) GEC_CASE(31) GEC_CASE(32)
#endif
        GEC_CASE(10)
#if defined(GEC_FAST_BUILD) && GEC_FAST_BUILD != 10
        GEC_CASE(GEC_FAST_BUILD)
#endif
#undef GEC_CASE
    default: return cudaErrorInvalidConfiguration;
    }
}

uint32_t items_per_stripe(size_t stride) { return (uint32_t)((stride / 16 + 31) / 32); }

template <int K, int MODE>
cudaError_t launch_pb_t(const garage_ec_ctx *ctx, const ApplyParams &p, cudaStream_t st)
{
    static std::atomic<int> configured_for_device{-1};  // per instantiation
    using CFG = PbCfg<K, MODE>;
    auto kern = pb_apply_kernel<K, MODE>;
    if ((size_t)CFG::kSmem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    if (configured_for_device.load(std::memory_order_acquire) != ctx->device) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CFG::kSmem);
        if (e != cudaSuccess) return e;
        configured_for_device.store(ctx->device, std::memory_order_release);
    }
    kern<<<ctx->sm_count, CFG::kThreads, CFG::kSmem, st>>>(p);
    return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_pb(garage_ec_ctx *ctx, const ApplyParams &p, cudaStream_t st)
{
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    switch (p.k) {
#define GEC_CASE(KK) case KK: return launch_pb_t<KK, MODE>(ctx, p, st);
        GEC_CASE(1) GEC_CASE(2) GEC_CASE(3) GEC_CASE(4) GEC_CASE(5) GEC_CASE(6) GEC_CASE(7) GEC_CASE(8)
        GEC_CASE(9) GEC_CASE(10) GEC_CASE(11) GEC_CASE(12) GEC_CASE(13) GEC_CASE(14) GEC_CASE(15) GEC_CASE(16)
#undef GEC_CASE
    default: return cudaErrorInvalidConfiguration;
    }
}

// PB encode / verify: one launch per batch slice, all m <= 4 rows in one pass (pb_apply_kernel)
int run_pb_uniform(garage_ec_ctx *ctx, int mode, const uint8_t *src, size_t src_pitch, uint8_t *dst, size_t dst_pitch,
                   uint32_t *mismatch, const uint32_t *shard_len, size_t stride, size_t n, cudaStream_t st)
{
    const uint32_t ips = (uint32_t)((stride / 32 + 31) / 32);  // 32-column chunks of the longest half
    const size_t max_n = 0xffffffffull / ips;
    TimedLaunch tl(ctx, st);
    for (size_t s0 = 0; s0 < n; s0 += max_n) {
        const size_t cnt = n - s0 < max_n ? n - s0 : max_n;
        ApplyParams p;
        memset(&p, 0, sizeof(p));
        p.src = src + s0 * src_pitch;
        p.src_pitch = src_pitch;
        p.dst = dst ? dst + s0 * dst_pitch : nullptr;
        p.dst_pitch = dst_pitch;
        p.shard_len = shard_len ? shard_len + s0 : nullptr;
        p.mismatch = mismatch ? mismatch + s0 : nullptr;
        p.stride = (uint32_t)stride;
        p.n = (uint32_t)cnt;
        p.k = (uint32_t)ctx->k;
        p.rows = (uint32_t)ctx->m;
        p.items_per_stripe = ips;
        p.row_bytes = 128;
        memcpy(p.coef, ctx->P, (size_t)ctx->k * ctx->m);
        cudaError_t e = mode == kModeEncode ? launch_pb<kModeEncode>(ctx, p, st) : launch_pb<kModeVerify>(ctx, p, st);
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "pb_apply_kernel launch");
    }
    return GARAGE_EC_OK;
}

// cuTensorMapEncodeTiled through the runtime (no link against libcuda)
using TensorMapEncodeFn = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                       const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
TensorMapEncodeFn tensor_map_encoder()
{
    static std::atomic<void *> cached{nullptr};
    static std::atomic<int> tried{0};
    if (!tried.load(std::memory_order_acquire)) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        (void)cudaGetLastError();
        cached.store(fn, std::memory_order_release);
        tried.store(1, std::memory_order_release);
    }
    return reinterpret_cast<TensorMapEncodeFn>(cached.load(std::memory_order_acquire));
}
// 2-D view of a shard array for the TMA path of the uniform kernels: dim0 = stride/4 uint32, dim1 = rows shards.
// false = no tensor map (the kernel then issues one 1-D bulk copy per row)
bool make_src_tensor_map(CUtensorMap *tm, const uint8_t *src, size_t stride, size_t rows, int box_rows)
{
#if GEC_TMAP
    TensorMapEncodeFn enc = tensor_map_encoder();
    if (!enc || stride < kStageRowBytes || rows == 0 || rows > 0xffffffffull || box_rows > 256) return false;
    const cuuint64_t gdim[2] = {(cuuint64_t)(stride / 4), (cuuint64_t)rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)stride};
    const cuuint32_t box[2] = {kStageRowBytes / 4, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<uint8_t *>(src), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
#else
    (void)tm, (void)src, (void)stride, (void)rows, (void)box_rows;
    return false;
#endif
}

// ---- Clay(k, m) (clay_kernels.cuh) ------------------------------------------------------------------------------
ClayParams clay_params(const garage_ec_ctx *ctx, size_t stride, size_t n)
{
    ClayParams c;
    memset(&c, 0, sizeof(c));
    c.stride = (uint32_t)stride;
    c.n = (uint32_t)n;
    c.k = (uint32_t)ctx->k;
    c.m = (uint32_t)ctx->m;
    c.s = (uint32_t)ctx->cg.s;
    c.q = (uint32_t)ctx->cg.q;
    c.t = (uint32_t)ctx->cg.t;
    c.alpha = (uint32_t)ctx->cg.alpha;
    c.ips = (uint32_t)((stride / ctx->cg.alpha + kClayColBytes - 1) / kClayColBytes);
    for (int y = 0, v = 1; y <= ctx->cg.t; y++, v *= ctx->cg.q) c.qpow[y] = (uint32_t)v;
    memcpy(c.coef, ctx->P, (size_t)(ctx->k + ctx->cg.s) * ctx->m);
    return c;
}
template <int MODE>
cudaError_t launch_clay(garage_ec_ctx *ctx, const ClayParams &c, cudaStream_t st)
{
    static std::atomic<int> configured_for_device{-1};  // per instantiation
    const size_t smem = (size_t)ctx->cg.alpha * clay_layer_words((uint32_t)ctx->cg.n) * 4;
    auto kern = clay_apply_kernel<MODE>;
    if (configured_for_device.load(std::memory_order_acquire) != ctx->device) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)(kClayMaxAlpha * clay_layer_words(kClayMaxNodes) * 4));
        if (e != cudaSuccess) return e;
        configured_for_device.store(ctx->device, std::memory_order_release);
    }
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    const size_t items = (size_t)c.n * c.ips;
    const unsigned grid = (unsigned)std::max<size_t>(1, std::min<size_t>(items, (size_t)ctx->sm_count * 16));
    kern<<<grid, kClayThreads, smem, st>>>(c);
    return cudaGetLastError();
}
// encode (mode 0) / verify (mode 2): one launch; n * items per stripe stays below 2^32 by the stride check
int run_clay(garage_ec_ctx *ctx, int mode, const uint8_t *src, size_t src_pitch, uint8_t *dst, size_t dst_pitch,
             uint32_t *mismatch, const uint32_t *shard_len, size_t stride, size_t n, cudaStream_t st)
{
    if (n == 0) return GARAGE_EC_OK;
    ClayParams c = clay_params(ctx, stride, n);
    c.src = src;
    c.src_pitch = src_pitch;
    c.shard_len = shard_len;
    c.mismatch = mismatch;
    if (mode == kModeEncode) {
        c.dst = dst;
        c.dst_pitch = dst_pitch;
    } else {  // verify reads the stored parities of the shard layout
        c.dst = const_cast<uint8_t *>(src);
        c.dst_pitch = src_pitch;
        c.par_off = (uint32_t)ctx->k;
    }
    TimedLaunch tl(ctx, st);
    cudaError_t e = mode == kModeEncode ? launch_clay<kModeEncode>(ctx, c, st) : launch_clay<kModeVerify>(ctx, c, st);
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "clay_apply_kernel launch");
    return GARAGE_EC_OK;
}

// Device-resident encode (mode 0) / verify (mode 2) of n stripes, split so that
// n * items_per_stripe stays below 2^32 and m > 4 runs in passes of 4 rows.
int run_uniform(garage_ec_ctx *ctx, int mode, const uint8_t *src, size_t src_pitch, uint8_t *dst,
                size_t dst_pitch, uint32_t *mismatch, const uint32_t *shard_len, size_t stride,
                size_t n, cudaStream_t st)
{
    if (ctx->pb) return run_pb_uniform(ctx, mode, src, src_pitch, dst, dst_pitch, mismatch, shard_len, stride, n, st);
    if (ctx->clay) return run_clay(ctx, mode, src, src_pitch, dst, dst_pitch, mismatch, shard_len, stride, n, st);
    const uint32_t ips = items_per_stripe(stride);
    // the kernel's work counter runs past the item count by at most two claimed runs per warp
    const size_t max_n = (0xffffffffull - (1ull << 24)) / ips;
    TimedLaunch tl(ctx, st);
    if (n == 0) return GARAGE_EC_OK;
    // one zeroed work counter per launch (rs_apply_kernel's dynamic schedule): stream-ordered scratch, so the
    // call stays capturable in a CUDA graph
    const size_t launches = (n + max_n - 1) / max_n * (size_t)((ctx->m + kRowsPerPass - 1) / kRowsPerPass);
    return with_stream_scratch(ctx, launches * sizeof(uint32_t), st, [&](uint8_t *scratch) -> int {
        uint32_t *counter = reinterpret_cast<uint32_t *>(scratch);
        cudaError_t e = cudaMemsetAsync(counter, 0, launches * sizeof(uint32_t), st);
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaMemsetAsync(counter)");
        for (size_t s0 = 0; s0 < n; s0 += max_n) {
            const size_t cnt = n - s0 < max_n ? n - s0 : max_n;
            for (int r0 = 0; r0 < ctx->m; r0 += kRowsPerPass) {
                ApplyParams p;
                memset(&p, 0, sizeof(p));
                p.src = src + s0 * src_pitch;
                p.src_pitch = src_pitch;
                p.dst = dst ? dst + s0 * dst_pitch + (size_t)r0 * stride : nullptr;
                p.dst_pitch = dst_pitch;
                p.shard_len = shard_len ? shard_len + s0 : nullptr;
                p.mismatch = mismatch ? mismatch + s0 : nullptr;
                p.counter = counter++;
                p.stride = (uint32_t)stride;
                p.n = (uint32_t)cnt;
                p.k = (uint32_t)ctx->k;
                p.rows = (uint32_t)(ctx->m - r0 < kRowsPerPass ? ctx->m - r0 : kRowsPerPass);
                p.row_off = (uint32_t)r0;
                p.items_per_stripe = ips;
                p.row_bytes = 128;
                p.rows_per_stripe = (uint32_t)(src_pitch / stride);
                p.use_tmap = (GEC_TMAP && ctx->k >= GEC_TMAP_FROM_K && make_src_tensor_map(&p.tmap, p.src, stride, cnt * p.rows_per_stripe,
                                                  (GEC_SPLIT_STAGE && ctx->k > 16) ? 16 : ctx->k)) ? 1u : 0u;  // box rows: StreamCfg::kSrcRows
                for (uint32_t i = 0; i < p.rows; i++)
                    memcpy(p.coef + i * ctx->k, ctx->P + (r0 + i) * ctx->k, ctx->k);
                e = mode == kModeEncode ? launch_apply<kModeEncode>(ctx, p, st) : launch_apply<kModeVerify>(ctx, p, st);
                if (e != cudaSuccess) return set_cuda_error(ctx, e, "rs_apply_kernel launch");
            }
        }
        return GARAGE_EC_OK;
    });
}

// Device scratch of run_reconstruct for n stripes: StripePlans | apply counter (16 B) | Clay: the present / want maps of
// the base code, n' bytes each per stripe
size_t plan_scratch_bytes(const garage_ec_ctx *ctx, size_t n)
{
    return n * sizeof(StripePlan) + 16 + (ctx->clay ? (2 * n * (size_t)ctx->cg.n + 15) / 16 * 16 : 0);
}

// Device-resident reconstruct.  plan_scratch: plan_scratch_bytes(ctx, n) of device memory.
int run_reconstruct(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present, const uint8_t *want,
                    int32_t *status, const uint32_t *shard_len, size_t stride, size_t n,
                    uint8_t *plan_scratch, cudaStream_t st, bool present_is_bad = false)
{
    StripePlan *plan = reinterpret_cast<StripePlan *>(plan_scratch);
    uint32_t *counter = reinterpret_cast<uint32_t *>(plan_scratch + n * sizeof(StripePlan));
    if (ctx->clay) {
        // the caller's maps onto the n' nodes of the base code, the base-code plan by plan_kernel, then the layered
        // decode / repair
        const int N = ctx->cg.n, kb = ctx->k + ctx->cg.s;
        uint8_t *present2 = reinterpret_cast<uint8_t *>(counter) + 16, *want2 = present2 + n * N;
        ClayParams c = clay_params(ctx, stride, n);
        c.src = shards;
        c.dst = shards;
        c.src_pitch = c.dst_pitch = (size_t)(ctx->k + ctx->m) * stride;
        c.par_off = (uint32_t)ctx->k;
        c.shard_len = shard_len;
        c.present = present;
        c.want = want;
        c.status = status;
        c.present_is_bad = present_is_bad ? 1u : 0u;
        c.plan = plan;
        clay_prep_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 4), 256, 0, st>>>(c, present2,
                                                                                                             want2);
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "clay_prep_kernel launch");
        PlanParams q;
        memset(&q, 0, sizeof(q));
        q.present = present2;
        q.want = want2;
        q.status = status;
        q.plan = plan;
        q.counter = counter;
        q.n = (uint32_t)n;
        q.k = (uint32_t)kb;
        q.m = (uint32_t)ctx->m;
        q.stride = (uint32_t)stride;
        memcpy(q.P, ctx->P, (size_t)kb * ctx->m);
        plan_kernel<<<(unsigned)((n + kPlanWarps - 1) / kPlanWarps), kPlanWarps * 32, 0, st>>>(q);
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
        e = cudaGetLastError();
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "plan_kernel launch");
        TimedLaunch tl(ctx, st);
        e = launch_clay<kModePlan>(ctx, c, st);
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "clay_apply_kernel<plan> launch");
        return GARAGE_EC_OK;
    }
    PlanParams q;
    memset(&q, 0, sizeof(q));
    q.present = present;
    q.want = want;
    q.status = status;
    q.plan = plan;
    q.counter = counter;
    q.n = (uint32_t)n;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.l = (uint32_t)ctx->l;
    q.pb = ctx->pb ? 1u : 0u;
    q.present_is_bad = present_is_bad ? 1u : 0u;
    q.shard_len = shard_len;
    q.stride = (uint32_t)stride;
    memcpy(q.P, ctx->P, (size_t)ctx->k * ctx->m);
    plan_kernel<<<(unsigned)((n + kPlanWarps - 1) / kPlanWarps), kPlanWarps * 32, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "plan_kernel launch");

    TimedLaunch tl(ctx, st);
    const size_t pitch = (size_t)(ctx->k + ctx->m) * stride;
    // PB: the plan is over half-rows, 2k sources and up to 2m outputs of length shard_len/2
    const int nout = ctx->pb ? 2 * ctx->m : ctx->m;
    for (int r0 = 0; r0 < nout; r0 += kRowsPerPass) {
        if (r0 > 0) {
            e = cudaMemsetAsync(counter, 0, sizeof(uint32_t), st);
            if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaMemsetAsync(counter)");
        }
        ApplyParams p;
        memset(&p, 0, sizeof(p));
        p.src = shards;
        p.dst = shards;
        p.src_pitch = p.dst_pitch = pitch;
        p.shard_len = shard_len;
        p.plan = plan;
        p.counter = counter;
        p.stride = (uint32_t)stride;
        p.n = (uint32_t)n;
        p.k = (uint32_t)(ctx->pb ? 2 * ctx->k : ctx->k);
        p.half = ctx->pb ? 1u : 0u;
        p.row_off = (uint32_t)r0;
        p.row_bytes = 128;
        e = launch_apply<kModePlan>(ctx, p, st);
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "rs_apply_kernel<plan> launch");
    }
    return GARAGE_EC_OK;
}

// The rows plan_kernel reads for one stripe (present / want: k+m bytes, want nullable = every absent shard): for PB
// bit 2i / 2i+1 of *rows = a- / b-half of shard i, for RS, LRC and Clay bit i = shard i (up to 40 shards: two bits
// each do not fit in 64).  read_halves gives the halves of shard i either way.  False if a wanted shard cannot be
// rebuilt.  HOST paths upload only these.
bool stripe_read_plan(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint64_t *rows)
{
    uint64_t pm = 0, wm = 0;
    for (int i = 0; i < ctx->k + ctx->m; i++) {
        pm |= (uint64_t)(present[i] != 0) << i;
        wm |= (uint64_t)(!want || want[i] != 0) << i;
    }
    *rows = 0;
    return ctx->clay ? clay_read_set(ctx->k, ctx->m, pm, wm, rows)
                     : h_read_plan(PlanCode{ctx->k, ctx->m, ctx->l, ctx->pb, ctx->P}, pm, wm, rows);
}
// bit 0 / 1: the a- / b-half of shard i is read (3 for every shard RS, LRC and Clay read)
unsigned read_halves(const garage_ec_ctx *ctx, uint64_t rows, size_t i)
{
    return ctx->pb ? (unsigned)(rows >> (2 * i)) & 3u : ((rows >> i) & 1) ? 3u : 0u;
}
bool stripe_read_set(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint64_t *read)
{
    uint64_t hv = 0;
    const bool ok = stripe_read_plan(ctx, present, want, &hv);
    *read = 0;
    for (int i = 0; i < ctx->k + ctx->m; i++)
        if (read_halves(ctx, hv, i)) *read |= 1ull << i;
    return ok;
}
// The pieces of shard i a HOST upload copies, as f(offset, bytes): `whole` bytes from 0 for a shard of the read set,
// (PB) each planned half of shard_len/2 bytes, or (Clay repair: every shard but one is read) the runs of the repair
// layers {z : z_y0 = x0} of the one absent shard f = (x0, y0), q^y0 sub-chunks every q^(y0+1)
template <class F>
void for_each_read_piece(const garage_ec_ctx *ctx, uint64_t rows, size_t i, size_t len, size_t whole, F &&f)
{
    const unsigned b = read_halves(ctx, rows, i);
    if (!b) return;
    if (ctx->clay) {
        const int tot = ctx->k + ctx->m;
        int nread = 0, f_shard = 0;
        for (int j = 0; j < tot; j++) {
            if (read_halves(ctx, rows, j)) nread++;
            else f_shard = j;
        }
        if (nread != tot - 1) return f((size_t)0, whole);
        const int a = clay_node(ctx->k, ctx->cg.s, f_shard), q = ctx->cg.q, x0 = a % q, y0 = a / q;
        size_t run = 1;
        for (int y = 0; y < y0; y++) run *= (size_t)q;
        const size_t sub = len / (size_t)ctx->cg.alpha, period = run * q;
        for (size_t z0 = x0 * run; z0 < (size_t)ctx->cg.alpha; z0 += period) f(z0 * sub, run * sub);
        return;
    }
    if (!ctx->pb) f((size_t)0, whole);
    else if (b == 3) f((size_t)0, len);
    else f(b == 1 ? (size_t)0 : len / 2, len / 2);
}
// The plan of unit g (DESIGN.md 2.10) of one stripe of shard length len (sp / wn: its k+m seg_present and want bytes,
// wn nullable): *rows as stripe_read_plan gives them for the unit's presence map, *work = a wanted shard is absent in
// the unit.  False if the unit cannot be rebuilt.  The HOST reconstruct by segment uploads, and
// garage_ec_segment_read_ranges names, the for_each_unit_piece pieces of these rows.
bool unit_read_plan(const garage_ec_ctx *ctx, const uint8_t *sp, const uint8_t *wn, uint32_t len, uint32_t g,
                    uint64_t *rows, bool *work)
{
    uint8_t up[GARAGE_EC_MAX_K + GARAGE_EC_MAX_M];
    *work = false;
    for (int i = 0; i < ctx->k + ctx->m; i++) {
        up[i] = unit_present(sp[i], len, g, ctx->pb) ? 1 : 0;
        *work |= !up[i] && (!wn || wn[i]);
    }
    return stripe_read_plan(ctx, up, wn, rows);
}
// The pieces of shard i that unit g's plan `rows` reads, as f(offset, bytes): the unit's columns, for PB those of each
// planned half
template <class F>
void for_each_unit_piece(const garage_ec_ctx *ctx, uint64_t rows, size_t i, uint32_t len, uint32_t g, F &&f)
{
    uint32_t base, ulen;
    unit_columns(len, g, ctx->pb, &base, &ulen);
    const unsigned b = read_halves(ctx, rows, i);
    for (unsigned h = 0; h < (ctx->pb ? 2u : 1u); h++)
        if ((b >> h) & 1) f(base + h * (size_t)(len / 2), (size_t)ulen);
}
// Every stripe's shard_len (NULL: stride) must be at most the stride and, for PB, a multiple of 32 so that the halves
// are 16-byte aligned; for Clay, a multiple of 16*alpha, so that every layer's sub-chunk is
bool shard_lens_ok(const garage_ec_ctx *ctx, const uint32_t *shard_len, size_t stride, size_t n)
{
    const size_t unit = ctx->clay ? (size_t)ctx->quantum : ctx->pb ? 32 : 1;
    if (!shard_len) return stride % unit == 0;
    for (size_t s = 0; s < n; s++)
        if ((shard_len[s] % unit) || shard_len[s] > stride) return false;
    return true;
}
// 64-bit: a PB or Clay length that does not fit in 32 bits is larger than any stride, so the stride checks reject it
uint64_t code_shard_len(const garage_ec_ctx *ctx, uint32_t block_len)
{
    return ::garage_ec::code_shard_len(block_len, ctx->k, ctx->quantum);
}

// ---- batched async copies ---------------------------------------------------------------
// Reconstruct moves many shard-sized pieces per stripe (only the k survivors go up, only the
// rebuilt shards come back).  One cudaMemcpyBatchAsync per chunk instead of thousands of
// cudaMemcpyAsync calls keeps the CPU off the critical path; adjacent pieces are merged.
struct CopyBatch {
    std::vector<void *> dst, src;
    std::vector<size_t> sz;
    bool use_batch = true;  // false: the host side is pageable memory, copied piece by piece
    void add(void *d, const void *s, size_t n)
    {
        if (!n) return;
        if (!dst.empty() && static_cast<uint8_t *>(dst.back()) + sz.back() == d &&
            static_cast<const uint8_t *>(src.back()) + sz.back() == s) {
            sz.back() += n;
            return;
        }
        dst.push_back(d);
        src.push_back(const_cast<void *>(s));
        sz.push_back(n);
    }
    int flush(garage_ec_ctx *ctx, cudaMemcpyKind kind, cudaStream_t st)
    {
        const size_t cnt = dst.size();
        if (!cnt) return GARAGE_EC_OK;
        if (fault_hit(ctx)) {
            dst.clear();
            src.clear();
            sz.clear();
            return set_cuda_error(ctx, cudaErrorUnknown, "injected fault at batched copy");
        }
        bool done = false;
        if (cnt > 1 && use_batch && ctx->batch_copy_ok.load(std::memory_order_relaxed)) {
            cudaMemcpyAttributes attr;
            memset(&attr, 0, sizeof(attr));
            attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
            size_t attr_idx = 0, fail = 0;
            cudaError_t e = cudaMemcpyBatchAsync(dst.data(), src.data(), sz.data(), cnt, &attr, &attr_idx, 1,
                                                 &fail, st);
            if (e == cudaSuccess) {
                done = true;
            } else {
                (void)cudaGetLastError();
                ctx->batch_copy_ok.store(0, std::memory_order_relaxed);
            }
        }
        if (!done)
            for (size_t i = 0; i < cnt; i++) CU_TRY(ctx, cudaMemcpyAsync(dst[i], src[i], sz[i], kind, st));
        dst.clear();
        src.clear();
        sz.clear();
        return GARAGE_EC_OK;
    }
};

// ---- host lanes -----------------------------------------------------------------------
// A lane's buffers are sized for a full pipeline chunk the first time they are needed (not for the
// batch at hand): a batching front-end calls with a different number of blocks every time, and every
// cudaFree + cudaMalloc to grow a lane synchronises the whole device -- with growth-on-demand the first few
// hundred calls of a fresh context paid milliseconds each
constexpr size_t kLaneFloorBytes = 128ull << 20, kLaneSmallFloorBytes = 2ull << 20;
int lane_reserve(garage_ec_ctx *ctx, HostLane &L, size_t buf_bytes, size_t small_bytes)
{
    if (buf_bytes < kLaneFloorBytes) buf_bytes = kLaneFloorBytes;
    if (small_bytes < kLaneSmallFloorBytes) small_bytes = kLaneSmallFloorBytes;
    if (!L.stream) CU_TRY(ctx, cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    if (L.d_cap < buf_bytes) {
        if (L.d_buf) cudaFree(L.d_buf);
        L.d_buf = nullptr;
        L.d_cap = 0;
        CU_TRY(ctx, cudaMalloc(&L.d_buf, buf_bytes));
        L.d_cap = buf_bytes;
    }
    if (L.small_cap < small_bytes) {
        if (L.d_small) cudaFree(L.d_small);
        L.d_small = nullptr;
        L.small_cap = 0;
        CU_TRY(ctx, cudaMalloc(&L.d_small, small_bytes));
        L.small_cap = small_bytes;
    }
    return GARAGE_EC_OK;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// A lane's small device buffer: 16-byte aligned regions, handed out in the order they are taken
struct SmallLayout {
    size_t bytes = 0;
    size_t take(size_t n)
    {
        const size_t o = bytes;
        bytes += align_up(n, 16);
        return o;
    }
};

// One chunk of a HOST-mode call: stripes [s0, s0 + cnt) on lane L, with the lane's pageable staging
struct HostChunk {
    HostLane *L = nullptr;
    uint8_t *host = nullptr;
    size_t s0 = 0, cnt = 0;
    bool pending = false;  // issued, not retired yet
};
using Retire = std::function<int(const HostChunk &)>;

// The chunk pipeline every HOST-mode call stages through: n stripes in chunks of cs (about kHostChunkBytes of
// bytes_per_stripe each), round robin over the three lanes of one leased lane set, so that H2D, kernels and D2H of
// consecutive chunks overlap.  bytes_per_stripe == 0: one chunk of all n stripes on lane 0 (zero-copy calls).
//
// It owns the lease and every host object a queued copy reads or writes: the copy lists, the per-lane pageable
// staging and the status array of a caller that passed none.  The destructor waits for every lane stream before the
// set goes back to the pool and before those members are freed, so no DMA touches the caller's buffers after a HOST
// call has returned, on every path including the early error returns ("the library keeps no pointer",
// include/garage_ec.h).  n == 0 takes no lease.
class HostPipeline {
public:
    static constexpr size_t kHostChunkBytes = 48ull << 20;  // target source bytes per chunk
    const size_t n, cs;
    CopyBatch up, down;  // the chunk being issued (or, in a retire step, the chunk being retired)
    std::function<void()> before_release;  // runs once every lane stream is idle, before the set goes back to the pool

    HostPipeline(garage_ec_ctx *ctx, size_t n, size_t bytes_per_stripe)
        : n(n), cs(bytes_per_stripe ? std::min(std::max<size_t>(kHostChunkBytes / bytes_per_stripe, 1), n) : n),
          ctx_(ctx), lanes_(bytes_per_stripe ? kHostLanes : 1)
    {
    }
    HostPipeline(const HostPipeline &) = delete;
    HostPipeline &operator=(const HostPipeline &) = delete;
    ~HostPipeline()
    {
        if (!set_) return;
        for (HostLane &L : set_->lanes)
            if (L.stream) (void)cudaStreamSynchronize(L.stream);
        (void)cudaGetLastError();
        if (before_release) before_release();  // the lanes are idle and still ours
        {
            std::lock_guard<std::mutex> lk(ctx_->pool_mu);
            ctx_->free_sets.push_back(set_);
        }
        ctx_->pool_cv.notify_one();
    }

    // lease a lane set and size its lanes: `buf` bytes of chunk buffer, `small` bytes of small buffer (SmallLayout)
    // and `host` bytes of pageable staging per lane
    int reserve(size_t buf, size_t small, size_t host = 0)
    {
        if (!n) return GARAGE_EC_OK;
        {
            std::unique_lock<std::mutex> lk(ctx_->pool_mu);
            ctx_->pool_cv.wait(lk, [&] { return !ctx_->free_sets.empty() || ctx_->n_sets < kMaxLaneSets; });
            if (!ctx_->free_sets.empty()) {
                set_ = ctx_->free_sets.back();
                ctx_->free_sets.pop_back();
            } else {
                set_ = new (std::nothrow) LaneSet();
                if (set_) ctx_->n_sets++;
            }
        }
        if (!set_) return GARAGE_EC_E_NOMEM;
        for (int l = 0; l < lanes_; l++) {
            int rc = lane_reserve(ctx_, set_->lanes[l], buf, small);
            if (rc) return rc;
        }
        host_stride_ = align_up(host, 16);
        host_.resize(host_stride_ * lanes_);
        return GARAGE_EC_OK;
    }

    // the caller's status array, or one of ours for the n stripes
    int32_t *status_out(int32_t *status)
    {
        if (status) return status;
        own_status_.assign(n, 0);
        return own_status_.data();
    }

    // issue(chunk) queues every chunk.  A lane whose previous chunk left work for the host -- a retire step, or the
    // lane's pageable staging, which the next chunk overwrites -- is waited for before it takes the next chunk, and
    // retire(previous chunk) runs then.
    template <class Issue>
    int run(Issue &&issue, const Retire &retire = nullptr)
    {
        size_t c = 0;
        for (size_t s0 = 0; s0 < n; s0 += cs, c++) {
            HostChunk &ch = chunks_[c % lanes_];
            if (ch.pending && (retire || host_stride_)) {
                int rc = retire_chunk(ch, retire);
                if (rc) return rc;
            }
            ch.L = &set_->lanes[c % lanes_];
            ch.host = host_.data() + (c % lanes_) * host_stride_;
            ch.s0 = s0;
            ch.cnt = n - s0 < cs ? n - s0 : cs;
            ch.pending = true;
            int rc = issue(ch);
            if (rc) return rc;
        }
        return GARAGE_EC_OK;
    }

    // retire every pending chunk, then wait for every lane
    int drain(const Retire &retire = nullptr)
    {
        if (!set_) return GARAGE_EC_OK;
        for (int l = 0; l < lanes_ && retire; l++) {
            if (!chunks_[l].pending) continue;
            int rc = retire_chunk(chunks_[l], retire);
            if (rc) return rc;
        }
        for (int l = 0; l < lanes_; l++) CU_TRY(ctx_, lane_wait(ctx_, set_->lanes[l]));
        return GARAGE_EC_OK;
    }

private:
    int retire_chunk(HostChunk &ch, const Retire &retire)
    {
        ch.pending = false;
        CU_TRY(ctx_, lane_wait(ctx_, *ch.L));
        return retire ? retire(ch) : GARAGE_EC_OK;
    }

    garage_ec_ctx *ctx_;
    const int lanes_;
    std::vector<uint8_t> host_;
    size_t host_stride_ = 0;
    std::vector<int32_t> own_status_;
    HostChunk chunks_[kHostLanes];
    LaneSet *set_ = nullptr;
};

int create_common(garage_ec_ctx **out, int device, int k, int m, const uint8_t *P, int kind, int l = 0, bool pb = false,
                  const ClayGeo *clay = nullptr)
{
    if (!out) return GARAGE_EC_E_INVALID;
    *out = nullptr;
    if (k < 1 || k > kMaxK || m < 1 || m > kMaxM) return GARAGE_EC_E_INVALID;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        (void)cudaGetLastError();
        return GARAGE_EC_E_NODEVICE;
    }
    if (device < 0 || device >= ndev) return GARAGE_EC_E_NODEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return GARAGE_EC_E_NODEVICE;
    if (prop.major != 9 || prop.minor != 0) return GARAGE_EC_E_NODEVICE;  // built for sm_90a only
    garage_ec_ctx *ctx = new (std::nothrow) garage_ec_ctx();
    if (!ctx) return GARAGE_EC_E_NOMEM;
    ctx->device = device;
    ctx->k = k;
    ctx->m = m;
    ctx->l = l;
    ctx->pb = pb;
    ctx->quantum = pb ? kPbQuantum : 1;
    if (clay) {
        ctx->clay = true;
        ctx->cg = *clay;
        ctx->quantum = kClayColBytes * (uint32_t)clay->alpha;
    }
    if (P) {
        memcpy(ctx->P, P, (size_t)k * m);
    } else if (!h_build_matrix(clay ? k + clay->s : k, m, kind, ctx->P)) {
        delete ctx;
        return GARAGE_EC_E_INVALID;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    if (cudaSetDevice(device) != cudaSuccess) {
        delete ctx;
        return GARAGE_EC_E_NODEVICE;
    }
    {
        cudaMemPoolProps props;
        memset(&props, 0, sizeof(props));
        props.allocType = cudaMemAllocationTypePinned;
        props.handleTypes = cudaMemHandleTypeNone;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = device;
        if (cudaMemPoolCreate(&ctx->pool, &props) == cudaSuccess) {
            unsigned long long keep = ~0ull;
            (void)cudaMemPoolSetAttribute(ctx->pool, cudaMemPoolAttrReleaseThreshold, &keep);
        } else {
            ctx->pool = nullptr;  // fall back to the default pool
        }
        (void)cudaGetLastError();
    }
    probe_numa(ctx);
    if (const char *b = getenv("GARAGE_EC_BATCHCOPY")) ctx->batch_copy_ok.store(b[0] != '0');
    *out = ctx;
    return GARAGE_EC_OK;
}

}  // namespace

// ======================================================================= C ABI
extern "C" {

int garage_ec_abi_version(void) { return GARAGE_EC_ABI_VERSION; }

const char *garage_ec_strerror(int code)
{
    switch (code) {
    case GARAGE_EC_OK: return "ok";
    case GARAGE_EC_E_INVALID: return "invalid argument or geometry";
    case GARAGE_EC_E_CUDA: return "CUDA runtime error";
    case GARAGE_EC_E_NOMEM: return "out of memory";
    case GARAGE_EC_E_UNRECOVERABLE: return "stripe unrecoverable: the present shards do not determine a wanted shard";
    case GARAGE_EC_E_NODEVICE: return "no usable sm_90 CUDA device (no CPU fallback)";
    case GARAGE_EC_E_ALIGN: return "pointer or stride not 16-byte aligned";
    case GARAGE_EC_E_AUTH: return "block failed authentication (GCM tag or chunk framing)";
    default: return "unknown error";
    }
}

int garage_ec_create(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind)
{
    if (matrix_kind != GARAGE_EC_VANDERMONDE && matrix_kind != GARAGE_EC_CAUCHY) {
        if (out) *out = nullptr;
        return GARAGE_EC_E_INVALID;
    }
    if (matrix_kind == GARAGE_EC_CAUCHY && k + m > 256) return GARAGE_EC_E_INVALID;
    return create_common(out, cuda_device, k, m, nullptr, matrix_kind);
}

int garage_ec_create_lrc(garage_ec_ctx **out, int cuda_device, int k, int l, int r)
{
    uint8_t P[kMaxM * kMaxK];
    if (!h_build_lrc(k, l, r, P)) {
        if (out) *out = nullptr;
        return GARAGE_EC_E_INVALID;
    }
    return create_common(out, cuda_device, k, l + r, P, 0, l);
}

int garage_ec_create_piggyback(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind)
{
    if (k < 1 || k > kPbMaxK || m < kPbMinM || m > kPbMaxM ||
        (matrix_kind != GARAGE_EC_VANDERMONDE && matrix_kind != GARAGE_EC_CAUCHY)) {
        if (out) *out = nullptr;
        return GARAGE_EC_E_INVALID;
    }
    return create_common(out, cuda_device, k, m, nullptr, matrix_kind, 0, true);
}

int garage_ec_create_clay(garage_ec_ctx **out, int cuda_device, int k, int m, int matrix_kind)
{
    ClayGeo g;
    if (!clay_geometry(k, m, &g) || (matrix_kind != GARAGE_EC_VANDERMONDE && matrix_kind != GARAGE_EC_CAUCHY)) {
        if (out) *out = nullptr;
        return GARAGE_EC_E_INVALID;
    }
    return create_common(out, cuda_device, k, m, nullptr, matrix_kind, 0, false, &g);
}

int garage_ec_clay_info(const garage_ec_ctx *ctx, int *q, int *t, int *alpha, int *virtual_nodes, uint8_t *base_rows)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (q) *q = ctx->clay ? ctx->cg.q : 0;
    if (t) *t = ctx->clay ? ctx->cg.t : 0;
    if (alpha) *alpha = ctx->clay ? ctx->cg.alpha : 1;
    if (virtual_nodes) *virtual_nodes = ctx->clay ? ctx->cg.s : 0;
    if (base_rows && ctx->clay) memcpy(base_rows, ctx->P, (size_t)(ctx->k + ctx->cg.s) * ctx->m);
    return GARAGE_EC_OK;
}

int garage_ec_read_ranges(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint32_t shard_len,
                          garage_ec_range *ranges, size_t cap, size_t *n_ranges)
{
    if (!ctx || !present || !n_ranges || (cap && !ranges)) return GARAGE_EC_E_INVALID;
    *n_ranges = 0;
    if (ctx->pb && (shard_len & 31)) return GARAGE_EC_E_INVALID;
    if (ctx->clay && shard_len % ctx->quantum) return GARAGE_EC_E_INVALID;
    uint64_t hv = 0;
    const bool ok = stripe_read_plan(ctx, present, want, &hv);
    if (!ok) return GARAGE_EC_E_UNRECOVERABLE;
    size_t cnt = 0;
    for (int i = 0; i < ctx->k + ctx->m; i++)
        for_each_read_piece(ctx, hv, (size_t)i, shard_len, shard_len, [&](size_t off, size_t bytes) {
            if (cnt && cnt <= cap && ranges[cnt - 1].shard == (uint32_t)i &&
                ranges[cnt - 1].offset + ranges[cnt - 1].len == off) {
                ranges[cnt - 1].len += (uint32_t)bytes;  // adjacent: merged
                return;
            }
            if (cnt < cap) ranges[cnt] = garage_ec_range{(uint32_t)i, (uint32_t)off, (uint32_t)bytes};
            cnt++;
        });
    *n_ranges = cnt;
    return cnt > cap ? GARAGE_EC_E_INVALID : GARAGE_EC_OK;
}

int garage_ec_piggyback_info(const garage_ec_ctx *ctx, int *groups, uint8_t *group_of)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (groups) *groups = ctx->pb ? ctx->m - 1 : 0;
    if (group_of)
        for (int j = 0; j < ctx->k; j++) group_of[j] = ctx->pb ? (uint8_t)pb_group_of(ctx->k, ctx->m, j) : 0;
    return GARAGE_EC_OK;
}

int garage_ec_code_shard_len(const garage_ec_ctx *ctx, uint32_t block_len, uint32_t *shard_len)
{
    if (!ctx || !shard_len) return GARAGE_EC_E_INVALID;
    const uint64_t L = code_shard_len(ctx, block_len);
    if (L > 0xffffffffull) return GARAGE_EC_E_INVALID;  // PB with k = 1 and block_len > 2^32 - 128
    *shard_len = (uint32_t)L;
    return GARAGE_EC_OK;
}

int garage_ec_read_plan(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint8_t *halves_out)
{
    if (!ctx || !present || !halves_out || ctx->clay) return GARAGE_EC_E_INVALID;
    uint64_t hv = 0;
    const bool ok = stripe_read_plan(ctx, present, want, &hv);
    for (int i = 0; i < ctx->k + ctx->m; i++) halves_out[i] = (uint8_t)read_halves(ctx, hv, i);
    return ok ? GARAGE_EC_OK : GARAGE_EC_E_UNRECOVERABLE;
}

int garage_ec_code_info(const garage_ec_ctx *ctx, int *local_groups, int *global_parity)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (local_groups) *local_groups = ctx->l;
    if (global_parity) *global_parity = ctx->m - ctx->l;
    return GARAGE_EC_OK;
}

int garage_ec_read_set(const garage_ec_ctx *ctx, const uint8_t *present, const uint8_t *want, uint8_t *read_out)
{
    if (!ctx || !present || !read_out) return GARAGE_EC_E_INVALID;
    uint64_t rd = 0;
    const bool ok = stripe_read_set(ctx, present, want, &rd);
    for (int i = 0; i < ctx->k + ctx->m; i++) read_out[i] = (uint8_t)((rd >> i) & 1);
    return ok ? GARAGE_EC_OK : GARAGE_EC_E_UNRECOVERABLE;
}

int garage_ec_create_with_matrix(garage_ec_ctx **out, int cuda_device, int k, int m,
                                 const uint8_t *parity_rows)
{
    if (!parity_rows) {
        if (out) *out = nullptr;
        return GARAGE_EC_E_INVALID;
    }
    return create_common(out, cuda_device, k, m, parity_rows, 0);
}

void garage_ec_destroy(garage_ec_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (LaneSet *set : ctx->free_sets) {
        for (HostLane &L : set->lanes) {
            if (L.stream) {
                cudaStreamSynchronize(L.stream);
                cudaStreamDestroy(L.stream);
            }
            if (L.d_buf) cudaFree(L.d_buf);
            if (L.d_small) cudaFree(L.d_small);
            if (L.done) cudaEventDestroy(L.done);
            if (L.h_key) cudaFreeHost(L.h_key);
        }
        delete set;
    }
    for (auto &pr : ctx->pending) {
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    for (cudaEvent_t e : ctx->free_events) cudaEventDestroy(e);
    if (ctx->pool) cudaMemPoolDestroy(ctx->pool);
    delete ctx;
}

int garage_ec_matrix(const garage_ec_ctx *ctx, uint8_t *out_m_by_k)
{
    if (!ctx || !out_m_by_k || ctx->clay) return GARAGE_EC_E_INVALID;
    memcpy(out_m_by_k, ctx->P, (size_t)ctx->k * ctx->m);
    return GARAGE_EC_OK;
}

int garage_ec_params(const garage_ec_ctx *ctx, int *k, int *m, int *cuda_device)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (k) *k = ctx->k;
    if (m) *m = ctx->m;
    if (cuda_device) *cuda_device = ctx->device;
    return GARAGE_EC_OK;
}

const char *garage_ec_last_error(const garage_ec_ctx *ctx) { return ctx ? ctx->last_error : ""; }

uint32_t garage_ec_shard_len(uint32_t block_len, int k)
{
    if (k < 1) return 0;
    return (uint32_t)(((unsigned long long)block_len + (unsigned)k - 1) / (unsigned)k);
}

size_t garage_ec_stride_for(uint32_t shard_len) { return align_up(shard_len ? shard_len : 1, 128); }

uint64_t garage_ec_launch_count(const garage_ec_ctx *ctx) { return ctx ? ctx->launches.load() : 0; }

int garage_ec_set_timing(garage_ec_ctx *ctx, int enabled)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    std::lock_guard<std::mutex> g(ctx->misc_mu);
    ctx->timing = enabled != 0;
    return GARAGE_EC_OK;
}

int garage_ec_timing_read(garage_ec_ctx *ctx, double *total_ms, uint64_t *launches)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    cudaSetDevice(ctx->device);
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> todo;
    {
        std::lock_guard<std::mutex> g(ctx->misc_mu);
        todo.swap(ctx->pending);
    }
    double sum = 0;
    uint64_t cnt = 0;
    int rc = GARAGE_EC_OK;
    for (auto &pr : todo) {
        float ms = 0;
        cudaError_t e = cudaEventSynchronize(pr.second);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, pr.first, pr.second);
        if (e == cudaSuccess) {
            sum += ms;
            cnt++;
        } else {
            rc = set_cuda_error(ctx, e, "timing event");
        }
    }
    {
        std::lock_guard<std::mutex> g(ctx->misc_mu);
        for (auto &pr : todo) {
            ctx->free_events.push_back(pr.first);
            ctx->free_events.push_back(pr.second);
        }
    }
    if (total_ms) *total_ms = sum;
    if (launches) *launches = cnt;
    return rc;
}

static int host_alloc_impl(garage_ec_ctx *ctx, void **out, size_t bytes, unsigned extra_flags);

int garage_ec_host_alloc(garage_ec_ctx *ctx, void **out, size_t bytes) { return host_alloc_impl(ctx, out, bytes, 0); }

int garage_ec_host_alloc_wc(garage_ec_ctx *ctx, void **out, size_t bytes)
{
    return host_alloc_impl(ctx, out, bytes, cudaHostAllocWriteCombined);
}

static int host_alloc_impl(garage_ec_ctx *ctx, void **out, size_t bytes, unsigned extra_flags)
{
    if (!ctx || !out || !bytes) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    // Place the pages on the GPU's NUMA node: the driver allocates and pins them inside this call,
    // under the calling thread's memory policy and CPU.  Both are set for the duration of the call
    // (preferred-node policy; where the sandbox forbids set_mempolicy, running on a CPU of the node
    // gives the same result through the default local-allocation policy) and restored afterwards.
    cpu_set_t saved_cpus;
    bool moved = false, policy_set = false;
    if (ctx->numa_node >= 0) {
        unsigned long mask[16] = {0};
        if (ctx->numa_node < (int)(sizeof(mask) * 8)) {
            mask[ctx->numa_node / (8 * sizeof(unsigned long))] |= 1ul << (ctx->numa_node % (8 * sizeof(unsigned long)));
            policy_set = syscall(SYS_set_mempolicy, MPOL_PREFERRED, mask, sizeof(mask) * 8) == 0;
        }
        if (ctx->have_node_cpus && sched_getaffinity(0, sizeof(saved_cpus), &saved_cpus) == 0) {
            cpu_set_t want;
            CPU_AND(&want, &saved_cpus, &ctx->node_cpus);
            if (CPU_COUNT(&want) > 0 && sched_setaffinity(0, sizeof(want), &want) == 0) moved = true;
        }
    }
    cudaError_t e = fault_hit(ctx) ? cudaErrorMemoryAllocation : cudaHostAlloc(out, bytes, cudaHostAllocPortable | extra_flags);
    if (moved) sched_setaffinity(0, sizeof(saved_cpus), &saved_cpus);
    if (policy_set) syscall(SYS_set_mempolicy, MPOL_DEFAULT, nullptr, 0ul);
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaHostAlloc");
    ctx->last_alloc_node = node_of_page(*out);
    return GARAGE_EC_OK;
}

int garage_ec_numa_info(const garage_ec_ctx *ctx, int *gpu_node, int *last_alloc_node)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (gpu_node) *gpu_node = ctx->numa_node;
    if (last_alloc_node) *last_alloc_node = ctx->last_alloc_node;
    return GARAGE_EC_OK;
}

int garage_ec_bind_thread(const garage_ec_ctx *ctx)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    if (ctx->numa_node < 0 || !ctx->have_node_cpus) return 1;  // nothing known: leave the thread alone
    cpu_set_t cur, want;
    if (sched_getaffinity(0, sizeof(cur), &cur) != 0) return 1;
    CPU_AND(&want, &cur, &ctx->node_cpus);
    if (CPU_COUNT(&want) == 0) return 1;  // the cgroup does not allow any CPU of that node
    return sched_setaffinity(0, sizeof(want), &want) == 0 ? GARAGE_EC_OK : 1;
}

int garage_ec_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}

void garage_ec_host_free(garage_ec_ctx *ctx, void *ptr)
{
    if (!ctx || !ptr) return;
    cudaSetDevice(ctx->device);
    cudaFreeHost(ptr);
}

int garage_ec_fill_random(garage_ec_ctx *ctx, uint8_t *dst_device, size_t len, uint64_t seed,
                          uint64_t offset, void *cuda_stream)
{
    if (!ctx || !dst_device || (len & 7) || (offset & 7) ||
        (reinterpret_cast<uintptr_t>(dst_device) & 7))
        return GARAGE_EC_E_INVALID;
    if (!len) return GARAGE_EC_OK;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    fill_random_kernel<<<ctx->sm_count * 8, 256, 0, (cudaStream_t)cuda_stream>>>(
        reinterpret_cast<unsigned long long *>(dst_device), len / 8, seed, offset / 8);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    return GARAGE_EC_OK;
}

// --------------------------------------------------------------------------- ENCODE
// pinned host memory the device addresses through the same pointer (cudaHostAlloc / cudaHostRegister under UVA)
static bool device_addressable_host(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost && a.devicePointer == p;
}

static int encode_host(garage_ec_ctx *ctx, const uint8_t *data, uint8_t *parity,
                       const uint32_t *shard_len, size_t stride, size_t n)
{
    const size_t k = ctx->k, m = ctx->m;
    HostPipeline p(ctx, n, k * stride);
    // pageable parity rows are copied piece by piece, as in reconstruct_host
    p.down.use_batch = device_addressable_host(parity);
    const size_t in_b = p.cs * k * stride, out_b = p.cs * m * stride;
    int rc = p.reserve(in_b + out_b, align_up(p.cs * 4, 16));
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_buf, data + ch.s0 * k * stride, ch.cnt * k * stride,
                                    cudaMemcpyHostToDevice, L.stream));
        const uint32_t *d_len = nullptr;
        if (shard_len) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small, shard_len + ch.s0, ch.cnt * 4, cudaMemcpyHostToDevice,
                                        L.stream));
            d_len = reinterpret_cast<const uint32_t *>(L.d_small);
        }
        int r = run_uniform(ctx, kModeEncode, L.d_buf, k * stride, L.d_buf + in_b, m * stride,
                            nullptr, d_len, stride, ch.cnt, L.stream);
        if (r) return r;
        // D2H: roundup16(shard_len) bytes of every parity row, never the caller's bytes past them (the lane buffer
        // holds stale data there); rows of stripes with shard_len == stride merge into one copy
        for (size_t s = ch.s0; s < ch.s0 + ch.cnt; s++) {
            const size_t bytes = shard_len ? align_up(shard_len[s], 16) : stride;
            for (size_t i = 0; i < m; i++)
                p.down.add(parity + (s * m + i) * stride, L.d_buf + in_b + ((s - ch.s0) * m + i) * stride, bytes);
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
    });
    return rc ? rc : p.drain();
}

int garage_ec_encode(garage_ec_ctx *ctx, const uint8_t *data, uint8_t *parity,
                     const uint32_t *shard_len, size_t stride, size_t n_stripes, int mem_kind,
                     void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE))
        return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!data || !parity) return GARAGE_EC_E_INVALID;
    if (!aligned16(data) || !aligned16(parity)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST && !shard_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_HOST) return encode_host(ctx, data, parity, shard_len, stride, n_stripes);
    return run_uniform(ctx, kModeEncode, data, (size_t)ctx->k * stride, parity, (size_t)ctx->m * stride,
                       nullptr, shard_len, stride, n_stripes, (cudaStream_t)cuda_stream);
}

// --------------------------------------------------------------------------- VERIFY
static int verify_host(garage_ec_ctx *ctx, const uint8_t *shards, uint32_t *mismatch,
                       const uint32_t *shard_len, size_t stride, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    HostPipeline p(ctx, n, tot * stride);
    SmallLayout sl;
    const size_t o_mm = sl.take(p.cs * 4), o_len = sl.take(p.cs * 4);
    int rc = p.reserve(p.cs * tot * stride, sl.bytes);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_buf, shards + ch.s0 * tot * stride, ch.cnt * tot * stride,
                                    cudaMemcpyHostToDevice, L.stream));
        uint32_t *d_mm = reinterpret_cast<uint32_t *>(L.d_small + o_mm);
        const uint32_t *d_len = nullptr;
        if (shard_len) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, shard_len + ch.s0, ch.cnt * 4,
                                        cudaMemcpyHostToDevice, L.stream));
            d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_len);
        }
        CU_TRY(ctx, cudaMemsetAsync(d_mm, 0, ch.cnt * 4, L.stream));
        int r = run_uniform(ctx, kModeVerify, L.d_buf, tot * stride, nullptr, 0, d_mm, d_len, stride,
                            ch.cnt, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(mismatch + ch.s0, d_mm, ch.cnt * 4, cudaMemcpyDeviceToHost, L.stream));
        return GARAGE_EC_OK;
    });
    return rc ? rc : p.drain();
}

int garage_ec_verify(garage_ec_ctx *ctx, const uint8_t *shards, uint32_t *mismatch,
                     const uint32_t *shard_len, size_t stride, size_t n_stripes, int mem_kind,
                     void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE))
        return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!shards || !mismatch) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST && !shard_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_HOST) return verify_host(ctx, shards, mismatch, shard_len, stride, n_stripes);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CU_TRY(ctx, cudaMemsetAsync(mismatch, 0, n_stripes * 4, st));
    return run_uniform(ctx, kModeVerify, shards, (size_t)(ctx->k + ctx->m) * stride, nullptr, 0, mismatch,
                       shard_len, stride, n_stripes, st);
}

// --------------------------------------------------------------------------- DEEP CHECK
// The block hash of every stripe (blake2sum_blocks_kernel, which also leaves L in shard_len and initialises mismatch),
// then the code's own verify launch with those lengths.  shard_len: n uint32 of device scratch.
static int run_deep_check(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *block_len, const uint8_t *hashes,
                          uint8_t *hash_bad, uint32_t *mismatch, uint32_t *shard_len, size_t stride, size_t n,
                          cudaStream_t st)
{
    BlockSumParams q;
    memset(&q, 0, sizeof(q));
    q.shards = shards;
    q.block_len = block_len;
    q.hashes = hashes;
    q.hash_bad = hash_bad;
    q.shard_len = shard_len;
    q.mismatch = mismatch;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    q.quantum = ctx->quantum;
    blake2sum_blocks_kernel<<<(unsigned)((n + kQuadThreads / 4 - 1) / (kQuadThreads / 4)), kQuadThreads, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "blake2sum_blocks_kernel launch");
    return run_uniform(ctx, kModeVerify, shards, (size_t)(ctx->k + ctx->m) * stride, nullptr, 0, mismatch, shard_len,
                       stride, n, st);
}

// HOST: chunks of whole stripes through the lanes; only roundup16(L) bytes of each shard go up
static int deep_check_host(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *block_len, const uint8_t *hashes,
                           uint8_t *hash_bad, uint32_t *mismatch, size_t stride, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    HostPipeline p(ctx, n, tot * stride);
    SmallLayout sl;
    const size_t o_blen = sl.take(p.cs * 4), o_hash = sl.take(p.cs * 32), o_sl = sl.take(p.cs * 4),
                 o_mm = sl.take(p.cs * 4), o_bad = sl.take(p.cs);
    int rc = p.reserve(p.cs * tot * stride, sl.bytes);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        for (size_t s = ch.s0; s < ch.s0 + ch.cnt; s++) {
            const size_t bytes = align_up(code_shard_len(ctx, block_len[s]), 16);
            for (size_t i = 0; i < tot; i++)
                p.up.add(L.d_buf + ((s - ch.s0) * tot + i) * stride, shards + (s * tot + i) * stride, bytes);
        }
        int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_blen, block_len + ch.s0, ch.cnt * 4, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_hash, hashes + ch.s0 * 32, ch.cnt * 32, cudaMemcpyHostToDevice, L.stream));
        uint32_t *d_mm = reinterpret_cast<uint32_t *>(L.d_small + o_mm);
        r = run_deep_check(ctx, L.d_buf, reinterpret_cast<const uint32_t *>(L.d_small + o_blen), L.d_small + o_hash,
                           L.d_small + o_bad, d_mm, reinterpret_cast<uint32_t *>(L.d_small + o_sl), stride, ch.cnt,
                           L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(hash_bad + ch.s0, L.d_small + o_bad, ch.cnt, cudaMemcpyDeviceToHost, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(mismatch + ch.s0, d_mm, ch.cnt * 4, cudaMemcpyDeviceToHost, L.stream));
        return GARAGE_EC_OK;
    });
    return rc ? rc : p.drain();
}

int garage_ec_deep_check(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *block_len, const uint8_t *hashes,
                         uint8_t *hash_bad, uint32_t *mismatch, size_t stride, size_t n_stripes, int mem_kind,
                         void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE)) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!shards || !block_len || !hashes || !hash_bad || !mismatch) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        // code_shard_len is a multiple of the code's framing unit, so a length that fits its stride is well framed
        for (size_t s = 0; s < n_stripes; s++)
            if (code_shard_len(ctx, block_len[s]) > stride) return GARAGE_EC_E_INVALID;
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        return deep_check_host(ctx, shards, block_len, hashes, hash_bad, mismatch, stride, n_stripes);
    }
    // the kernel reads the hashes as 8-byte words and the lengths / writes the mismatch words as 4-byte words
    if ((reinterpret_cast<uintptr_t>(hashes) & 7) || (reinterpret_cast<uintptr_t>(block_len) & 3) ||
        (reinterpret_cast<uintptr_t>(mismatch) & 3))
        return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    return with_stream_scratch(ctx, n_stripes * 4, st, [&](uint8_t *scratch) {
        return run_deep_check(ctx, shards, block_len, hashes, hash_bad, mismatch, reinterpret_cast<uint32_t *>(scratch),
                              stride, n_stripes, st);
    });
}

// --------------------------------------------------------------------------- RECONSTRUCT
// `stripes` != NULL: stripe s lives at stripes[s] (its k+m shards `stride` apart) instead of
// shards + s*(k+m)*stride -- the gather form used by batching front-ends whose callers each own
// a pinned slot (garage_ec_reconstruct_stripes)
static int reconstruct_host(garage_ec_ctx *ctx, uint8_t *shards, uint8_t *const *stripes, const uint8_t *present,
                            const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                            size_t stride, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    auto shard_at = [&](size_t s, size_t i) -> uint8_t * {
        return stripes ? stripes[s] + i * stride : shards + (s * tot + i) * stride;
    };
    // pinned (device-addressable) buffer: one chunk of all n stripes, in which the kernel reads the survivors from, and
    // writes the rebuilt shards into, the caller's buffer over PCIe -- nothing staged
    const bool zero_copy = !ctx->clay && !stripes && device_addressable_host(shards);
    HostPipeline p(ctx, n, zero_copy ? 0 : tot * stride);
    // cudaMemcpyBatchAsync gets pinned stripes only.  Batches of thousands of pageable survivor pieces (ragged
    // lengths, PB halves, Clay repair runs) crashed the process or faulted the context; pageable stripes are copied
    // piece by piece, which the driver stages through its own pinned buffers.
    bool pinned = !zero_copy;
    for (size_t s = 0; pinned && s < (stripes ? n : 1); s++) pinned = device_addressable_host(stripes ? stripes[s] : shards);
    p.up.use_batch = p.down.use_batch = pinned;
    SmallLayout sl;
    const size_t o_present = sl.take(p.cs * tot), o_want = sl.take(p.cs * tot), o_status = sl.take(p.cs * 4),
                 o_len = sl.take(p.cs * 4), o_plan = sl.take(plan_scratch_bytes(ctx, p.cs));
    int rc = p.reserve(zero_copy ? 0 : p.cs * tot * stride, sl.bytes);
    if (rc) return rc;
    int32_t *st_out = p.status_out(status);
    std::vector<uint8_t> rec_ok(p.cs);  // per stripe of the chunk: stripe_read_set succeeded
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t s0 = ch.s0, cnt = ch.cnt;
        uint8_t *d_sh = zero_copy ? shards : L.d_buf;
        // H2D: only the survivors the kernel reads (stripe_read_set) of stripes that have work to do
        for (size_t s = s0; s < s0 + cnt && !zero_copy; s++) {
            uint64_t hv = 0;
            bool work = false;  // a wanted shard is absent
            for (size_t i = 0; i < tot; i++) work |= !present[s * tot + i] && (!want || want[s * tot + i]);
            rec_ok[s - s0] = stripe_read_plan(ctx, present + s * tot, want ? want + s * tot : nullptr, &hv);
            if (!rec_ok[s - s0] || !work) continue;
            const size_t len = shard_len ? shard_len[s] : stride;
            for (size_t i = 0; i < tot; i++)
                for_each_read_piece(ctx, hv, i, len, stride, [&](size_t off, size_t bytes) {
                    p.up.add(d_sh + ((s - s0) * tot + i) * stride + off, shard_at(s, i) + off, bytes);
                });
        }
        int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, present + s0 * tot, cnt * tot,
                                    cudaMemcpyHostToDevice, L.stream));
        const uint8_t *d_want = nullptr;
        if (want) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_want, want + s0 * tot, cnt * tot,
                                        cudaMemcpyHostToDevice, L.stream));
            d_want = L.d_small + o_want;
        }
        const uint32_t *d_len = nullptr;
        if (shard_len) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, shard_len + s0, cnt * 4, cudaMemcpyHostToDevice,
                                        L.stream));
            d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_len);
        }
        r = run_reconstruct(ctx, d_sh, L.d_small + o_present, d_want, reinterpret_cast<int32_t *>(L.d_small + o_status),
                            d_len, stride, cnt, L.d_small + o_plan, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(st_out + s0, L.d_small + o_status, cnt * 4, cudaMemcpyDeviceToHost,
                                    L.stream));
        // D2H: exactly the shards that were rebuilt
        for (size_t s = s0; s < s0 + cnt && !zero_copy; s++) {
            const uint8_t *pr = present + s * tot;
            if (!rec_ok[s - s0]) continue;
            const size_t len = shard_len ? shard_len[s] : stride;
            const size_t bytes = align_up(len, 16);
            for (size_t i = 0; i < tot; i++) {
                if (pr[i] || (want && !want[s * tot + i])) continue;
                p.down.add(shard_at(s, i), d_sh + ((s - s0) * tot + i) * stride, bytes);
            }
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
    });
    if (!rc) rc = p.drain();
    if (rc) return rc;
    for (size_t s = 0; s < n; s++)
        if (st_out[s] != 0) return GARAGE_EC_E_UNRECOVERABLE;
    return GARAGE_EC_OK;
}

int garage_ec_reconstruct(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present,
                          const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                          size_t stride, size_t n_stripes, int mem_kind, void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE))
        return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!shards || !present) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST && !shard_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_HOST)
        return reconstruct_host(ctx, shards, nullptr, present, want, status, shard_len, stride, n_stripes);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    return with_stream_scratch(ctx, plan_scratch_bytes(ctx, n_stripes), st, [&](uint8_t *scratch) {
        return run_reconstruct(ctx, shards, present, want, status, shard_len, stride, n_stripes, scratch, st);
    });
}

int garage_ec_reconstruct_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes, const uint8_t *present,
                                  const uint8_t *want, int32_t *status, const uint32_t *shard_len, size_t stride,
                                  size_t n_stripes)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!stripes || !present) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n_stripes; s++) {
        if (!stripes[s]) return GARAGE_EC_E_INVALID;
        if (!aligned16(stripes[s])) return GARAGE_EC_E_ALIGN;
    }
    if (!shard_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return reconstruct_host(ctx, nullptr, stripes, present, want, status, shard_len, stride, n_stripes);
}

// --------------------------------------------------------------------------- RECONSTRUCT BY SEGMENT (DESIGN.md 2.10)
}  // extern "C"

namespace {

// Device scratch of run_segments for n stripes: unit plans | apply counter (16 B) | unit presence | unit want |
// unit status | work list
struct SegScratch {
    size_t plan, counter, present, want, ustatus, units, bytes;
    SegScratch(const garage_ec_ctx *ctx, size_t n)
    {
        const size_t nu = n * units_per_stripe(ctx->pb), tot = ctx->k + ctx->m;
        plan = 0;
        counter = nu * sizeof(StripePlan);
        present = counter + 16;
        want = present + align_up(nu * tot, 16);
        ustatus = want + align_up(nu * tot, 16);
        units = ustatus + nu * 4;
        bytes = units + align_up((1 + nu) * 4, 16);
    }
};

// n * U unit rows of k+m shards must stay below 2^32 (plan rows and work-list ids are 32-bit)
bool seg_count_ok(const garage_ec_ctx *ctx, size_t n)
{
    return (unsigned long long)n * units_per_stripe(ctx->pb) * (ctx->k + ctx->m) < (1ull << 32);
}

// Device-resident reconstruct by unit.  scratch: SegScratch(ctx, n).bytes of device memory.
int run_segments(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *seg_present, const uint8_t *want, int32_t *status,
                 const uint32_t *shard_len, size_t stride, size_t n, uint8_t *scratch, cudaStream_t st)
{
    const SegScratch sc(ctx, n);
    const size_t nu = n * units_per_stripe(ctx->pb), tot = ctx->k + ctx->m;
    StripePlan *plan = reinterpret_cast<StripePlan *>(scratch + sc.plan);
    uint32_t *counter = reinterpret_cast<uint32_t *>(scratch + sc.counter);
    uint32_t *units = reinterpret_cast<uint32_t *>(scratch + sc.units);
    int32_t *ustatus = reinterpret_cast<int32_t *>(scratch + sc.ustatus);
    cudaError_t e = cudaMemsetAsync(units, 0, sizeof(uint32_t), st);
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaMemsetAsync(units)");
    UnitParams u;
    memset(&u, 0, sizeof(u));
    u.seg_present = seg_present;
    u.want = want;
    u.shard_len = shard_len;
    u.unit_present = scratch + sc.present;
    u.unit_want = want ? scratch + sc.want : nullptr;
    u.unit_status = ustatus;
    u.plan = plan;
    u.status = status;
    u.units = units;
    u.n = (uint32_t)n;
    u.tot = (uint32_t)tot;
    u.stride = (uint32_t)stride;
    u.pb = ctx->pb ? 1u : 0u;
    unit_prep_kernel<<<(unsigned)((nu * tot + 255) / 256), 256, 0, st>>>(u);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "unit_prep_kernel launch");
    // the one survivor planner, over unit rows; shard_len NULL with stride 0: unit_prep_kernel already judged the
    // stripe's geometry, and a malformed stripe's units are all present
    PlanParams q;
    memset(&q, 0, sizeof(q));
    q.present = scratch + sc.present;
    q.want = u.unit_want;
    q.status = ustatus;
    q.plan = plan;
    q.counter = counter;
    q.n = (uint32_t)nu;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.l = (uint32_t)ctx->l;
    q.pb = ctx->pb ? 1u : 0u;
    memcpy(q.P, ctx->P, (size_t)ctx->k * ctx->m);
    plan_kernel<<<(unsigned)((nu + kPlanWarps - 1) / kPlanWarps), kPlanWarps * 32, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "plan_kernel launch");
    unit_fold_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(u);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "unit_fold_kernel launch");

    TimedLaunch tl(ctx, st);
    const int nout = ctx->pb ? 2 * ctx->m : ctx->m;
    for (int r0 = 0; r0 < nout; r0 += kRowsPerPass) {
        if (r0 > 0) {
            e = cudaMemsetAsync(counter, 0, sizeof(uint32_t), st);
            if (e != cudaSuccess) return set_cuda_error(ctx, e, "cudaMemsetAsync(counter)");
        }
        ApplyParams p;
        memset(&p, 0, sizeof(p));
        p.src = shards;
        p.dst = shards;
        p.src_pitch = p.dst_pitch = tot * stride;
        p.shard_len = shard_len;
        p.plan = plan;
        p.units = units;
        p.counter = counter;
        p.stride = (uint32_t)stride;
        p.n = (uint32_t)n;
        p.k = (uint32_t)(ctx->pb ? 2 * ctx->k : ctx->k);
        p.half = ctx->pb ? 1u : 0u;
        p.row_off = (uint32_t)r0;
        p.row_bytes = 128;
        e = launch_apply<kModeUnits>(ctx, p, st);
        if (e != cudaSuccess) return set_cuda_error(ctx, e, "rs_apply_kernel<units> launch");
    }
    return GARAGE_EC_OK;
}

// HOST form (garage_ec_reconstruct_segments(MEM_HOST) / _stripes): the chunk pipeline of reconstruct_host, by unit.  Up:
// the read-set pieces of every unit that has work, of stripes whose every unit is recoverable.  Down: the rebuilt units
// of those stripes (RS / LRC: with the zero tail of the shard's last unit).
int segments_host(garage_ec_ctx *ctx, uint8_t *shards, uint8_t *const *stripes, const uint8_t *seg_present,
                  const uint8_t *want, int32_t *status, const uint32_t *shard_len, size_t stride, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    const uint32_t U = units_per_stripe(ctx->pb);
    auto shard_at = [&](size_t s, size_t i) -> uint8_t * {
        return stripes ? stripes[s] + i * stride : shards + (s * tot + i) * stride;
    };
    const bool zero_copy = !stripes && device_addressable_host(shards);
    HostPipeline p(ctx, n, zero_copy ? 0 : tot * stride);
    bool pinned = !zero_copy;
    for (size_t s = 0; pinned && s < (stripes ? n : 1); s++) pinned = device_addressable_host(stripes ? stripes[s] : shards);
    p.up.use_batch = p.down.use_batch = pinned;
    SmallLayout sl;
    const SegScratch sc(ctx, p.cs);
    const size_t o_present = sl.take(p.cs * tot), o_want = sl.take(p.cs * tot), o_status = sl.take(p.cs * 4),
                 o_len = sl.take(p.cs * 4), o_scratch = sl.take(sc.bytes);
    int rc = p.reserve(zero_copy ? 0 : p.cs * tot * stride, sl.bytes);
    if (rc) return rc;
    int32_t *st_out = p.status_out(status);
    // per unit of the chunk: the read plan (0 = no work or a stripe that will not be rebuilt)
    std::vector<uint64_t> rows(p.cs * U);
    std::vector<uint8_t> has_work(p.cs * U);
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t s0 = ch.s0, cnt = ch.cnt;
        uint8_t *d_sh = zero_copy ? shards : L.d_buf;
        for (size_t s = s0; s < s0 + cnt; s++) {
            const uint32_t len = shard_len ? shard_len[s] : (uint32_t)stride;
            const uint8_t *sp = seg_present + s * tot, *wn = want ? want + s * tot : nullptr;
            bool ok = true;
            for (uint32_t g = 0; g < U; g++) {
                uint64_t hv = 0;
                bool work = false;  // a wanted shard is absent in this unit
                ok &= unit_read_plan(ctx, sp, wn, len, g, &hv, &work);
                rows[(s - s0) * U + g] = hv;
                has_work[(s - s0) * U + g] = work;
            }
            if (!ok)
                for (uint32_t g = 0; g < U; g++) has_work[(s - s0) * U + g] = 0;
        }
        // H2D: the pieces of each unit's read set
        for (size_t s = s0; s < s0 + cnt && !zero_copy; s++) {
            const uint32_t len = shard_len ? shard_len[s] : (uint32_t)stride;
            for (uint32_t g = 0; g < U; g++) {
                if (!has_work[(s - s0) * U + g]) continue;
                for (size_t i = 0; i < tot; i++)
                    for_each_unit_piece(ctx, rows[(s - s0) * U + g], i, len, g, [&](size_t off, size_t ulen) {
                        p.up.add(d_sh + ((s - s0) * tot + i) * stride + off, shard_at(s, i) + off, align_up(ulen, 16));
                    });
            }
        }
        int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, seg_present + s0 * tot, cnt * tot, cudaMemcpyHostToDevice,
                                    L.stream));
        const uint8_t *d_want = nullptr;
        if (want) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_want, want + s0 * tot, cnt * tot, cudaMemcpyHostToDevice, L.stream));
            d_want = L.d_small + o_want;
        }
        const uint32_t *d_len = nullptr;
        if (shard_len) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, shard_len + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_len);
        }
        r = run_segments(ctx, d_sh, L.d_small + o_present, d_want, reinterpret_cast<int32_t *>(L.d_small + o_status), d_len,
                         stride, cnt, L.d_small + o_scratch, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(st_out + s0, L.d_small + o_status, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
        // D2H: exactly the rebuilt units
        for (size_t s = s0; s < s0 + cnt && !zero_copy; s++) {
            const uint32_t len = shard_len ? shard_len[s] : (uint32_t)stride;
            const uint8_t *sp = seg_present + s * tot, *wn = want ? want + s * tot : nullptr;
            for (uint32_t g = 0; g < U; g++) {
                if (!has_work[(s - s0) * U + g]) continue;
                uint32_t base, ulen;
                unit_columns(len, g, ctx->pb, &base, &ulen);
                for (size_t i = 0; i < tot; i++) {
                    if (unit_present(sp[i], len, g, ctx->pb) || (wn && !wn[i])) continue;
                    for (unsigned h = 0; h < (ctx->pb ? 2u : 1u); h++) {
                        const size_t off = base + h * (size_t)(len / 2);
                        p.down.add(shard_at(s, i) + off, d_sh + ((s - s0) * tot + i) * stride + off, align_up(ulen, 16));
                    }
                }
            }
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
    });
    if (!rc) rc = p.drain();
    if (rc) return rc;
    for (size_t s = 0; s < n; s++)
        if (st_out[s] != 0) return GARAGE_EC_E_UNRECOVERABLE;
    return GARAGE_EC_OK;
}

// every stripe's L within the stride and, for PB, a multiple of 128 (HOST forms check before any GPU work)
bool seg_lens_ok(const garage_ec_ctx *ctx, const uint32_t *shard_len, size_t stride, size_t n)
{
    const size_t unit = ctx->pb ? 128 : 1;
    if (!shard_len) return stride % unit == 0;
    for (size_t s = 0; s < n; s++)
        if (shard_len[s] % unit || shard_len[s] > stride) return false;
    return true;
}

}  // namespace

extern "C" {

int garage_ec_reconstruct_segments(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *seg_present, const uint8_t *want,
                                   int32_t *status, const uint32_t *shard_len, size_t stride, size_t n_stripes,
                                   int mem_kind, void *cuda_stream)
{
    if (!ctx || ctx->clay || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE))
        return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!shards || !seg_present || !seg_count_ok(ctx, n_stripes)) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST && !seg_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_HOST)
        return segments_host(ctx, shards, nullptr, seg_present, want, status, shard_len, stride, n_stripes);
    cudaStream_t st = (cudaStream_t)cuda_stream;
    return with_stream_scratch(ctx, SegScratch(ctx, n_stripes).bytes, st, [&](uint8_t *scratch) {
        return run_segments(ctx, shards, seg_present, want, status, shard_len, stride, n_stripes, scratch, st);
    });
}

int garage_ec_reconstruct_segments_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes, const uint8_t *seg_present,
                                           const uint8_t *want, int32_t *status, const uint32_t *shard_len,
                                           size_t stride, size_t n_stripes)
{
    if (!ctx || ctx->clay) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!stripes || !seg_present || !seg_count_ok(ctx, n_stripes)) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n_stripes; s++) {
        if (!stripes[s]) return GARAGE_EC_E_INVALID;
        if (!aligned16(stripes[s])) return GARAGE_EC_E_ALIGN;
    }
    if (!seg_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return segments_host(ctx, nullptr, stripes, seg_present, want, status, shard_len, stride, n_stripes);
}

// --------------------------------------------------------------------------- RANGED READS (DESIGN.md 2.5)
}  // extern "C"
namespace {

// One request's window (rs_kernels.cuh) and the survivor plan of its absent touched data shards.  GARAGE_EC_E_INVALID
// for a range past the block or a shard length past `stride`.
struct RangeReq {
    RangeWindow r{0, 0, 0, 0, 0};
    uint64_t halves = 0;
    bool ok = true;  // the absent touched data shards can be rebuilt
};
int range_request(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t block_len, uint32_t off,
                         uint32_t len, uint64_t stride, RangeReq *q)
{
    const uint64_t L = code_shard_len(ctx, block_len);
    if ((uint64_t)off + len > block_len || L > stride) return GARAGE_EC_E_INVALID;
    q->r = range_window((uint32_t)L, range_unit((uint32_t)L, ctx->pb, ctx->clay ? ctx->cg.alpha : 1), off, len, present);
    if (!q->r.w) return GARAGE_EC_OK;
    uint8_t want[kMaxK + kMaxM] = {0};
    for (int j = 0; j < ctx->k; j++) want[j] = (uint8_t)((q->r.want >> j) & 1);
    q->ok = stripe_read_plan(ctx, present, want, &q->halves);
    return GARAGE_EC_OK;
}
// The range's bytes in each touched data shard j, as f(j, offset c in the shard, offset in the range, bytes)
template <class F>
void for_each_range_piece(const RangeWindow &r, uint64_t off, uint64_t len, F &&f)
{
    for (uint64_t j = r.L ? off / r.L : 0, end = off + len; len && j * r.L < end; j++) {
        const uint64_t base = j * r.L, c0 = std::max(off, base) - base, c1 = std::min(end, base + r.L) - base;
        f((size_t)j, (size_t)c0, (size_t)(base + c0 - off), (size_t)(c1 - c0));
    }
}
// The window runs of shard i that the sub-stripe decode reads -- the pieces of stripe_read_plan cut to the window --
// as f(offset in the shard, offset in the sub-stripe's shard, bytes)
template <class F>
void for_each_window_run(const garage_ec_ctx *ctx, const RangeReq &q, size_t i, F &&f)
{
    const RangeWindow &r = q.r;
    for_each_read_piece(ctx, q.halves, i, r.L, r.L, [&](size_t off, size_t bytes) {
        for (size_t z = off / r.unit; z * r.unit < off + bytes; z++) f(z * r.unit + r.w0, z * r.w, (size_t)r.w);
    });
}
// Rebuilt bytes [c0, c0 + bytes) of an absent data shard, cut at run edges, as f(offset in the sub-stripe's shard,
// offset from c0, bytes)
template <class F>
void for_each_rebuilt_piece(const RangeWindow &r, size_t c0, size_t bytes, F &&f)
{
    for (size_t c = c0, e = c0 + bytes; c < e;) {
        const size_t z = c / r.unit, ce = std::min(e, (z + 1) * r.unit);
        f(z * r.w + (c - z * r.unit) - r.w0, c - c0, ce - c);
        c = ce;
    }
}


// The unmerged runs garage_ec_range_plan names for one request, appended to `runs`; *needs_gpu |= an absent touched
// data shard.
int range_runs(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t block_len, uint32_t offset, uint32_t len,
               std::vector<garage_ec_range> &runs, int *needs_gpu)
{
    RangeReq q;
    int rc = range_request(ctx, present, block_len, offset, len, UINT64_MAX, &q);
    if (rc) return rc;
    if (q.r.w) *needs_gpu = 1;
    if (!q.ok) return GARAGE_EC_E_UNRECOVERABLE;
    for_each_range_piece(q.r, offset, len, [&](size_t j, size_t c, size_t, size_t bytes) {
        if (present[j]) runs.push_back(garage_ec_range{(uint32_t)j, (uint32_t)c, (uint32_t)bytes});
    });
    for (int i = 0; q.r.w && i < ctx->k + ctx->m; i++)
        for_each_window_run(ctx, q, (size_t)i, [&](size_t off, size_t, size_t bytes) {
            runs.push_back(garage_ec_range{(uint32_t)i, (uint32_t)off, (uint32_t)bytes});
        });
    return GARAGE_EC_OK;
}

// runs in shard then offset order, overlapping or adjacent runs merged, into ranges[0, cap)
int merge_runs(std::vector<garage_ec_range> &runs, garage_ec_range *ranges, size_t cap, size_t *n_ranges)
{
    std::sort(runs.begin(), runs.end(), [](const garage_ec_range &a, const garage_ec_range &b) {
        return a.shard != b.shard ? a.shard < b.shard : a.offset < b.offset;
    });
    std::vector<garage_ec_range> merged;
    for (const garage_ec_range &r : runs) {
        garage_ec_range *b = merged.empty() ? nullptr : &merged.back();
        if (b && b->shard == r.shard && r.offset <= b->offset + b->len)  // overlapping or adjacent: merged
            b->len = std::max(b->offset + b->len, r.offset + r.len) - b->offset;
        else
            merged.push_back(r);
    }
    for (size_t x = 0; x < merged.size() && x < cap; x++) ranges[x] = merged[x];
    *n_ranges = merged.size();
    return merged.size() > cap ? GARAGE_EC_E_INVALID : GARAGE_EC_OK;
}

}  // namespace
extern "C" {

int garage_ec_segment_read_ranges(const garage_ec_ctx *ctx, const uint8_t *seg_present, const uint8_t *want,
                                  uint32_t shard_len, garage_ec_range *ranges, size_t cap, size_t *n_ranges)
{
    if (!ctx || !seg_present || !n_ranges || (cap && !ranges)) return GARAGE_EC_E_INVALID;
    *n_ranges = 0;
    if (ctx->clay || (ctx->pb && shard_len % 128)) return GARAGE_EC_E_INVALID;
    std::vector<garage_ec_range> runs;
    for (uint32_t g = 0; g < units_per_stripe(ctx->pb); g++) {
        uint64_t hv = 0;
        bool work = false;
        if (!unit_read_plan(ctx, seg_present, want, shard_len, g, &hv, &work)) return GARAGE_EC_E_UNRECOVERABLE;
        for (int i = 0; work && i < ctx->k + ctx->m; i++)
            for_each_unit_piece(ctx, hv, (size_t)i, shard_len, g, [&](size_t off, size_t bytes) {
                runs.push_back(garage_ec_range{(uint32_t)i, (uint32_t)off, (uint32_t)bytes});
            });
    }
    return merge_runs(runs, ranges, cap, n_ranges);
}

int garage_ec_range_plan(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t block_len, uint32_t offset,
                         uint32_t len, garage_ec_range *ranges, size_t cap, size_t *n_ranges, int *needs_gpu)
{
    if (!ctx || !present || !n_ranges || (cap && !ranges)) return GARAGE_EC_E_INVALID;
    *n_ranges = 0;
    if (needs_gpu) *needs_gpu = 0;
    std::vector<garage_ec_range> runs;
    int gpu = 0;
    const int rc = range_runs(ctx, present, block_len, offset, len, runs, &gpu);
    if (needs_gpu) *needs_gpu = gpu;
    if (rc) return rc;
    return merge_runs(runs, ranges, cap, n_ranges);
}

// HOST ranged decode.  stripes / outs != NULL: the gather form (garage_ec_decode_range_stripes).  Only the window runs
// of the plan go up, packed into sub-stripes; only the rebuilt range bytes come down; present range bytes are
// copied on the host.
static int decode_range_host(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *const *stripes,
                             const uint8_t *present, const uint32_t *block_len, const uint32_t *offset,
                             const uint32_t *len, size_t stride, uint8_t *out, size_t out_stride, uint8_t *const *outs,
                             int32_t *status, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    auto shard_at = [&](size_t s, size_t i) -> const uint8_t * {
        return stripes ? stripes[s] + i * stride : shards + (s * tot + i) * stride;
    };
    auto out_at = [&](size_t s) -> uint8_t * { return outs ? outs[s] : out + s * out_stride; };
    std::vector<RangeReq> rq(n);
    std::vector<size_t> need;
    size_t sub_max = 16;
    bool any_bad = false, pinned = true;
    for (size_t s = 0; s < n; s++) {
        int rc = range_request(ctx, present + s * tot, block_len[s], offset[s], len[s], stride, &rq[s]);
        if (rc) return rc;
        if (len[s] && !out_at(s)) return GARAGE_EC_E_INVALID;
    }
    for (size_t s = 0; s < n; s++) {
        if (status) status[s] = rq[s].ok ? 0 : GARAGE_EC_E_UNRECOVERABLE;
        any_bad |= !rq[s].ok;
        if (!rq[s].ok || !rq[s].r.w) continue;
        need.push_back(s);
        sub_max = std::max<size_t>(sub_max, (size_t)(rq[s].r.L / rq[s].r.unit) * rq[s].r.w);
        pinned = pinned && device_addressable_host(shard_at(s, 0)) && device_addressable_host(out_at(s));
    }
    const size_t sub_stride = align_up(sub_max, 16);
    std::vector<int32_t> dec_status(need.size(), 0);  // the decode's own verdicts (outlives the pipeline's copies)
    HostPipeline p(ctx, need.size(), tot * sub_stride);
    // pageable pieces go one by one (see reconstruct_host)
    p.up.use_batch = p.down.use_batch = pinned;
    const size_t cs = p.cs;
    SmallLayout sl;
    const size_t o_present = sl.take(cs * tot), o_want = sl.take(cs * tot), o_status = sl.take(cs * 4),
                 o_len = sl.take(cs * 4), o_plan = sl.take(plan_scratch_bytes(ctx, cs));
    // pageable staging per lane: sub-stripe length | present | want
    int rc = p.reserve(cs * tot * sub_stride, sl.bytes, cs * 4 + 2 * cs * tot);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t q0 = ch.s0, cnt = ch.cnt;
        uint32_t *hl = reinterpret_cast<uint32_t *>(ch.host);
        uint8_t *hp = ch.host + cs * 4, *hw = hp + cs * tot;
        for (size_t q = 0; q < cnt; q++) {
            const size_t s = need[q0 + q];
            const RangeReq &r = rq[s];
            memcpy(hp + q * tot, present + s * tot, tot);
            for (size_t i = 0; i < tot; i++) hw[q * tot + i] = (uint8_t)((r.r.want >> i) & 1);
            hl[q] = (r.r.L / r.r.unit) * r.r.w;
            uint8_t *d_st = L.d_buf + q * tot * sub_stride;
            for (size_t i = 0; i < tot; i++)
                for_each_window_run(ctx, r, i, [&](size_t so, size_t sub, size_t bytes) {
                    p.up.add(d_st + i * sub_stride + sub, shard_at(s, i) + so, bytes);
                });
        }
        int e = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (e) return e;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, hp, cnt * tot, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_want, hw, cnt * tot, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, hl, cnt * 4, cudaMemcpyHostToDevice, L.stream));
        e = run_reconstruct(ctx, L.d_buf, L.d_small + o_present, L.d_small + o_want,
                            reinterpret_cast<int32_t *>(L.d_small + o_status),
                            reinterpret_cast<const uint32_t *>(L.d_small + o_len), sub_stride, cnt, L.d_small + o_plan,
                            L.stream);
        if (e) return e;
        CU_TRY(ctx, cudaMemcpyAsync(dec_status.data() + q0, L.d_small + o_status, cnt * 4, cudaMemcpyDeviceToHost,
                                    L.stream));
        // D2H: the rebuilt range bytes only, straight into the caller's output
        for (size_t q = 0; q < cnt; q++) {
            const size_t s = need[q0 + q];
            const RangeReq &r = rq[s];
            for_each_range_piece(r.r, offset[s], len[s], [&](size_t j, size_t c, size_t pos, size_t bytes) {
                if (present[s * tot + j]) return;
                const uint8_t *d_sh = L.d_buf + (q * tot + j) * sub_stride;
                for_each_rebuilt_piece(r.r, c, bytes, [&](size_t sub, size_t rel, size_t b) {
                    p.down.add(out_at(s) + pos + rel, d_sh + sub, b);
                });
            });
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
    });
    if (rc) return rc;
    // the present range bytes, while the GPU works
    for (size_t s = 0; s < n; s++) {
        if (!rq[s].ok) continue;
        for_each_range_piece(rq[s].r, offset[s], len[s], [&](size_t j, size_t c, size_t pos, size_t bytes) {
            if (present[s * tot + j]) memcpy(out_at(s) + pos, shard_at(s, j) + c, bytes);
        });
    }
    rc = p.drain();
    if (rc) return rc;
    for (size_t q = 0; q < need.size(); q++)  // the host plan said yes; the decode's verdict has the last word
        if (dec_status[q]) {
            if (status) status[need[q]] = dec_status[q];
            any_bad = true;
        }
    return any_bad ? GARAGE_EC_E_UNRECOVERABLE : GARAGE_EC_OK;
}

// DEVICE ranged decode: geometry, pack the window runs into sub-stripes, the code's own decode on them, join.  Request
// s reads stripe s >> shift of `shards`; `sc` holds a RangeScratch.
struct RangeScratch {
    size_t o_sub, o_geo, o_len, o_want, o_st, o_plan, bytes;
    RangeScratch(const garage_ec_ctx *ctx, size_t n, size_t stride)
    {
        const size_t tot = ctx->k + ctx->m;
        SmallLayout sl;
        o_sub = sl.take(n * tot * stride);
        o_geo = sl.take(n * 16);
        o_len = sl.take(n * 4);
        o_want = sl.take(n * tot);
        o_st = sl.take(n * 4);
        o_plan = sl.take(plan_scratch_bytes(ctx, n));
        bytes = sl.bytes;
    }
};
static int run_decode_range(garage_ec_ctx *ctx, const uint8_t *shards, uint32_t shift, const uint8_t *present,
                            const uint32_t *block_len, const uint32_t *offset, const uint32_t *len, size_t stride,
                            uint8_t *out, size_t out_stride, int32_t *status, size_t n, uint8_t *sc, cudaStream_t st)
{
    const size_t pitch = (size_t)(ctx->k + ctx->m) * stride;
    const RangeScratch rs(ctx, n, stride);
    const size_t o_sub = rs.o_sub, o_geo = rs.o_geo, o_len = rs.o_len, o_want = rs.o_want, o_st = rs.o_st,
                 o_plan = rs.o_plan;
    RangeParams q;
    memset(&q, 0, sizeof(q));
    q.shards = shards;
    q.sub = sc + o_sub;
    q.present = present;
    q.block_len = block_len;
    q.offset = offset;
    q.len = len;
    q.out = out;
    q.geo = reinterpret_cast<uint4 *>(sc + o_geo);
    q.sub_len = reinterpret_cast<uint32_t *>(sc + o_len);
    q.want = sc + o_want;
    q.plan_status = reinterpret_cast<const int32_t *>(sc + o_st);
    q.status = status;
    q.pitch = pitch;
    q.out_stride = out_stride;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    q.quantum = ctx->quantum;
    q.alpha = ctx->clay ? (uint32_t)ctx->cg.alpha : 1u;
    q.pb = ctx->pb ? 1u : 0u;
    q.shift = shift;
    const unsigned per_req = (unsigned)std::min<size_t>(n, (size_t)ctx->sm_count * 8);
    range_geo_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 4), 256, 0, st>>>(q);
    range_pack_kernel<<<per_req, 256, 0, st>>>(q);
    ctx->launches.fetch_add(2, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    int r = run_reconstruct(ctx, q.sub, present, q.want, reinterpret_cast<int32_t *>(sc + o_st), q.sub_len, stride, n,
                            sc + o_plan, st);
    if (r) return r;
    range_join_kernel<<<per_req, 256, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    return GARAGE_EC_OK;
}
static int decode_range_device(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present,
                               const uint32_t *block_len, const uint32_t *offset, const uint32_t *len, size_t stride,
                               uint8_t *out, size_t out_stride, int32_t *status, size_t n, cudaStream_t st)
{
    return with_stream_scratch(ctx, RangeScratch(ctx, n, stride).bytes, st, [&](uint8_t *sc) -> int {
        return run_decode_range(ctx, shards, 0, present, block_len, offset, len, stride, out, out_stride, status, n, sc,
                                st);
    });
}

int garage_ec_decode_range(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present, const uint32_t *block_len,
                           const uint32_t *offset, const uint32_t *len, size_t stride, uint8_t *out, size_t out_stride,
                           int32_t *status, size_t n, int mem_kind, void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE)) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, ctx->k + ctx->m);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!shards || !present || !block_len || !offset || !len || !out) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_HOST)
        return decode_range_host(ctx, shards, nullptr, present, block_len, offset, len, stride, out, out_stride, nullptr,
                                 status, n);
    if (!aligned16(out) || (out_stride & 15)) return GARAGE_EC_E_ALIGN;
    return decode_range_device(ctx, shards, present, block_len, offset, len, stride, out, out_stride, status, n,
                               (cudaStream_t)cuda_stream);
}

int garage_ec_decode_range_stripes(garage_ec_ctx *ctx, const uint8_t *const *stripes, const uint8_t *present,
                                   const uint32_t *block_len, const uint32_t *offset, const uint32_t *len, size_t stride,
                                   uint8_t *const *outs, int32_t *status, size_t n)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, ctx->k + ctx->m);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!stripes || !present || !block_len || !offset || !len || !outs) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n; s++) {
        if (!stripes[s]) return GARAGE_EC_E_INVALID;
        if (!aligned16(stripes[s])) return GARAGE_EC_E_ALIGN;
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return decode_range_host(ctx, nullptr, stripes, present, block_len, offset, len, stride, nullptr, 0, outs, status, n);
}

// --------------------------------------------------------------------------- SHARD SUMS
static int run_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *expect, const uint32_t *shard_len,
                    size_t stride, size_t n_shards, int per_stripe, uint8_t *sums, uint8_t *bad, cudaStream_t st,
                    int out_per_stripe = 0, int out_off = 0, const uint8_t *shards2 = nullptr, size_t n_shards2 = 0,
                    int per_stripe2 = 1, int out_off2 = 0)
{
    SumParams q;
    memset(&q, 0, sizeof(q));
    q.base = shards;
    q.shard_len = shard_len;
    q.expect = expect;
    q.sums = sums;
    q.bad = bad;
    q.stride = (uint32_t)stride;
    q.per_stripe = (uint32_t)per_stripe;
    q.n_shards = (uint32_t)(n_shards + n_shards2);
    q.out_per_stripe = (uint32_t)(out_per_stripe ? out_per_stripe : per_stripe);
    q.out_off = (uint32_t)out_off;
    q.base2 = shards2;
    q.n_first = (uint32_t)n_shards;
    q.per_stripe2 = (uint32_t)per_stripe2;
    q.out_off2 = (uint32_t)out_off2;
    n_shards += n_shards2;
    // few shards: four lanes per shard (4x the parallelism, but the quad shuffles make it
    // LSU-bound: measured 5.4 ms vs 7.6 ms at 18 432 shards and 6.0 vs 5.7 ms at 28 672);
    // from ~24 000 shards on one thread per shard keeps the schedulers busy enough
    if (ctx->sum_kind.load(std::memory_order_relaxed) == GARAGE_EC_SUM_ADLER8) {
        // one warp per (shard, segment), 8 warps per block, persistent grid
        if (n_shards >= (1u << 29)) return GARAGE_EC_E_INVALID;
        if (expect && bad) {
            // segments OR their verdict into the shard's flag: clear the flags of this launch first.  Flags of
            // one launch are contiguous when out_per_stripe == per_stripe (check_sums / scrub_repair)
            const size_t nflags = (n_shards / (size_t)q.per_stripe) * q.out_per_stripe;
            cudaError_t e0 = cudaMemsetAsync(bad, 0, nflags, st);
            if (e0 != cudaSuccess) return set_cuda_error(ctx, e0, "cudaMemsetAsync(bad)");
        }
        const unsigned blocks = (unsigned)std::min<size_t>(n_shards, (size_t)ctx->sm_count * 8);
        adler8_shards_kernel<<<blocks, 256, 0, st>>>(q);
    } else if (n_shards < 24000)
        blake2sum_shards_quad_kernel<<<(unsigned)((n_shards + kQuadThreads / 4 - 1) / (kQuadThreads / 4)), kQuadThreads, 0,
                                       st>>>(q);
    else
        blake2sum_shards_kernel<<<(unsigned)((n_shards + 127) / 128), 128, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(ctx, e, "blake2sum_shards_kernel launch");
    return GARAGE_EC_OK;
}

static int sums_common(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *expect, const uint32_t *shard_len,
                       size_t stride, size_t n, int per, uint8_t *sums_out, uint8_t *bad_out, int mem_kind,
                       void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE)) return GARAGE_EC_E_INVALID;
    if (per < 1 || per > kMaxK + kMaxM) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, per);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!shards || (!sums_out && !bad_out)) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (n * (size_t)per > 0xffffffffull) return GARAGE_EC_E_INVALID;
    if (mem_kind == GARAGE_EC_MEM_HOST && shard_len)  // tags of any length are legal, but not past the stride
        for (size_t s = 0; s < n; s++)
            if (shard_len[s] > stride) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_DEVICE)
        return run_sums(ctx, shards, expect, shard_len, stride, n * per, per, sums_out, bad_out,
                        (cudaStream_t)cuda_stream);
    // HOST: chunked through the lanes (H2D shards [+ expect], kernel, D2H sums / bad flags)
    HostPipeline p(ctx, n, (size_t)per * stride);
    SmallLayout sl;
    const size_t o_len = sl.take(p.cs * 4), o_exp = sl.take(p.cs * per * 32), o_sum = sl.take(p.cs * per * 32),
                 o_bad = sl.take(p.cs * per);
    rc = p.reserve(p.cs * per * stride, sl.bytes);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t s0 = ch.s0, cnt = ch.cnt;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_buf, shards + s0 * per * stride, cnt * per * stride, cudaMemcpyHostToDevice,
                                    L.stream));
        const uint32_t *d_len = nullptr;
        if (shard_len) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, shard_len + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_len);
        }
        const uint8_t *d_exp = nullptr;
        if (expect) {
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_exp, expect + s0 * per * 32, cnt * per * 32,
                                        cudaMemcpyHostToDevice, L.stream));
            d_exp = L.d_small + o_exp;
        }
        int r = run_sums(ctx, L.d_buf, d_exp, d_len, stride, cnt * per, per, sums_out ? L.d_small + o_sum : nullptr,
                         bad_out ? L.d_small + o_bad : nullptr, L.stream);
        if (r) return r;
        if (sums_out)
            CU_TRY(ctx, cudaMemcpyAsync(sums_out + s0 * per * 32, L.d_small + o_sum, cnt * per * 32,
                                        cudaMemcpyDeviceToHost, L.stream));
        if (bad_out)
            CU_TRY(ctx, cudaMemcpyAsync(bad_out + s0 * per, L.d_small + o_bad, cnt * per, cudaMemcpyDeviceToHost,
                                        L.stream));
        return GARAGE_EC_OK;
    });
    return rc ? rc : p.drain();
}

int garage_ec_shard_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *shard_len, size_t stride,
                         size_t n_stripes, int shards_per_stripe, uint8_t *sums_out, int mem_kind, void *cuda_stream)
{
    if (!sums_out) return GARAGE_EC_E_INVALID;
    return sums_common(ctx, shards, nullptr, shard_len, stride, n_stripes, shards_per_stripe, sums_out, nullptr,
                       mem_kind, cuda_stream);
}

int garage_ec_check_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *expect, const uint32_t *shard_len,
                         size_t stride, size_t n_stripes, int shards_per_stripe, uint8_t *bad_out, int mem_kind,
                         void *cuda_stream)
{
    if (!expect || !bad_out) return GARAGE_EC_E_INVALID;
    return sums_common(ctx, shards, expect, shard_len, stride, n_stripes, shards_per_stripe, nullptr, bad_out,
                       mem_kind, cuda_stream);
}

void garage_ec_blake2sum(const uint8_t *data, size_t len, uint8_t out32[32]) { blake2sum_host(data, len, out32); }

// A plain memcpy leaves the destination lines modified in the writing core's cache, and the DMA read that follows has
// to pull them out of there snoop by snoop, several times slower than an upload of the same batch at rest in DRAM.
// Non-temporal stores send the lines to memory instead.  GARAGE_EC_NT_COPY=0 falls back to memcpy (A/B measurements).
void garage_ec_copy_for_dma(void *dst_v, const void *src_v, size_t n)
{
    uint8_t *dst = static_cast<uint8_t *>(dst_v);
    const uint8_t *src = static_cast<const uint8_t *>(src_v);
#if defined(__x86_64__)
    static const bool nt = [] {
        const char *e = getenv("GARAGE_EC_NT_COPY");
        return !(e && e[0] == '0');
    }();
    if (nt && n >= 4096) {
        const size_t head = (size_t)(-(uintptr_t)dst & 63);
        memcpy(dst, src, head);
        dst += head, src += head, n -= head;
        const size_t body = n & ~(size_t)63;
        for (size_t i = 0; i < body; i += 64) {
            const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i *>(src + i));
            const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i *>(src + i + 16));
            const __m128i c = _mm_loadu_si128(reinterpret_cast<const __m128i *>(src + i + 32));
            const __m128i d = _mm_loadu_si128(reinterpret_cast<const __m128i *>(src + i + 48));
            _mm_stream_si128(reinterpret_cast<__m128i *>(dst + i), a);
            _mm_stream_si128(reinterpret_cast<__m128i *>(dst + i + 16), b);
            _mm_stream_si128(reinterpret_cast<__m128i *>(dst + i + 32), c);
            _mm_stream_si128(reinterpret_cast<__m128i *>(dst + i + 48), d);
        }
        _mm_sfence();
        memcpy(dst + body, src + body, n - body);
        return;
    }
#endif
    if (n) memcpy(dst, src, n);
}

int garage_ec_set_wait_mode(garage_ec_ctx *ctx, int blocking)
{
    if (!ctx || (blocking != 0 && blocking != 1)) return GARAGE_EC_E_INVALID;
    ctx->wait_blocking.store(blocking, std::memory_order_relaxed);
    return GARAGE_EC_OK;
}

int garage_ec_set_sum_kind(garage_ec_ctx *ctx, int kind)
{
    if (!ctx || (kind != GARAGE_EC_SUM_BLAKE2 && kind != GARAGE_EC_SUM_ADLER8)) return GARAGE_EC_E_INVALID;
    ctx->sum_kind.store(kind, std::memory_order_relaxed);
    return GARAGE_EC_OK;
}

// Host-side adler8 with AVX2 (the read path checks the tag of every shard it touches: at 2.8 GB/s the scalar loop
// was a third of the CPU time of a GET in the block manager).  Adler-32 over a run of N = 32 * blocks bytes:
//   a' = a + sum d,   b' = b + N a + sum_{j,i} (N - 32 j - i) d[j][i]
// and N - 32 j - i = (32 - i) + 32 (blocks - 1 - j): a weighted sum inside each 32-byte block (pmaddubsw with the
// taps 32..1) plus 32 times, for every block, the byte sum of all blocks before it.  Runs are capped like zlib's
// NMAX so that nothing overflows 32 bits.  Same values as adler8_host (blake2b.h) and zlib.adler32.
#if defined(__x86_64__)
__attribute__((target("avx2"))) static uint32_t adler32_avx2(const uint8_t *p, size_t n)
{
    uint32_t a = 1, b = 0;
    const __m256i tap = _mm256_setr_epi8(32, 31, 30, 29, 28, 27, 26, 25, 24, 23, 22, 21, 20, 19, 18, 17, 16, 15, 14, 13, 12, 11,
                                         10, 9, 8, 7, 6, 5, 4, 3, 2, 1);
    const __m256i ones = _mm256_set1_epi16(1), zero = _mm256_setzero_si256();
    while (n >= 32) {
        size_t blocks = n / 32;
        if (blocks > 5552 / 32) blocks = 5552 / 32;
        n -= blocks * 32;
        uint64_t bb = (uint64_t)b + (uint64_t)a * (uint64_t)(blocks * 32);
        __m256i v_before = zero, v_sum = zero, v_tap = zero;
        for (size_t j = 0; j < blocks; j++, p += 32) {
            const __m256i d = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(p));
            v_before = _mm256_add_epi32(v_before, v_sum);
            v_sum = _mm256_add_epi32(v_sum, _mm256_sad_epu8(d, zero));
            v_tap = _mm256_add_epi32(v_tap, _mm256_madd_epi16(_mm256_maddubs_epi16(d, tap), ones));
        }
        alignas(32) uint32_t s[8], t[8], w[8];
        _mm256_store_si256(reinterpret_cast<__m256i *>(s), v_sum);
        _mm256_store_si256(reinterpret_cast<__m256i *>(t), v_tap);
        _mm256_store_si256(reinterpret_cast<__m256i *>(w), v_before);
        uint64_t aa = a;
        for (int i = 0; i < 8; i++) {
            aa += s[i];
            bb += (uint64_t)t[i] + 32ull * w[i];
        }
        a = (uint32_t)(aa % 65521);
        b = (uint32_t)(bb % 65521);
    }
    for (; n; n--, p++) {
        a += *p;
        b += a;
    }
    a %= 65521;
    b %= 65521;
    return (b << 16) | a;
}

static void adler8_host_fast(const uint8_t *data, size_t len, uint8_t out[32])
{
    static const bool avx2 = __builtin_cpu_supports("avx2");
    if (!avx2 || len > 0xffffffffull) return adler8_host(data, len, out);
    const size_t seg = adler8_seg_bytes((uint32_t)len);
    for (int s = 0; s < 8; s++) {
        const size_t start = (size_t)s * seg;
        uint32_t v = 1;  // Adler-32 of nothing
        if (start < len) v = adler32_avx2(data + start, len < start + seg ? len - start : seg);
        memcpy(out + 4 * s, &v, 4);  // little endian
    }
}
#else
static void adler8_host_fast(const uint8_t *data, size_t len, uint8_t out[32]) { adler8_host(data, len, out); }
#endif

// zlib Adler-32 of one buffer
static uint32_t adler32_one(const uint8_t *p, size_t n)
{
#if defined(__x86_64__)
    static const bool avx2 = __builtin_cpu_supports("avx2");
    if (avx2) return adler32_avx2(p, n);
#endif
    uint32_t a = 1, b = 0;
    while (n) {
        const size_t run = n > 5552 ? 5552 : n;  // zlib's NMAX: the sums cannot overflow 32 bits
        for (size_t i = 0; i < run; i++) {
            a += p[i];
            b += a;
        }
        a %= 65521;
        b %= 65521;
        p += run;
        n -= run;
    }
    return (b << 16) | a;
}

int garage_ec_shard_sum_host(int kind, const uint8_t *data, size_t len, uint8_t out32[32])
{
    if (!out32 || (!data && len)) return GARAGE_EC_E_INVALID;
    if (kind == GARAGE_EC_SUM_BLAKE2) blake2sum_host(data, len, out32);
    else if (kind == GARAGE_EC_SUM_ADLER8) adler8_host_fast(data, len, out32);
    else return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

int garage_ec_tag_span(int kind, uint32_t shard_len, uint32_t off, uint32_t len, uint32_t *span_off, uint32_t *span_len)
{
    if (!span_off || !span_len || (uint64_t)off + len > shard_len) return GARAGE_EC_E_INVALID;
    if (kind == GARAGE_EC_SUM_BLAKE2) {  // one hash over the whole shard
        *span_off = 0;
        *span_len = shard_len;
        return GARAGE_EC_OK;
    }
    if (kind != GARAGE_EC_SUM_ADLER8) return GARAGE_EC_E_INVALID;
    if (!len) {
        *span_off = off;
        *span_len = 0;
        return GARAGE_EC_OK;
    }
    const uint64_t seg = adler8_seg_bytes(shard_len), a = off / seg * seg,
                   b = std::min<uint64_t>(((uint64_t)off + len + seg - 1) / seg * seg, shard_len);
    *span_off = (uint32_t)a;
    *span_len = (uint32_t)(b - a);
    return GARAGE_EC_OK;
}

int garage_ec_check_shard_span_host(int kind, const uint8_t *bytes, uint32_t shard_len, uint32_t span_off,
                                    uint32_t span_len, const uint8_t tag32[32])
{
    if (!tag32 || (!bytes && span_len) || (uint64_t)span_off + span_len > shard_len) return GARAGE_EC_E_INVALID;
    if (kind == GARAGE_EC_SUM_BLAKE2) {
        if (span_off || span_len != shard_len) return GARAGE_EC_E_INVALID;
        uint8_t h[32];
        blake2sum_host(bytes, shard_len, h);
        return memcmp(h, tag32, 32) ? 1 : GARAGE_EC_OK;
    }
    if (kind != GARAGE_EC_SUM_ADLER8) return GARAGE_EC_E_INVALID;
    if (!span_len) return GARAGE_EC_OK;
    // whole segments only: the span starts on a segment edge and ends on one or at the shard's end
    const uint64_t seg = adler8_seg_bytes(shard_len), end = (uint64_t)span_off + span_len;
    if (span_off % seg || (end % seg && end != shard_len)) return GARAGE_EC_E_INVALID;
    for (uint64_t a = span_off; a < end; a += seg) {
        const uint32_t v = adler32_one(bytes + (a - span_off), std::min<uint64_t>(seg, end - a));
        uint32_t want;
        memcpy(&want, tag32 + 4 * (a / seg), 4);  // little endian
        if (v != want) return 1;
    }
    return GARAGE_EC_OK;
}

int garage_ec_check_shard_half_host(int kind, const uint8_t *half_bytes, uint32_t shard_len, int which,
                                    const uint8_t tag32[32])
{
    if (kind != GARAGE_EC_SUM_ADLER8 || (shard_len % 128) || (which != 0 && which != 1) || !tag32 ||
        (!half_bytes && shard_len))
        return GARAGE_EC_E_INVALID;
    if (!shard_len) {  // four empty segments: Adler-32 = 1 each
        for (int t = 0; t < 4; t++) {
            uint32_t want;
            memcpy(&want, tag32 + 4 * (4 * which + t), 4);
            if (want != 1u) return 1;
        }
        return GARAGE_EC_OK;
    }
    // shard_len % 128 == 0: the 8 segments are shard_len/8 bytes each, and half `which` is segments 4*which..+3
    return garage_ec_check_shard_span_host(kind, half_bytes, shard_len, (uint32_t)which * (shard_len / 2), shard_len / 2,
                                           tag32);
}

// --------------------------------------------------------------------------- SCRUB + REPAIR
int garage_ec_scrub_repair(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *expect_sums, uint8_t *bad_out,
                           int32_t *status, const uint32_t *shard_len, size_t stride, size_t n_stripes, int mem_kind,
                           void *cuda_stream)
{
    if (!ctx || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE)) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_stripes, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!shards || !expect_sums || !bad_out) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    const size_t tot = ctx->k + ctx->m;
    if (n_stripes * tot > 0xffffffffull) return GARAGE_EC_E_INVALID;
    if (mem_kind == GARAGE_EC_MEM_HOST && !shard_lens_ok(ctx, shard_len, stride, n_stripes)) return GARAGE_EC_E_INVALID;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (mem_kind == GARAGE_EC_MEM_DEVICE) {
        cudaStream_t st = (cudaStream_t)cuda_stream;
        rc = run_sums(ctx, shards, expect_sums, shard_len, stride, n_stripes * tot, (int)tot, nullptr, bad_out, st);
        if (rc) return rc;
        return with_stream_scratch(ctx, plan_scratch_bytes(ctx, n_stripes), st, [&](uint8_t *scratch) {
            return run_reconstruct(ctx, shards, bad_out, nullptr, status, shard_len, stride, n_stripes, scratch, st,
                                   /*present_is_bad=*/true);
        });
    }
    // HOST: every shard goes up (it has to be hashed); only the rebuilt shards come back.  The
    // rebuilt set is known once the bad flags are on the host, so each lane's chunk is retired
    // (flags read, copies issued) when the lane comes round again.
    HostPipeline p(ctx, n_stripes, tot * stride);
    SmallLayout sl;
    const size_t o_exp = sl.take(p.cs * tot * 32), o_bad = sl.take(p.cs * tot), o_status = sl.take(p.cs * 4),
                 o_len = sl.take(p.cs * 4), o_plan = sl.take(plan_scratch_bytes(ctx, p.cs));
    rc = p.reserve(p.cs * tot * stride, sl.bytes);
    if (rc) return rc;
    int32_t *st_out = p.status_out(status);
    const Retire retire = [&](const HostChunk &ch) -> int {  // bad flags + status of this chunk are on the host
        for (size_t s = ch.s0; s < ch.s0 + ch.cnt; s++) {
            if (st_out[s] != 0) continue;
            const size_t len = shard_len ? shard_len[s] : stride;
            for (size_t i = 0; i < tot; i++)
                if (bad_out[s * tot + i])
                    p.down.add(shards + (s * tot + i) * stride, ch.L->d_buf + ((s - ch.s0) * tot + i) * stride,
                               align_up(len, 16));
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, ch.L->stream);
    };
    rc = p.run(
        [&](const HostChunk &ch) -> int {
            HostLane &L = *ch.L;
            const size_t s0 = ch.s0, cnt = ch.cnt;
            CU_TRY(ctx, cudaMemcpyAsync(L.d_buf, shards + s0 * tot * stride, cnt * tot * stride, cudaMemcpyHostToDevice,
                                        L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_exp, expect_sums + s0 * tot * 32, cnt * tot * 32,
                                        cudaMemcpyHostToDevice, L.stream));
            const uint32_t *d_len = nullptr;
            if (shard_len) {
                CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, shard_len + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
                d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_len);
            }
            int r = run_sums(ctx, L.d_buf, L.d_small + o_exp, d_len, stride, cnt * tot, (int)tot, nullptr,
                             L.d_small + o_bad, L.stream);
            if (r) return r;
            r = run_reconstruct(ctx, L.d_buf, L.d_small + o_bad, nullptr, reinterpret_cast<int32_t *>(L.d_small + o_status),
                                d_len, stride, cnt, L.d_small + o_plan, L.stream, true);
            if (r) return r;
            CU_TRY(ctx, cudaMemcpyAsync(bad_out + s0 * tot, L.d_small + o_bad, cnt * tot, cudaMemcpyDeviceToHost, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(st_out + s0, L.d_small + o_status, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            return GARAGE_EC_OK;
        },
        retire);
    if (!rc) rc = p.drain(retire);
    if (rc) return rc;
    for (size_t s = 0; s < n_stripes; s++)
        if (st_out[s] != 0) return GARAGE_EC_E_UNRECOVERABLE;
    return GARAGE_EC_OK;
}

// --------------------------------------------------------------------------- BLOCK-LEVEL
int garage_ec_encode_blocks(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *block_len,
                            size_t n_blocks, uint8_t *parity_out, size_t stride)
{
    return garage_ec_encode_blocks_with_sums(ctx, blocks, block_len, n_blocks, parity_out, nullptr, stride);
}

int garage_ec_encode_blocks_with_sums(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *block_len,
                                      size_t n_blocks, uint8_t *parity_out, uint8_t *sums_out, size_t stride)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_blocks, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_blocks == 0) return GARAGE_EC_OK;
    if (!blocks || !block_len || !parity_out) return GARAGE_EC_E_INVALID;
    const size_t k = ctx->k, m = ctx->m;
    uint32_t max_len = 0;
    for (size_t s = 0; s < n_blocks; s++) {
        if (!blocks[s] && block_len[s]) return GARAGE_EC_E_INVALID;
        if (code_shard_len(ctx, block_len[s]) > stride) return GARAGE_EC_E_INVALID;
        max_len = block_len[s] > max_len ? block_len[s] : max_len;
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    HostPipeline p(ctx, n_blocks, k * stride);
    const size_t cs = p.cs;
    // per lane: [blocks as they arrive, contiguous, `pitch` apart][k data shards][m parity shards]
    const size_t pitch = align_up((size_t)max_len + 16, 16);  // + one aligned word of slack for the split kernel
    const size_t blk_b = align_up(cs * pitch, 256), in_b = cs * k * stride, out_b = cs * m * stride;
    // small: [shard_len | block_len] (staged through the lane's pageable slot of the same layout) | tags
    SmallLayout sl;
    const size_t o_lens = sl.take(cs * 8), o_blen = o_lens + cs * 4, o_sums = sl.take(cs * (k + m) * 32);
    rc = p.reserve(blk_b + in_b + out_b, sl.bytes, cs * 8);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t s0 = ch.s0, cnt = ch.cnt;
        uint32_t *hl = reinterpret_cast<uint32_t *>(ch.host), *hb = hl + cs;
        uint8_t *d_blk = L.d_buf, *d_data = L.d_buf + blk_b, *d_par = d_data + in_b;
        for (size_t s = 0; s < cnt; s++) {
            hl[s] = code_shard_len(ctx, block_len[s0 + s]);
            hb[s] = block_len[s0 + s];
            // H2D: the block as ONE contiguous copy; the framing happens on the device
            p.up.add(d_blk + s * pitch, blocks[s0 + s], block_len[s0 + s]);
        }
        int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_lens, hl, cnt * 4, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_blen, hb, cnt * 4, cudaMemcpyHostToDevice, L.stream));
        SplitParams sp;
        sp.blocks = d_blk;
        sp.block_len = reinterpret_cast<const uint32_t *>(L.d_small + o_blen);
        sp.shards = d_data;
        sp.block_pitch = pitch;
        sp.stride = (uint32_t)stride;
        sp.k = (uint32_t)k;
        sp.n = (uint32_t)cnt;
        sp.quantum = ctx->quantum;
        // ~4 CTAs per SM whatever the batch size (one CTA per block left 13 SMs copying 1 MiB each: 150 us)
        sp.parts = (uint32_t)std::max<size_t>(1, std::min<size_t>(64, ((size_t)ctx->sm_count * 4 + cnt - 1) / cnt));
        split_blocks_kernel<<<(unsigned)std::min<size_t>(cnt * sp.parts, (size_t)ctx->sm_count * 8), 256, 0, L.stream>>>(sp);
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
        CU_TRY(ctx, cudaGetLastError());
        const uint32_t *d_len = reinterpret_cast<const uint32_t *>(L.d_small + o_lens);
        r = run_uniform(ctx, kModeEncode, d_data, k * stride, d_par, m * stride, nullptr, d_len, stride, cnt, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(parity_out + s0 * m * stride, d_par, cnt * m * stride, cudaMemcpyDeviceToHost, L.stream));
        if (sums_out) {
            // per-shard tags of all k+m shards while they are on the device (row f2): [s][k+m][32]
            r = run_sums(ctx, d_data, nullptr, d_len, stride, cnt * k, (int)k, L.d_small + o_sums, nullptr, L.stream,
                         (int)(k + m), 0, d_par, cnt * m, (int)m, (int)k);
            if (r) return r;
            CU_TRY(ctx, cudaMemcpyAsync(sums_out + s0 * (k + m) * 32, L.d_small + o_sums, cnt * (k + m) * 32,
                                        cudaMemcpyDeviceToHost, L.stream));
        }
        return GARAGE_EC_OK;
    });
    return rc ? rc : p.drain();
}

int garage_ec_decode_blocks(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present,
                            const uint32_t *block_len, size_t n_blocks, size_t stride,
                            uint8_t *const *blocks_out, int32_t *status)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n_blocks, ctx->k + ctx->m);
    if (rc) return rc;
    if (n_blocks == 0) return GARAGE_EC_OK;
    if (!shards || !present || !block_len || !blocks_out) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    const size_t k = ctx->k, tot = ctx->k + ctx->m;
    CU_TRY(ctx, cudaSetDevice(ctx->device));

    // stripes with an absent data shard go to the GPU; the rest is a host-side join
    std::vector<size_t> need;
    std::vector<uint64_t> reads(n_blocks);  // survivors (halves) the kernel reads, data shards wanted
    std::vector<uint8_t> ok(n_blocks);
    std::vector<uint8_t> want_data(tot);
    for (size_t i = 0; i < tot; i++) want_data[i] = i < k ? 1 : 0;
    bool any_bad = false;
    for (size_t s = 0; s < n_blocks; s++) {
        const uint8_t *pr = present + s * tot;
        bool data_missing = false;
        for (size_t j = 0; j < k; j++) data_missing |= !pr[j];
        if (code_shard_len(ctx, block_len[s]) > stride) return GARAGE_EC_E_INVALID;
        ok[s] = stripe_read_plan(ctx, pr, want_data.data(), &reads[s]);
        if (!ok[s]) {
            if (status) status[s] = GARAGE_EC_E_UNRECOVERABLE;
            any_bad = true;
            continue;
        }
        if (status) status[s] = 0;
        if (data_missing) need.push_back(s);
    }
    // the data-shard pieces of block s (framing: block = shard0|shard1|...), as f(j, offset in the block, bytes)
    auto for_each_data_piece = [&](size_t s, auto &&f) {
        const size_t Ls = code_shard_len(ctx, block_len[s]);
        for (size_t j = 0; j < k && j * Ls < block_len[s]; j++) f(j, j * Ls, std::min<size_t>(block_len[s] - j * Ls, Ls));
    };
    HostPipeline p(ctx, need.size(), tot * stride);
    const size_t cs = p.cs;
    SmallLayout sl;
    const size_t o_present = sl.take(cs * tot), o_want = sl.take(cs * tot), o_status = sl.take(cs * 4),
                 o_len = sl.take(cs * 4), o_plan = sl.take(plan_scratch_bytes(ctx, cs));
    // pageable staging per lane: shard_len | present | want
    rc = p.reserve(cs * tot * stride, sl.bytes, cs * 4 + 2 * cs * tot);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &L = *ch.L;
        const size_t q0 = ch.s0, cnt = ch.cnt;
        uint32_t *hl = reinterpret_cast<uint32_t *>(ch.host);
        uint8_t *hp = ch.host + cs * 4, *hw = hp + cs * tot;
        for (size_t q = 0; q < cnt; q++) {
            const size_t s = need[q0 + q];
            memcpy(hp + q * tot, present + s * tot, tot);
            memcpy(hw + q * tot, want_data.data(), tot);  // data shards only
            hl[q] = code_shard_len(ctx, block_len[s]);
            // H2D: only the survivors the kernel reads -- the GET path is PCIe-bound, absent and
            // surplus shards stay on the host
            for (size_t i = 0; i < tot; i++)
                for_each_read_piece(ctx, reads[s], i, hl[q], align_up(hl[q], 16), [&](size_t off, size_t bytes) {
                    p.up.add(L.d_buf + (q * tot + i) * stride + off, shards + (s * tot + i) * stride + off, bytes);
                });
        }
        int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
        if (r) return r;
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, hp, cnt * tot, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_want, hw, cnt * tot, cudaMemcpyHostToDevice, L.stream));
        CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, hl, cnt * 4, cudaMemcpyHostToDevice, L.stream));
        r = run_reconstruct(ctx, L.d_buf, L.d_small + o_present, L.d_small + o_want,
                            reinterpret_cast<int32_t *>(L.d_small + o_status),
                            reinterpret_cast<const uint32_t *>(L.d_small + o_len), stride, cnt, L.d_small + o_plan,
                            L.stream);
        if (r) return r;
        // rebuilt data shards land directly in the output blocks
        for (size_t q = 0; q < cnt; q++) {
            const size_t s = need[q0 + q];
            for_each_data_piece(s, [&](size_t j, size_t off, size_t bytes) {
                if (!present[s * tot + j]) p.down.add(blocks_out[s] + off, L.d_buf + (q * tot + j) * stride, bytes);
            });
        }
        return p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
    });
    if (rc) return rc;
    // host-side join of the data shards that did arrive, while the GPU works
    for (size_t s = 0; s < n_blocks; s++) {
        if (!ok[s]) continue;
        for_each_data_piece(s, [&](size_t j, size_t off, size_t bytes) {
            if (present[s * tot + j]) memcpy(blocks_out[s] + off, shards + (s * tot + j) * stride, bytes);
        });
    }
    rc = p.drain();
    if (rc) return rc;
    return any_bad ? GARAGE_EC_E_UNRECOVERABLE : GARAGE_EC_OK;
}

// --------------------------------------------------------------------------- TRANSCODE
}  // extern "C"
namespace {

// device scratch of run_transcode for n stripes: src_len | dst_len | geo | status (caller passed none) | want | plan
struct TranscodeScratch {
    size_t o_src_len, o_dst_len, o_geo, o_status, o_want, o_plan, bytes;
    TranscodeScratch(const garage_ec_ctx *src, size_t n, size_t src_tot, bool degraded)
    {
        const size_t a = align_up(n * 4, 16);
        o_src_len = 0;
        o_dst_len = a;
        o_geo = 2 * a;
        o_status = 3 * a;
        o_want = 4 * a;
        o_plan = o_want + (degraded ? align_up(n * src_tot, 16) : 0);
        bytes = o_plan + (degraded ? plan_scratch_bytes(src, n) : 0);
    }
};

// Device-resident transcode of n stripes (DESIGN.md 2.3): lengths, the source reconstruct of absent data shards (only
// when `present` is given), the reframe into dst's data shards, dst's encode in place and dst's tags.  src == NULL:
// whole blocks, `s_stride` apart.  status: device, nullable.
int run_transcode(garage_ec_ctx *dst, garage_ec_ctx *src, uint8_t *s_sh, size_t s_stride, const uint8_t *present,
                  const uint32_t *block_len, uint8_t *d_sh, size_t d_stride, uint8_t *sums, int32_t *status, size_t n,
                  uint8_t *scratch, cudaStream_t st)
{
    const size_t s_tot = src ? src->k + src->m : 1, d_tot = dst->k + dst->m;
    const TranscodeScratch L(src, n, s_tot, present != nullptr);
    TranscodeParams q;
    memset(&q, 0, sizeof(q));
    q.src = s_sh;
    q.block_len = block_len;
    q.dst = d_sh;
    q.src_len = reinterpret_cast<uint32_t *>(scratch + L.o_src_len);
    q.dst_len = reinterpret_cast<uint32_t *>(scratch + L.o_dst_len);
    q.geo = reinterpret_cast<int32_t *>(scratch + L.o_geo);
    q.status = status ? status : reinterpret_cast<int32_t *>(scratch + L.o_status);
    q.rec_status = present ? q.status : nullptr;
    q.src_pitch = s_tot * s_stride;
    q.dst_pitch = d_tot * d_stride;
    q.src_stride = (uint32_t)s_stride;
    q.dst_stride = (uint32_t)d_stride;
    q.ks = src ? (uint32_t)src->k : 1u;
    q.kd = (uint32_t)dst->k;
    q.src_whole = src ? 0u : 1u;
    q.src_quantum = src ? src->quantum : 1u;
    q.dst_quantum = dst->quantum;
    q.n = (uint32_t)n;
    q.parts = (uint32_t)std::max<size_t>(1, std::min<size_t>(64, ((size_t)dst->sm_count * 4 + n - 1) / n));
    transcode_lens_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)dst->sm_count * 4), 256, 0, st>>>(q);
    dst->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(dst, cudaGetLastError());
    if (present) {
        // absent source data shards first, by the source code's own plan; the plan kernel skips intact stripes
        uint8_t *want = scratch + L.o_want;
        CU_TRY(dst, cudaMemsetAsync(want, 0, n * s_tot, st));
        CU_TRY(dst, cudaMemset2DAsync(want, s_tot, 1, q.ks, n, st));
        int rc = run_reconstruct(src, s_sh, present, want, q.status, q.src_len, s_stride, n, scratch + L.o_plan, st);
        if (rc) return rc;
    }
    {
        TimedLaunch tl(dst, st);
        transcode_reframe_kernel<<<(unsigned)std::min<size_t>(n * q.parts, (size_t)dst->sm_count * 8), 256, 0, st>>>(q);
        dst->launches.fetch_add(1, std::memory_order_relaxed);
        CU_TRY(dst, cudaGetLastError());
    }
    int rc = run_uniform(dst, kModeEncode, d_sh, q.dst_pitch, d_sh + (size_t)dst->k * d_stride, q.dst_pitch, nullptr, q.dst_len,
                         d_stride, n, st);
    if (rc) return rc;
    if (sums) return run_sums(dst, d_sh, nullptr, q.dst_len, d_stride, n * d_tot, (int)d_tot, sums, nullptr, st);
    return GARAGE_EC_OK;
}

// HOST mode: chunks through the lanes.  Uploads the present source data shards and, for a stripe with an absent data
// shard, the pieces of the source read plan; downloads the destination shards (and tags) of the stripes that
// converted.  src_shards is never written.
int transcode_host(garage_ec_ctx *dst, garage_ec_ctx *src, const uint8_t *src_shards, const uint8_t *src_present,
                   const uint32_t *block_len, size_t s_stride, uint8_t *dst_shards, size_t d_stride, uint8_t *dst_sums,
                   int32_t *status, size_t n)
{
    const size_t ks = src ? src->k : 1, s_tot = src ? src->k + src->m : 1, d_tot = dst->k + dst->m;
    std::vector<uint64_t> reads(n, 0);
    std::vector<uint8_t> ok(n, 1), degraded(n, 0);
    std::vector<uint8_t> want_data(s_tot, 0);
    for (size_t i = 0; i < ks; i++) want_data[i] = 1;
    for (size_t s = 0; s < n && src_present; s++) {
        const uint8_t *pr = src_present + s * s_tot;
        for (size_t j = 0; j < ks; j++) degraded[s] |= !pr[j];
        if (degraded[s]) ok[s] = stripe_read_plan(src, pr, want_data.data(), &reads[s]);
    }
    auto src_len = [&](size_t s) -> size_t { return src ? (size_t)code_shard_len(src, block_len[s]) : block_len[s]; };
    HostPipeline p(dst, n, s_tot * s_stride + d_tot * d_stride);
    const size_t cs = p.cs;
    const TranscodeScratch scr(src, cs, s_tot, src_present != nullptr);
    SmallLayout sl;
    const size_t o_len = sl.take(cs * 4), o_present = sl.take(cs * s_tot), o_status = sl.take(cs * 4),
                 o_sums = sl.take(dst_sums ? cs * d_tot * 32 : 0), o_scr = sl.take(scr.bytes);
    const size_t d_src_b = cs * s_tot * s_stride;
    int rc = p.reserve(d_src_b + cs * d_tot * d_stride, sl.bytes);
    if (rc) return rc;
    rc = p.run([&](const HostChunk &ch) -> int {
        HostLane &Ln = *ch.L;
        const size_t s0 = ch.s0, cnt = ch.cnt;
        uint8_t *d_src = Ln.d_buf, *d_dst = Ln.d_buf + d_src_b;
        bool any_degraded = false;
        for (size_t s = s0; s < s0 + cnt; s++) {
            if (!ok[s]) continue;
            any_degraded |= degraded[s] != 0;
            const size_t Ls = src_len(s), q = s - s0;
            for (size_t i = 0; i < s_tot; i++) {
                const uint8_t *from = src_shards + (s * s_tot + i) * s_stride;
                uint8_t *to = d_src + (q * s_tot + i) * s_stride;
                if (i < ks) {
                    if (!src_present || src_present[s * s_tot + i]) p.up.add(to, from, align_up(Ls, 16));
                } else if (degraded[s]) {
                    for_each_read_piece(src, reads[s], i, Ls, align_up(Ls, 16),
                                        [&](size_t off, size_t bytes) { p.up.add(to + off, from + off, bytes); });
                }
            }
        }
        int r = p.up.flush(dst, cudaMemcpyHostToDevice, Ln.stream);
        if (r) return r;
        CU_TRY(dst, cudaMemcpyAsync(Ln.d_small + o_len, block_len + s0, cnt * 4, cudaMemcpyHostToDevice, Ln.stream));
        const uint8_t *d_present = nullptr;
        if (any_degraded) {
            CU_TRY(dst, cudaMemcpyAsync(Ln.d_small + o_present, src_present + s0 * s_tot, cnt * s_tot, cudaMemcpyHostToDevice,
                                        Ln.stream));
            d_present = Ln.d_small + o_present;
        }
        r = run_transcode(dst, src, d_src, s_stride, d_present, reinterpret_cast<const uint32_t *>(Ln.d_small + o_len), d_dst,
                          d_stride, dst_sums ? Ln.d_small + o_sums : nullptr,
                          reinterpret_cast<int32_t *>(Ln.d_small + o_status), cnt, Ln.d_small + o_scr, Ln.stream);
        if (r) return r;
        for (size_t s = s0; s < s0 + cnt; s++) {
            if (!ok[s]) continue;
            const size_t bytes = align_up(code_shard_len(dst, block_len[s]), 16), q = s - s0;
            for (size_t i = 0; i < d_tot; i++)
                p.down.add(dst_shards + (s * d_tot + i) * d_stride, d_dst + (q * d_tot + i) * d_stride, bytes);
            if (dst_sums) p.down.add(dst_sums + s * d_tot * 32, Ln.d_small + o_sums + q * d_tot * 32, d_tot * 32);
        }
        return p.down.flush(dst, cudaMemcpyDeviceToHost, Ln.stream);
    });
    if (!rc) rc = p.drain();
    if (rc) return rc;
    bool any_bad = false;
    for (size_t s = 0; s < n; s++) {
        if (status) status[s] = ok[s] ? 0 : GARAGE_EC_E_UNRECOVERABLE;
        any_bad |= !ok[s];
    }
    return any_bad ? GARAGE_EC_E_UNRECOVERABLE : GARAGE_EC_OK;
}

}  // namespace
extern "C" {

int garage_ec_transcode(garage_ec_ctx *dst, garage_ec_ctx *src, uint8_t *src_shards, const uint8_t *src_present,
                        const uint32_t *block_len, size_t src_stride, uint8_t *dst_shards, size_t dst_stride,
                        uint8_t *dst_sums, int32_t *status, size_t n_stripes, int mem_kind, void *cuda_stream)
{
    if (!dst || (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE)) return GARAGE_EC_E_INVALID;
    if (src && src->device != dst->device) return GARAGE_EC_E_INVALID;
    if (!src && src_present) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(dst, dst_stride, n_stripes, dst->k + dst->m);
    if (rc) return rc;
    rc = src ? check_geometry(src, src_stride, n_stripes, src->k + src->m) : check_geometry(dst, src_stride, n_stripes, 1);
    if (rc) return rc;
    if (n_stripes == 0) return GARAGE_EC_OK;
    if (!src_shards || !block_len || !dst_shards) return GARAGE_EC_E_INVALID;
    if (!aligned16(src_shards) || !aligned16(dst_shards)) return GARAGE_EC_E_ALIGN;
    if (dst_sums && n_stripes * (size_t)(dst->k + dst->m) > 0xffffffffull) return GARAGE_EC_E_INVALID;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        for (size_t s = 0; s < n_stripes; s++) {
            const uint64_t ls = src ? code_shard_len(src, block_len[s]) : block_len[s];
            if (ls > src_stride || code_shard_len(dst, block_len[s]) > dst_stride) return GARAGE_EC_E_INVALID;
        }
        CU_TRY(dst, cudaSetDevice(dst->device));
        return transcode_host(dst, src, src_shards, src_present, block_len, src_stride, dst_shards, dst_stride, dst_sums,
                              status, n_stripes);
    }
    CU_TRY(dst, cudaSetDevice(dst->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const TranscodeScratch scr(src, n_stripes, src ? src->k + src->m : 1, src_present != nullptr);
    return with_stream_scratch(dst, scr.bytes, st, [&](uint8_t *scratch) {
        return run_transcode(dst, src, src_shards, src_stride, src_present, block_len, dst_shards, dst_stride, dst_sums,
                             status, n_stripes, scratch, st);
    });
}

// --------------------------------------------------------------------------- SSE-C SEAL / OPEN (DESIGN.md 2.6, 4.9)
}  // extern "C"
namespace {

// Device scratch of a seal or open of n blocks: key material | len(B) | L | (seal) checksum accumulators | (open)
// reconstruct status | want | plan.  The key material comes first so that one memset clears every secret.
struct SseScratch {
    size_t o_keys, o_blen, o_len, o_crc, o_rec, o_want, o_plan, bytes;
    SseScratch(const garage_ec_ctx *ctx, size_t n, bool open)
    {
        size_t b = 0;
        auto take = [&](size_t x) {
            const size_t o = b;
            b += align_up(x, 256);
            return o;
        };
        o_keys = take(n * sizeof(sse::SseKey));
        o_blen = take(n * 4);
        o_len = take(n * 4);
        o_crc = open ? 0 : take(n * 4);
        o_rec = open ? take(n * 4) : 0;
        o_want = open ? take(n * (size_t)(ctx->k + ctx->m)) : 0;
        o_plan = open ? take(plan_scratch_bytes(ctx, n)) : 0;
        bytes = b;
    }
};

int sse_launch_lens(garage_ec_ctx *ctx, const sse::LensParams &q, size_t n, cudaStream_t st)
{
    sse::sse_lens_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 4), 256, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "sse_lens_kernel launch");
}

int sse_launch_setup(garage_ec_ctx *ctx, const uint8_t *keys, sse::SseKey *ks, size_t n, cudaStream_t st)
{
    sse::SetupParams q;
    q.keys = keys;
    q.ks = ks;
    q.n = (uint32_t)n;
    sse::sse_setup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "sse_setup_kernel launch");
}

template <int MODE>
int sse_launch_chunks(garage_ec_ctx *ctx, sse::ChunkParams q, cudaStream_t st)
{
    // work items are (block, chunk) pairs over the chunks a block of plain_stride bytes can have (ranged: the caller's)
    if (!q.cmax) q.cmax = (uint32_t)std::max<unsigned long long>(1, (q.plain_stride + sse::kChunk - 1) / sse::kChunk);
    const unsigned long long items = (unsigned long long)q.n * q.cmax;
    const unsigned grid = (unsigned)std::min<unsigned long long>((items + sse::kWarps - 1) / sse::kWarps,
                                                                 (unsigned long long)ctx->sm_count * 4);
    TimedLaunch tl(ctx, st);
    sse::sse_chunk_kernel<MODE><<<grid, sse::kWarps * 32, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "sse_chunk_kernel launch");
}

// the checksum passes around a kCrc chunk kernel (sse_crc_pass_kernel)
int sse_launch_crc_pass(garage_ec_ctx *ctx, const sse::CrcPassParams &q, cudaStream_t st)
{
    sse::sse_crc_pass_kernel<<<(unsigned)std::min<size_t>((q.n + 255) / 256, (size_t)ctx->sm_count * 4), 256, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "sse_crc_pass_kernel launch");
}

int sse_launch_block_sums(garage_ec_ctx *ctx, const uint8_t *shards, const uint32_t *blen, const uint8_t *hashes,
                          uint8_t *hash_bad, uint8_t *digest, size_t stride, size_t n, cudaStream_t st)
{
    BlockSumParams q;
    memset(&q, 0, sizeof(q));
    q.shards = shards;
    q.block_len = blen;
    q.hashes = hashes;
    q.hash_bad = hash_bad;
    q.digest = digest;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    q.quantum = ctx->quantum;
    blake2sum_blocks_kernel<<<(unsigned)((n + kQuadThreads / 4 - 1) / (kQuadThreads / 4)), kQuadThreads, 0, st>>>(q);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "blake2sum_blocks_kernel launch");
}

// Seal n blocks on the device: lengths, key schedules, the GCM chunks into the data shards (crc_kind != NULL: and the
// plaintext checksums into crcs), the code's encode, the content hash and (sums != NULL) the shard tags.  The caller
// zeroes the key material of `scratch`.
int run_seal(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint32_t *plain_len,
             const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes, uint8_t *sums,
             const uint8_t *crc_kind, uint32_t *crcs, size_t n, uint8_t *scratch, cudaStream_t st)
{
    const SseScratch sc(ctx, n, false);
    sse::SseKey *ks = keys ? reinterpret_cast<sse::SseKey *>(scratch + sc.o_keys) : nullptr;
    uint32_t *blen = reinterpret_cast<uint32_t *>(scratch + sc.o_blen), *L = reinterpret_cast<uint32_t *>(scratch + sc.o_len);
    const size_t tot = ctx->k + ctx->m;
    sse::LensParams lp;
    memset(&lp, 0, sizeof(lp));
    lp.plain_len = plain_len;
    lp.blen = blen;
    lp.shard_len = L;
    lp.plain_stride = plain_stride;
    lp.stride = (uint32_t)stride;
    lp.k = (uint32_t)ctx->k;
    lp.m = (uint32_t)ctx->m;
    lp.n = (uint32_t)n;
    lp.quantum = ctx->quantum;
    lp.keyed = keys ? 1u : 0u;
    int rc = sse_launch_lens(ctx, lp, n, st);
    sse::CrcPassParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.kind = crc_kind;
    cp.acc = reinterpret_cast<uint32_t *>(scratch + sc.o_crc);
    cp.shard_len = L;
    cp.blen = blen;
    cp.plain_len = plain_len;
    cp.crcs = crcs;
    cp.n = (uint32_t)n;
    if (!rc && crc_kind) rc = sse_launch_crc_pass(ctx, cp, st);
    if (!rc && keys) rc = sse_launch_setup(ctx, keys, ks, n, st);
    if (rc) return rc;
    sse::ChunkParams q;
    memset(&q, 0, sizeof(q));
    q.plain_in = plain;
    q.plain_stride = plain_stride;
    q.plain_len = plain_len;
    q.blen = blen;
    q.shard_len = L;
    q.nonces = nonces;
    q.ks = ks;
    q.shards = shards;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    q.crc_kind = crc_kind;
    q.crc_acc = cp.acc;
    rc = crc_kind ? sse_launch_chunks<sse::kSeal | sse::kCrc>(ctx, q, st) : sse_launch_chunks<sse::kSeal>(ctx, q, st);
    cp.final = 1;
    if (!rc && crc_kind) rc = sse_launch_crc_pass(ctx, cp, st);
    if (!rc)
        rc = run_uniform(ctx, kModeEncode, shards, tot * stride, shards + (size_t)ctx->k * stride, tot * stride, nullptr, L,
                         stride, n, st);
    if (!rc) rc = sse_launch_block_sums(ctx, shards, blen, nullptr, nullptr, hashes, stride, n, st);
    if (!rc && sums) rc = run_sums(ctx, shards, nullptr, L, stride, n * tot, (int)tot, sums, nullptr, st);
    return rc;
}

// Open n stored blocks on the device: framing, key schedules, the rebuild of absent data shards, the content hash,
// every chunk's tag, then the plaintext of the blocks that passed.
int run_open(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present, const uint32_t *sealed, const uint8_t *hashes,
             const uint8_t *keys, uint8_t *plain, size_t plain_stride, uint32_t *plain_len_out, uint8_t *hash_bad,
             int32_t *status, size_t stride, size_t n, uint8_t *scratch, cudaStream_t st)
{
    const SseScratch sc(ctx, n, true);
    sse::SseKey *ks = reinterpret_cast<sse::SseKey *>(scratch + sc.o_keys);
    uint32_t *L = reinterpret_cast<uint32_t *>(scratch + sc.o_len);
    int32_t *rec = reinterpret_cast<int32_t *>(scratch + sc.o_rec);
    uint8_t *want = scratch + sc.o_want;
    sse::LensParams lp;
    memset(&lp, 0, sizeof(lp));
    lp.sealed_in = sealed;
    lp.shard_len = L;
    lp.status = status;
    lp.want = want;
    lp.plain_stride = plain_stride;
    lp.stride = (uint32_t)stride;
    lp.k = (uint32_t)ctx->k;
    lp.m = (uint32_t)ctx->m;
    lp.n = (uint32_t)n;
    lp.quantum = ctx->quantum;
    lp.keyed = 1;
    lp.open = 1;
    int rc = sse_launch_lens(ctx, lp, n, st);
    if (!rc) rc = sse_launch_setup(ctx, keys, ks, n, st);
    if (!rc) rc = run_reconstruct(ctx, shards, present, want, rec, L, stride, n, scratch + sc.o_plan, st);
    if (!rc) rc = sse_launch_block_sums(ctx, shards, sealed, hashes, hash_bad, nullptr, stride, n, st);
    if (rc) return rc;
    sse::ChunkParams q;
    memset(&q, 0, sizeof(q));
    q.plain_out = plain;
    q.plain_stride = plain_stride;
    q.plain_len_out = plain_len_out;
    q.blen = sealed;
    q.shard_len = L;
    q.ks = ks;
    q.shards = shards;
    q.status = status;
    q.rec_status = rec;
    q.hash_bad = hash_bad;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    rc = sse_launch_chunks<sse::kCheck>(ctx, q, st);
    if (!rc) rc = sse_launch_chunks<sse::kOpen>(ctx, q, st);
    return rc;
}

// plaintext length of a sealed length, or -1 if the STREAM framing cannot hold it
int64_t sse_plain_len(uint32_t sealed)
{
    if (sealed < sse::kPrefix + 16) return -1;
    const uint32_t r = (sealed - sse::kPrefix) % sse::kFrame;
    if (r >= 1 && r < 16) return -1;
    return (int64_t)sealed - sse::kPrefix - 16 * (int64_t)((sealed - sse::kPrefix + sse::kFrame - 1) / sse::kFrame);
}

// a lane's pinned key staging of at least `bytes`
int lane_key_staging(garage_ec_ctx *ctx, HostLane &L, size_t bytes)
{
    if (L.h_key_cap >= bytes) return GARAGE_EC_OK;
    if (L.h_key) cudaFreeHost(L.h_key);
    L.h_key = nullptr;
    L.h_key_cap = 0;
    bytes = std::max<size_t>(bytes, 64 << 10);
    CU_TRY(ctx, cudaHostAlloc(reinterpret_cast<void **>(&L.h_key), bytes, cudaHostAllocDefault));
    memset(L.h_key, 0, bytes);
    L.h_key_cap = bytes;
    return GARAGE_EC_OK;
}

// Clears the secrets a HOST call left in its lanes once nothing queued reads them any more and before another call
// can lease the lanes: wipe() is the call's HostPipeline::before_release.  `dev_off` / `dev_bytes`: the keys, nonces
// and key material in each lane's small buffer (already cleared on the stream unless the call failed half-way).
struct LaneKeyWipe {
    std::vector<HostLane *> lanes;
    size_t dev_off = 0, dev_bytes = 0;
    bool failed = true;
    void use(HostLane *L)
    {
        if (std::find(lanes.begin(), lanes.end(), L) == lanes.end()) lanes.push_back(L);
    }
    void wipe()
    {
        for (HostLane *L : lanes) {
            if (L->h_key) memset(L->h_key, 0, L->h_key_cap);
            if (failed && L->d_small && dev_bytes) (void)cudaMemset(L->d_small + dev_off, 0, dev_bytes);
        }
        (void)cudaGetLastError();
    }
};

int seal_host(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint8_t *const *blocks,
              const uint32_t *plain_len, const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride,
              uint8_t *hashes, uint8_t *sums, const uint8_t *crc_kind, uint32_t *crcs, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    auto block_at = [&](size_t s) { return blocks ? blocks[s] : plain + s * plain_stride; };
    uint32_t max_len = 0;
    for (size_t s = 0; s < n; s++) max_len = std::max(max_len, plain_len[s]);
    const size_t pitch = align_up((size_t)max_len + 16, 16);
    LaneKeyWipe wipe;
    HostPipeline p(ctx, n, pitch + tot * stride);
    p.before_release = [&wipe] { wipe.wipe(); };
    const size_t cs = p.cs;
    SmallLayout sl;
    const SseScratch sc(ctx, cs, false);
    const size_t o_scr = sl.take(sc.bytes), o_key = sl.take(cs * 40), o_len = sl.take(cs * 4), o_hash = sl.take(cs * 32),
                 o_sums = sl.take(sums ? cs * tot * 32 : 0), o_kind = sl.take(crc_kind ? cs : 0),
                 o_crcs = sl.take(crc_kind ? cs * 4 : 0);
    wipe.dev_off = o_scr;
    wipe.dev_bytes = o_len - o_scr;  // key material, keys and nonces
    const size_t blk_b = align_up(cs * pitch, 256);
    int rc = p.reserve(blk_b + cs * tot * stride, sl.bytes);
    if (rc) return rc;
    // batched copies for pinned buffers only, as in reconstruct_host
    bool pinned = true;
    for (size_t s = 0; pinned && s < (blocks ? n : 1); s++) pinned = !plain_len[s] || device_addressable_host(block_at(s));
    p.up.use_batch = pinned;
    p.down.use_batch = device_addressable_host(shards);
    const Retire clear_keys = [&](const HostChunk &ch) -> int {
        memset(ch.L->h_key, 0, ch.L->h_key_cap);
        return GARAGE_EC_OK;
    };
    rc = p.run(
        [&](const HostChunk &ch) -> int {
            HostLane &L = *ch.L;
            wipe.use(&L);
            const size_t s0 = ch.s0, cnt = ch.cnt;
            uint8_t *d_blk = L.d_buf, *d_sh = L.d_buf + blk_b;
            for (size_t q = 0; q < cnt; q++) p.up.add(d_blk + q * pitch, block_at(s0 + q), plain_len[s0 + q]);
            int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
            if (r) return r;
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, plain_len + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            const uint8_t *d_keys = nullptr, *d_nonces = nullptr;
            if (keys) {
                r = lane_key_staging(ctx, L, cs * 40);
                if (r) return r;
                memcpy(L.h_key, keys + s0 * 32, cnt * 32);
                memcpy(L.h_key + cs * 32, nonces + s0 * 8, cnt * 8);
                CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_key, L.h_key, cs * 40, cudaMemcpyHostToDevice, L.stream));
                d_keys = L.d_small + o_key;
                d_nonces = L.d_small + o_key + cs * 32;
            }
            if (crc_kind)
                CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_kind, crc_kind + s0, cnt, cudaMemcpyHostToDevice, L.stream));
            uint32_t *d_crcs = reinterpret_cast<uint32_t *>(L.d_small + o_crcs);
            r = run_seal(ctx, d_blk, pitch, reinterpret_cast<const uint32_t *>(L.d_small + o_len), d_keys, d_nonces, d_sh,
                         stride, L.d_small + o_hash, sums ? L.d_small + o_sums : nullptr,
                         crc_kind ? L.d_small + o_kind : nullptr, d_crcs, cnt, L.d_small + o_scr, L.stream);
            if (r) return r;
            if (keys) CU_TRY(ctx, cudaMemsetAsync(L.d_small + o_scr, 0, o_len - o_scr, L.stream));
            // D2H: roundup16(L) bytes of all k+m shards (the data shards are ciphertext now)
            for (size_t q = 0; q < cnt; q++) {
                const uint64_t b = keys ? sse::sealed_len(plain_len[s0 + q]) : plain_len[s0 + q];
                const size_t bytes = align_up(code_shard_len(ctx, (uint32_t)b), 16);
                for (size_t i = 0; i < tot; i++)
                    p.down.add(shards + ((s0 + q) * tot + i) * stride, d_sh + (q * tot + i) * stride, bytes);
            }
            r = p.down.flush(ctx, cudaMemcpyDeviceToHost, L.stream);
            if (r) return r;
            CU_TRY(ctx, cudaMemcpyAsync(hashes + s0 * 32, L.d_small + o_hash, cnt * 32, cudaMemcpyDeviceToHost, L.stream));
            if (sums)
                CU_TRY(ctx, cudaMemcpyAsync(sums + s0 * tot * 32, L.d_small + o_sums, cnt * tot * 32, cudaMemcpyDeviceToHost,
                                            L.stream));
            if (crc_kind) CU_TRY(ctx, cudaMemcpyAsync(crcs + s0, d_crcs, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            return GARAGE_EC_OK;
        },
        keys ? clear_keys : Retire());
    if (!rc) rc = p.drain(keys ? clear_keys : Retire());
    wipe.failed = rc != 0;
    return rc;
}

int open_host(garage_ec_ctx *ctx, uint8_t *shards, uint8_t *const *stripes, const uint8_t *present,
              const uint32_t *sealed, const uint8_t *hashes, const uint8_t *keys, uint8_t *plain, size_t plain_stride,
              uint8_t *const *outs, uint32_t *plain_len_out, uint8_t *hash_bad, int32_t *status, size_t stride, size_t n)
{
    const size_t k = ctx->k, tot = ctx->k + ctx->m;
    auto shard_at = [&](size_t s, size_t i) { return stripes ? stripes[s] + i * stride : shards + (s * tot + i) * stride; };
    auto out_at = [&](size_t s) { return outs ? outs[s] : plain + s * plain_stride; };
    int64_t max_plain = 0;
    for (size_t s = 0; s < n; s++) max_plain = std::max(max_plain, sse_plain_len(sealed[s]));
    const size_t pitch = align_up((size_t)max_plain + 16, 16);
    std::vector<uint8_t> want(tot);
    for (size_t i = 0; i < tot; i++) want[i] = i < k;
    LaneKeyWipe wipe;
    HostPipeline p(ctx, n, tot * stride + pitch);
    p.before_release = [&wipe] { wipe.wipe(); };
    const size_t cs = p.cs;
    SmallLayout sl;
    const SseScratch sc(ctx, cs, true);
    const size_t o_scr = sl.take(sc.bytes), o_key = sl.take(cs * 32), o_present = sl.take(cs * tot),
                 o_sealed = sl.take(cs * 4), o_hash = sl.take(cs * 32), o_bad = sl.take(cs), o_status = sl.take(cs * 4),
                 o_plen = sl.take(cs * 4);
    wipe.dev_off = o_scr;
    wipe.dev_bytes = o_key + cs * 32 - o_scr;
    const size_t sh_b = align_up(cs * tot * stride, 256);
    int rc = p.reserve(sh_b + cs * pitch, sl.bytes, cs * 4);
    if (rc) return rc;
    bool pinned = true;
    for (size_t s = 0; pinned && s < (stripes ? n : 1); s++) pinned = device_addressable_host(shard_at(s, 0));
    for (size_t s = 0; pinned && s < (outs ? n : 1); s++) pinned = device_addressable_host(out_at(s));
    p.up.use_batch = p.down.use_batch = pinned;
    const Retire retire = [&](const HostChunk &ch) -> int {
        memset(ch.L->h_key, 0, ch.L->h_key_cap);
        const uint32_t *plen = reinterpret_cast<const uint32_t *>(ch.host);
        for (size_t q = 0; q < ch.cnt; q++) {
            const size_t s = ch.s0 + q;
            if (status[s] || hash_bad[s]) continue;
            plain_len_out[s] = plen[q];
            p.down.add(out_at(s), ch.L->d_buf + sh_b + q * pitch, plen[q]);
        }
        int r = p.down.flush(ctx, cudaMemcpyDeviceToHost, ch.L->stream);
        if (r) return r;
        CU_TRY(ctx, lane_wait(ctx, *ch.L));
        return GARAGE_EC_OK;
    };
    rc = p.run(
        [&](const HostChunk &ch) -> int {
            HostLane &L = *ch.L;
            wipe.use(&L);
            const size_t s0 = ch.s0, cnt = ch.cnt;
            uint8_t *d_sh = L.d_buf;
            // H2D: the present data shards (the block's bytes) and what the code's plan reads to rebuild the others
            for (size_t s = s0; s < s0 + cnt; s++) {
                uint64_t hv = 0;
                const uint8_t *pr = present + s * tot;
                const size_t len = code_shard_len(ctx, sealed[s]);
                const bool ok = stripe_read_plan(ctx, pr, want.data(), &hv);
                for (size_t i = 0; i < tot; i++) {
                    uint8_t *d = d_sh + ((s - s0) * tot + i) * stride;
                    if (i < k && pr[i]) p.up.add(d, shard_at(s, i), align_up(len, 16));
                    else if (ok && i >= k)
                        for_each_read_piece(ctx, hv, i, len, align_up(len, 16),
                                            [&](size_t off, size_t bytes) { p.up.add(d + off, shard_at(s, i) + off, bytes); });
                }
            }
            int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
            if (r) return r;
            r = lane_key_staging(ctx, L, cs * 32);
            if (r) return r;
            memcpy(L.h_key, keys + s0 * 32, cnt * 32);
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_key, L.h_key, cnt * 32, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, present + s0 * tot, cnt * tot, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_sealed, sealed + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_hash, hashes + s0 * 32, cnt * 32, cudaMemcpyHostToDevice, L.stream));
            int32_t *d_status = reinterpret_cast<int32_t *>(L.d_small + o_status);
            r = run_open(ctx, d_sh, L.d_small + o_present, reinterpret_cast<const uint32_t *>(L.d_small + o_sealed),
                         L.d_small + o_hash, L.d_small + o_key, d_sh + sh_b, pitch,
                         reinterpret_cast<uint32_t *>(L.d_small + o_plen), L.d_small + o_bad, d_status, stride, cnt,
                         L.d_small + o_scr, L.stream);
            if (r) return r;
            CU_TRY(ctx, cudaMemsetAsync(L.d_small + o_scr, 0, wipe.dev_bytes, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(status + s0, d_status, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(hash_bad + s0, L.d_small + o_bad, cnt, cudaMemcpyDeviceToHost, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(ch.host, L.d_small + o_plen, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            return GARAGE_EC_OK;
        },
        retire);
    if (!rc) rc = p.drain(retire);
    wipe.failed = rc != 0;
    if (rc) return rc;
    int worst = GARAGE_EC_OK;
    for (size_t s = 0; s < n; s++) {
        if (status[s] == GARAGE_EC_E_UNRECOVERABLE) return GARAGE_EC_E_UNRECOVERABLE;
        if (status[s]) worst = status[s];
    }
    return worst;
}

// checks shared by every seal form; plain_len values are host memory (HOST) or not looked at (DEVICE)
int seal_args(garage_ec_ctx *ctx, const uint8_t *keys, const uint8_t *nonces, const uint8_t *shards, size_t stride,
              const uint8_t *hashes, const uint8_t *sums, const uint8_t *crc_kind, const uint32_t *crcs, size_t n)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, ctx->k + ctx->m);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!shards || !hashes || (!keys) != (!nonces) || (crc_kind && !crcs)) return GARAGE_EC_E_INVALID;
    if (sums && n * (size_t)(ctx->k + ctx->m) > 0xffffffffull) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    return GARAGE_EC_OK;
}

// HOST: every checksum kind is known
int crc_kinds_ok(const uint8_t *crc_kind, size_t n)
{
    for (size_t s = 0; crc_kind && s < n; s++)
        if (crc_kind[s] > GARAGE_EC_CRC_CRC32C) return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

// HOST: every block's shard length must fit the stride
int seal_host_lens_ok(garage_ec_ctx *ctx, const uint32_t *plain_len, bool keyed, size_t stride, size_t n)
{
    for (size_t s = 0; s < n; s++) {
        const uint64_t b = keyed ? sse::sealed_len(plain_len[s]) : plain_len[s];
        if (b > 0xffffffffull || code_shard_len(ctx, (uint32_t)b) > stride) return GARAGE_EC_E_INVALID;
    }
    return GARAGE_EC_OK;
}

}  // namespace
extern "C" {

int garage_ec_sealed_len(uint32_t plain_len, uint32_t *sealed_len)
{
    if (!sealed_len) return GARAGE_EC_E_INVALID;
    const uint64_t b = sse::sealed_len(plain_len);
    if (b > 0xffffffffull) return GARAGE_EC_E_INVALID;
    *sealed_len = (uint32_t)b;
    return GARAGE_EC_OK;
}

int garage_ec_seal_crc(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint32_t *plain_len,
                       const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                       uint8_t *sums, const uint8_t *crc_kind, uint32_t *crcs, size_t n, int mem_kind, void *cuda_stream)
{
    if (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE) return GARAGE_EC_E_INVALID;
    int rc = seal_args(ctx, keys, nonces, shards, stride, hashes, sums, crc_kind, crcs, n);
    if (rc || n == 0) return rc;
    if (!plain || !plain_len || (plain_stride & 15)) return GARAGE_EC_E_INVALID;
    if (!aligned16(plain)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        for (size_t s = 0; s < n; s++)
            if (plain_len[s] > plain_stride) return GARAGE_EC_E_INVALID;
        rc = seal_host_lens_ok(ctx, plain_len, keys != nullptr, stride, n);
        if (!rc) rc = crc_kinds_ok(crc_kind, n);
        if (rc) return rc;
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        return seal_host(ctx, plain, plain_stride, nullptr, plain_len, keys, nonces, shards, stride, hashes, sums,
                         crc_kind, crcs, n);
    }
    if ((reinterpret_cast<uintptr_t>(plain_len) & 3) || (reinterpret_cast<uintptr_t>(hashes) & 7) ||
        (reinterpret_cast<uintptr_t>(sums) & 7) || (crc_kind && (reinterpret_cast<uintptr_t>(crcs) & 3)))
        return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const SseScratch sc(ctx, n, false);
    return with_stream_scratch(ctx, sc.bytes, st, [&](uint8_t *scratch) {
        const int r = run_seal(ctx, plain, plain_stride, plain_len, keys, nonces, shards, stride, hashes, sums, crc_kind,
                               crcs, n, scratch, st);
        const cudaError_t e = keys ? cudaMemsetAsync(scratch + sc.o_keys, 0, n * sizeof(sse::SseKey), st) : cudaSuccess;
        if (r) return r;
        return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "cudaMemsetAsync(key material)");
    });
}

int garage_ec_seal(garage_ec_ctx *ctx, const uint8_t *plain, size_t plain_stride, const uint32_t *plain_len,
                   const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                   uint8_t *sums, size_t n, int mem_kind, void *cuda_stream)
{
    return garage_ec_seal_crc(ctx, plain, plain_stride, plain_len, keys, nonces, shards, stride, hashes, sums, nullptr,
                              nullptr, n, mem_kind, cuda_stream);
}

int garage_ec_seal_blocks_crc(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *plain_len,
                              const uint8_t *keys, const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes,
                              uint8_t *sums, const uint8_t *crc_kind, uint32_t *crcs, size_t n)
{
    int rc = seal_args(ctx, keys, nonces, shards, stride, hashes, sums, crc_kind, crcs, n);
    if (rc || n == 0) return rc;
    if (!blocks || !plain_len) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n; s++)
        if (!blocks[s] && plain_len[s]) return GARAGE_EC_E_INVALID;
    rc = seal_host_lens_ok(ctx, plain_len, keys != nullptr, stride, n);
    if (!rc) rc = crc_kinds_ok(crc_kind, n);
    if (rc) return rc;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return seal_host(ctx, nullptr, 0, blocks, plain_len, keys, nonces, shards, stride, hashes, sums, crc_kind, crcs, n);
}

int garage_ec_seal_blocks(garage_ec_ctx *ctx, const uint8_t *const *blocks, const uint32_t *plain_len, const uint8_t *keys,
                          const uint8_t *nonces, uint8_t *shards, size_t stride, uint8_t *hashes, uint8_t *sums, size_t n)
{
    return garage_ec_seal_blocks_crc(ctx, blocks, plain_len, keys, nonces, shards, stride, hashes, sums, nullptr, nullptr,
                                     n);
}

int garage_ec_crc_combine(int kind, uint32_t crc_a, uint32_t crc_b, uint64_t len_b, uint32_t *out)
{
    if (!out || kind < GARAGE_EC_CRC_CRC32 || kind > GARAGE_EC_CRC_CRC32C) return GARAGE_EC_E_INVALID;
    *out = sse::crc_shift(sse::kCrcHost, kind - 1, crc_a, len_b) ^ crc_b;
    return GARAGE_EC_OK;
}

static int open_args(garage_ec_ctx *ctx, const void *shards, const uint8_t *present, const uint32_t *sealed,
                     const uint8_t *hashes, const uint8_t *keys, const uint32_t *plain_len_out, const uint8_t *hash_bad,
                     const int32_t *status, size_t stride, size_t n)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, ctx->k + ctx->m);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!shards || !present || !sealed || !hashes || !keys || !plain_len_out || !hash_bad || !status)
        return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

// HOST: a stored block whose shard length does not fit the stride is a caller error, not a verdict on the data
static int open_host_lens_ok(garage_ec_ctx *ctx, const uint32_t *sealed, size_t stride, size_t n)
{
    for (size_t s = 0; s < n; s++)
        if (code_shard_len(ctx, sealed[s]) > stride) return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

int garage_ec_open(garage_ec_ctx *ctx, uint8_t *shards, const uint8_t *present, const uint32_t *sealed_len,
                   const uint8_t *hashes, const uint8_t *keys, uint8_t *plain, size_t plain_stride,
                   uint32_t *plain_len_out, uint8_t *hash_bad, int32_t *status, size_t stride, size_t n, int mem_kind,
                   void *cuda_stream)
{
    if (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE) return GARAGE_EC_E_INVALID;
    int rc = open_args(ctx, shards, present, sealed_len, hashes, keys, plain_len_out, hash_bad, status, stride, n);
    if (rc || n == 0) return rc;
    if (!plain || (plain_stride & 15)) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards) || !aligned16(plain)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        rc = open_host_lens_ok(ctx, sealed_len, stride, n);
        if (rc) return rc;
        for (size_t s = 0; s < n; s++)
            if (sse_plain_len(sealed_len[s]) > (int64_t)plain_stride) return GARAGE_EC_E_INVALID;
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        return open_host(ctx, shards, nullptr, present, sealed_len, hashes, keys, plain, plain_stride, nullptr,
                         plain_len_out, hash_bad, status, stride, n);
    }
    if ((reinterpret_cast<uintptr_t>(sealed_len) & 3) || (reinterpret_cast<uintptr_t>(hashes) & 7) ||
        (reinterpret_cast<uintptr_t>(plain_len_out) & 3) || (reinterpret_cast<uintptr_t>(status) & 3))
        return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const SseScratch sc(ctx, n, true);
    return with_stream_scratch(ctx, sc.bytes, st, [&](uint8_t *scratch) {
        const int r = run_open(ctx, shards, present, sealed_len, hashes, keys, plain, plain_stride, plain_len_out, hash_bad,
                               status, stride, n, scratch, st);
        const cudaError_t e = cudaMemsetAsync(scratch + sc.o_keys, 0, n * sizeof(sse::SseKey), st);
        if (r) return r;
        return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "cudaMemsetAsync(key material)");
    });
}

int garage_ec_open_stripes(garage_ec_ctx *ctx, uint8_t *const *stripes, const uint8_t *present, const uint32_t *sealed_len,
                           const uint8_t *hashes, const uint8_t *keys, uint8_t *const *plains, uint32_t *plain_len_out,
                           uint8_t *hash_bad, int32_t *status, size_t stride, size_t n)
{
    int rc = open_args(ctx, stripes, present, sealed_len, hashes, keys, plain_len_out, hash_bad, status, stride, n);
    if (rc || n == 0) return rc;
    if (!plains) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n; s++) {
        if (!stripes[s] || !plains[s]) return GARAGE_EC_E_INVALID;
        if (!aligned16(stripes[s])) return GARAGE_EC_E_ALIGN;
    }
    rc = open_host_lens_ok(ctx, sealed_len, stride, n);
    if (rc) return rc;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return open_host(ctx, nullptr, stripes, present, sealed_len, hashes, keys, nullptr, 0, plains, plain_len_out,
                     hash_bad, status, stride, n);
}

// --------------------------------------------------------------------------- SSE-C RANGED OPEN (DESIGN.md 2.7, 4.10)
}  // extern "C"
namespace {

// The unmerged runs of the prefix B[0, 8) and the span of plaintext bytes [o, o + len) of a block sealed to S bytes,
// appended to `runs` (garage_ec_range_plan's runs of each); nothing for an empty range.
int open_range_runs(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t S, uint32_t o, uint32_t len,
                    std::vector<garage_ec_range> &runs, int *needs_gpu)
{
    uint32_t so, sl, c0, nch;
    int rc = sse::sealed_range(S, o, len, &so, &sl, &c0, &nch);
    if (rc || !len) return rc;
    rc = range_runs(ctx, present, S, 0, sse::kPrefix, runs, needs_gpu);
    return rc ? rc : range_runs(ctx, present, S, so, sl, runs, needs_gpu);
}

// Device scratch of a ranged open of n requests: key material first (one memset clears every secret), then the rows
// (2s: the prefix, 2s + 1: the span), the two decodes per request and their arguments.  A range of at most out_stride
// bytes touches at most out_stride / 4096 + 2 chunks: that bounds a span row.
struct OpenRangeScratch {
    size_t cmax, row_pitch, o_keys, o_rows, o_dec, o_blen2, o_off2, o_len2, o_present2, o_st2, bytes;
    OpenRangeScratch(const garage_ec_ctx *ctx, size_t n, size_t stride, size_t out_stride)
    {
        cmax = out_stride / sse::kChunk + 2;
        row_pitch = align_up(cmax * sse::kFrame, 16);
        SmallLayout sl;
        o_keys = sl.take(n * sizeof(sse::SseKey));
        o_rows = sl.take(2 * n * row_pitch);
        o_dec = sl.take(RangeScratch(ctx, 2 * n, stride).bytes);
        o_blen2 = sl.take(2 * n * 4);
        o_off2 = sl.take(2 * n * 4);
        o_len2 = sl.take(2 * n * 4);
        o_present2 = sl.take(2 * n * (size_t)(ctx->k + ctx->m));
        o_st2 = sl.take(2 * n * 4);
        bytes = sl.bytes;
    }
};

// Open plaintext ranges of n stored blocks on the device: framing and geometry, key schedules, each request's prefix
// and span decoded into its two rows, every touched chunk's tag, then the range bytes of the requests that passed.
// The caller zeroes the key material of `sc`.
int run_open_range(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present, const uint32_t *sealed,
                   const uint8_t *keys, const uint32_t *offset, const uint32_t *len, size_t stride, uint8_t *out,
                   size_t out_stride, int32_t *status, size_t n, uint8_t *sc, cudaStream_t st)
{
    const OpenRangeScratch o(ctx, n, stride, out_stride);
    sse::SseKey *ks = reinterpret_cast<sse::SseKey *>(sc + o.o_keys);
    uint32_t *blen2 = reinterpret_cast<uint32_t *>(sc + o.o_blen2), *off2 = reinterpret_cast<uint32_t *>(sc + o.o_off2),
             *len2 = reinterpret_cast<uint32_t *>(sc + o.o_len2);
    int32_t *st2 = reinterpret_cast<int32_t *>(sc + o.o_st2);
    sse::RangeLensParams lp;
    memset(&lp, 0, sizeof(lp));
    lp.sealed = sealed;
    lp.offset = offset;
    lp.len = len;
    lp.present = present;
    lp.status = status;
    lp.blen2 = blen2;
    lp.off2 = off2;
    lp.len2 = len2;
    lp.present2 = sc + o.o_present2;
    lp.out_stride = out_stride;
    lp.stride = (uint32_t)stride;
    lp.k = (uint32_t)ctx->k;
    lp.m = (uint32_t)ctx->m;
    lp.n = (uint32_t)n;
    lp.quantum = ctx->quantum;
    sse::sse_range_lens_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 4), 256, 0, st>>>(lp);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    int rc = sse_launch_setup(ctx, keys, ks, n, st);
    if (!rc)
        rc = run_decode_range(ctx, shards, 1, sc + o.o_present2, blen2, off2, len2, stride, sc + o.o_rows, o.row_pitch,
                              st2, 2 * n, sc + o.o_dec, st);
    if (rc) return rc;
    sse::ChunkParams q;
    memset(&q, 0, sizeof(q));
    q.plain_out = out;
    q.plain_stride = out_stride;
    q.rows = sc + o.o_rows;
    q.row_pitch = o.row_pitch;
    q.offset = offset;
    q.len = len;
    q.blen = sealed;
    q.ks = ks;
    q.status = status;
    q.rec_status = st2;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n;
    q.cmax = (uint32_t)o.cmax;
    rc = sse_launch_chunks<sse::kRangeCheck>(ctx, q, st);
    if (!rc) rc = sse_launch_chunks<sse::kRangeOpen>(ctx, q, st);
    return rc;
}

// HOST ranged open.  stripes / outs != NULL: the gather form.  Only the planned runs of the prefix and the span go up
// (ciphertext: the present ones too), into a stripe of the lane's buffer; only the len plaintext bytes come down.
int open_range_host(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *const *stripes, const uint8_t *present,
                    const uint32_t *sealed, const uint8_t *keys, const uint32_t *offset, const uint32_t *len,
                    size_t stride, uint8_t *out, size_t out_stride, uint8_t *const *outs, int32_t *status, size_t n)
{
    const size_t tot = ctx->k + ctx->m;
    auto shard_at = [&](size_t s, size_t i) { return stripes ? stripes[s] + i * stride : shards + (s * tot + i) * stride; };
    auto out_at = [&](size_t s) { return outs ? outs[s] : out + s * out_stride; };
    uint32_t max_len = 0;
    for (size_t s = 0; s < n; s++) {
        uint32_t so, sl, c0, nch;
        if (code_shard_len(ctx, sealed[s]) > stride ||
            sse::sealed_range(sealed[s], offset[s], len[s], &so, &sl, &c0, &nch) == GARAGE_EC_E_INVALID ||
            (len[s] && !out_at(s)))
            return GARAGE_EC_E_INVALID;
        max_len = std::max(max_len, len[s]);
    }
    const size_t opitch = align_up(std::max<size_t>(max_len, 16), 16);
    LaneKeyWipe wipe;
    HostPipeline p(ctx, n, tot * stride + opitch);
    p.before_release = [&wipe] { wipe.wipe(); };
    const size_t cs = p.cs;
    SmallLayout sl;
    const size_t o_key = sl.take(cs * 32), o_present = sl.take(cs * tot), o_sealed = sl.take(cs * 4),
                 o_off = sl.take(cs * 4), o_len = sl.take(cs * 4), o_status = sl.take(cs * 4);
    wipe.dev_off = o_key;
    wipe.dev_bytes = cs * 32;
    const size_t sh_b = align_up(cs * tot * stride, 256);
    int rc = p.reserve(sh_b + cs * opitch, sl.bytes);
    if (rc) return rc;
    bool pinned = true;
    for (size_t s = 0; pinned && s < (stripes ? n : 1); s++) pinned = device_addressable_host(shard_at(s, 0));
    for (size_t s = 0; pinned && outs && s < n; s++) pinned = !len[s] || device_addressable_host(outs[s]);
    if (!outs) pinned = pinned && device_addressable_host(out);
    p.up.use_batch = p.down.use_batch = pinned;
    const OpenRangeScratch osc(ctx, cs, stride, opitch);
    const Retire retire = [&](const HostChunk &ch) -> int {
        memset(ch.L->h_key, 0, ch.L->h_key_cap);
        for (size_t q = 0; q < ch.cnt; q++) {
            const size_t s = ch.s0 + q;
            if (!status[s]) p.down.add(out_at(s), ch.L->d_buf + sh_b + q * opitch, len[s]);
        }
        int r = p.down.flush(ctx, cudaMemcpyDeviceToHost, ch.L->stream);
        if (r) return r;
        CU_TRY(ctx, lane_wait(ctx, *ch.L));
        return GARAGE_EC_OK;
    };
    std::vector<garage_ec_range> runs;
    rc = p.run(
        [&](const HostChunk &ch) -> int {
            HostLane &L = *ch.L;
            wipe.use(&L);
            const size_t s0 = ch.s0, cnt = ch.cnt;
            uint8_t *d_sh = L.d_buf;
            // H2D: the planned runs; a request the plan cannot serve uploads nothing and fails on the device too
            for (size_t s = s0; s < s0 + cnt; s++) {
                int gpu = 0;
                runs.clear();
                if (open_range_runs(ctx, present + s * tot, sealed[s], offset[s], len[s], runs, &gpu)) continue;
                for (const garage_ec_range &r : runs)
                    p.up.add(d_sh + ((s - s0) * tot + r.shard) * stride + r.offset, shard_at(s, r.shard) + r.offset, r.len);
            }
            int r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
            if (r) return r;
            r = lane_key_staging(ctx, L, cs * 32);
            if (r) return r;
            memcpy(L.h_key, keys + s0 * 32, cnt * 32);
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_key, L.h_key, cnt * 32, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, present + s0 * tot, cnt * tot, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_sealed, sealed + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_off, offset + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_len, len + s0, cnt * 4, cudaMemcpyHostToDevice, L.stream));
            int32_t *d_status = reinterpret_cast<int32_t *>(L.d_small + o_status);
            r = with_stream_scratch(ctx, osc.bytes, L.stream, [&](uint8_t *sc) {
                const int e = run_open_range(ctx, d_sh, L.d_small + o_present,
                                             reinterpret_cast<const uint32_t *>(L.d_small + o_sealed), L.d_small + o_key,
                                             reinterpret_cast<const uint32_t *>(L.d_small + o_off),
                                             reinterpret_cast<const uint32_t *>(L.d_small + o_len), stride, d_sh + sh_b,
                                             opitch, d_status, cnt, sc, L.stream);
                const cudaError_t z = cudaMemsetAsync(sc + osc.o_keys, 0, cnt * sizeof(sse::SseKey), L.stream);
                if (e) return e;
                return z == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, z, "cudaMemsetAsync(key material)");
            });
            if (r) return r;
            CU_TRY(ctx, cudaMemsetAsync(L.d_small + o_key, 0, wipe.dev_bytes, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(status + s0, d_status, cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            return GARAGE_EC_OK;
        },
        retire);
    if (!rc) rc = p.drain(retire);
    wipe.failed = rc != 0;
    if (rc) return rc;
    int worst = GARAGE_EC_OK;
    for (size_t s = 0; s < n; s++) {
        if (status[s] == GARAGE_EC_E_UNRECOVERABLE) return GARAGE_EC_E_UNRECOVERABLE;
        if (status[s]) worst = status[s];
    }
    return worst;
}

int open_range_args(garage_ec_ctx *ctx, const void *shards, const uint8_t *present, const uint32_t *sealed,
                    const uint8_t *keys, const uint32_t *offset, const uint32_t *len, const int32_t *status,
                    size_t stride, size_t n)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, n, ctx->k + ctx->m);
    if (rc) return rc;
    if (n == 0) return GARAGE_EC_OK;
    if (!shards || !present || !sealed || !keys || !offset || !len || !status) return GARAGE_EC_E_INVALID;
    return GARAGE_EC_OK;
}

}  // namespace
extern "C" {

int garage_ec_sealed_range(uint32_t sealed_len, uint32_t offset, uint32_t len, uint32_t *span_off, uint32_t *span_len,
                           uint32_t *c0, uint32_t *n_chunks)
{
    if (!span_off || !span_len || !c0 || !n_chunks) return GARAGE_EC_E_INVALID;
    return sse::sealed_range(sealed_len, offset, len, span_off, span_len, c0, n_chunks);
}

int garage_ec_open_range_plan(const garage_ec_ctx *ctx, const uint8_t *present, uint32_t sealed_len, uint32_t offset,
                              uint32_t len, garage_ec_range *ranges, size_t cap, size_t *n_ranges, int *needs_gpu)
{
    if (!ctx || !present || !n_ranges || (cap && !ranges)) return GARAGE_EC_E_INVALID;
    *n_ranges = 0;
    if (needs_gpu) *needs_gpu = 0;
    std::vector<garage_ec_range> runs;
    int gpu = 0;
    const int rc = open_range_runs(ctx, present, sealed_len, offset, len, runs, &gpu);
    if (needs_gpu) *needs_gpu = gpu;
    if (rc) return rc;
    return merge_runs(runs, ranges, cap, n_ranges);
}

int garage_ec_open_range(garage_ec_ctx *ctx, const uint8_t *shards, const uint8_t *present, const uint32_t *sealed_len,
                         const uint8_t *keys, const uint32_t *offset, const uint32_t *len, size_t stride, uint8_t *out,
                         size_t out_stride, int32_t *status, size_t n, int mem_kind, void *cuda_stream)
{
    if (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE) return GARAGE_EC_E_INVALID;
    int rc = open_range_args(ctx, shards, present, sealed_len, keys, offset, len, status, stride, n);
    if (rc || n == 0) return rc;
    if (!out) return GARAGE_EC_E_INVALID;
    if (!aligned16(shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        return open_range_host(ctx, shards, nullptr, present, sealed_len, keys, offset, len, stride, out, out_stride,
                               nullptr, status, n);
    }
    if (!aligned16(out) || (out_stride & 15) || (reinterpret_cast<uintptr_t>(sealed_len) & 3) ||
        (reinterpret_cast<uintptr_t>(offset) & 3) || (reinterpret_cast<uintptr_t>(len) & 3) ||
        (reinterpret_cast<uintptr_t>(status) & 3))
        return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const OpenRangeScratch sc(ctx, n, stride, out_stride);
    return with_stream_scratch(ctx, sc.bytes, st, [&](uint8_t *scratch) {
        const int r = run_open_range(ctx, shards, present, sealed_len, keys, offset, len, stride, out, out_stride, status,
                                     n, scratch, st);
        const cudaError_t e = cudaMemsetAsync(scratch + sc.o_keys, 0, n * sizeof(sse::SseKey), st);
        if (r) return r;
        return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "cudaMemsetAsync(key material)");
    });
}

int garage_ec_open_range_stripes(garage_ec_ctx *ctx, const uint8_t *const *stripes, const uint8_t *present,
                                 const uint32_t *sealed_len, const uint8_t *keys, const uint32_t *offset,
                                 const uint32_t *len, size_t stride, uint8_t *const *outs, int32_t *status, size_t n)
{
    int rc = open_range_args(ctx, stripes, present, sealed_len, keys, offset, len, status, stride, n);
    if (rc || n == 0) return rc;
    if (!outs) return GARAGE_EC_E_INVALID;
    for (size_t s = 0; s < n; s++) {
        if (!stripes[s]) return GARAGE_EC_E_INVALID;
        if (!aligned16(stripes[s])) return GARAGE_EC_E_ALIGN;
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return open_range_host(ctx, nullptr, stripes, present, sealed_len, keys, offset, len, stride, nullptr, 0, outs,
                           status, n);
}

// --------------------------------------------------------------------------- SSE-C RESEAL (DESIGN.md 2.8, 4.11)
}  // extern "C"
namespace {

static_assert(sizeof(garage_ec_piece) == 12, "garage_ec_piece is three uint32 words");

// Device scratch of a reseal of n_src sources into n_dst destinations: key material (sources, then destinations) |
// source L | reconstruct status | want | plan | destination |Q|, len(B'), L', checksum accumulator.  The key material
// comes first so that one memset clears every secret.
struct ResealScratch {
    size_t o_keys, keys_bytes, o_src_L, o_rec, o_want, o_plan, o_plen, o_blen, o_dst_L, o_crc, bytes;
    ResealScratch(const garage_ec_ctx *ctx, size_t n_src, size_t n_dst)
    {
        size_t b = 0;
        auto take = [&](size_t x) {
            const size_t o = b;
            b += align_up(x, 256);
            return o;
        };
        keys_bytes = (n_src + n_dst) * sizeof(sse::SseKey);
        o_keys = take(keys_bytes);
        o_src_L = take(n_src * 4);
        o_rec = take(n_src * 4);
        o_want = take(n_src * (size_t)(ctx->k + ctx->m));
        o_plan = take(plan_scratch_bytes(ctx, n_src));
        o_plen = take(n_dst * 4);
        o_blen = take(n_dst * 4);
        o_dst_L = take(n_dst * 4);
        o_crc = take(n_dst * 4);
        bytes = b;
    }
};

// Reseal on the device: framing, piece lists and lengths, key schedules, the rebuild of absent source data shards,
// the sources' content hashes and (keyed) every chunk tag, the destinations' verdicts, the fused decrypt-and-seal
// into the destination data shards (crc_kind != NULL: and the checksums of Q_d into crcs), the code's encode, the
// destinations' content hashes and (sums != NULL) their shard tags.  The caller zeroes the key material of `scratch`.
int run_reseal(garage_ec_ctx *ctx, uint8_t *src_shards, const uint8_t *src_present, const uint32_t *src_len,
               const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src, const uint32_t *pieces,
               const uint32_t *piece_start, const uint8_t *dst_keys, const uint8_t *dst_nonces, uint8_t *dst_shards,
               uint8_t *dst_hashes, uint8_t *dst_sums, uint32_t *dst_len_out, uint8_t *src_hash_bad,
               int32_t *src_status, int32_t *status, const uint8_t *crc_kind, uint32_t *crcs, size_t stride,
               size_t n_dst, uint8_t *scratch, cudaStream_t st)
{
    const ResealScratch sc(ctx, n_src, n_dst);
    const size_t tot = ctx->k + ctx->m, nmax = std::max(n_src, n_dst);
    sse::SseKey *ks = reinterpret_cast<sse::SseKey *>(scratch + sc.o_keys);
    uint32_t *src_L = reinterpret_cast<uint32_t *>(scratch + sc.o_src_L), *plen = reinterpret_cast<uint32_t *>(scratch + sc.o_plen),
             *blen = reinterpret_cast<uint32_t *>(scratch + sc.o_blen), *dst_L = reinterpret_cast<uint32_t *>(scratch + sc.o_dst_L);
    int32_t *rec = reinterpret_cast<int32_t *>(scratch + sc.o_rec);
    const unsigned grid = (unsigned)std::min<size_t>((nmax + 255) / 256, (size_t)ctx->sm_count * 4);
    sse::ResealLensParams lp;
    memset(&lp, 0, sizeof(lp));
    lp.src_len = src_len;
    lp.pieces = pieces;
    lp.piece_start = piece_start;
    lp.src_status = src_status;
    lp.src_L = src_L;
    lp.want = scratch + sc.o_want;
    lp.status = status;
    lp.dst_plen = plen;
    lp.dst_blen = blen;
    lp.dst_L = dst_L;
    lp.stride = (uint32_t)stride;
    lp.k = (uint32_t)ctx->k;
    lp.m = (uint32_t)ctx->m;
    lp.n_src = (uint32_t)n_src;
    lp.n_dst = (uint32_t)n_dst;
    lp.quantum = ctx->quantum;
    lp.keyed = src_keys ? 1u : 0u;
    sse::sse_reseal_lens_kernel<<<grid, 256, 0, st>>>(lp);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    sse::CrcPassParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.kind = crc_kind;
    cp.acc = reinterpret_cast<uint32_t *>(scratch + sc.o_crc);
    cp.shard_len = dst_L;
    cp.status = status;
    cp.plain_len = plen;
    cp.crcs = crcs;
    cp.n = (uint32_t)n_dst;
    int rc = crc_kind ? sse_launch_crc_pass(ctx, cp, st) : GARAGE_EC_OK;
    if (!rc && src_keys && n_src) rc = sse_launch_setup(ctx, src_keys, ks, n_src, st);
    if (!rc) rc = sse_launch_setup(ctx, dst_keys, ks + n_src, n_dst, st);
    if (!rc && n_src)
        rc = run_reconstruct(ctx, src_shards, src_present, scratch + sc.o_want, rec, src_L, stride, n_src,
                             scratch + sc.o_plan, st);
    if (!rc && n_src) rc = sse_launch_block_sums(ctx, src_shards, src_len, src_hashes, src_hash_bad, nullptr, stride, n_src, st);
    if (rc) return rc;
    const uint32_t cmax = (uint32_t)std::max<size_t>(1, ((size_t)ctx->k * stride + sse::kChunk - 1) / sse::kChunk);
    sse::ChunkParams q;
    memset(&q, 0, sizeof(q));
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.cmax = cmax;
    if (src_keys && n_src) {
        q.blen = src_len;
        q.shard_len = src_L;
        q.ks = ks;
        q.shards = src_shards;
        q.status = src_status;
        q.rec_status = rec;
        q.n = (uint32_t)n_src;
        rc = sse_launch_chunks<sse::kCheck>(ctx, q, st);
        if (rc) return rc;
    }
    sse::ResealVerdictParams vp;
    memset(&vp, 0, sizeof(vp));
    vp.pieces = pieces;
    vp.piece_start = piece_start;
    vp.rec = rec;
    vp.hash_bad = src_hash_bad;
    vp.src_status = src_status;
    vp.status = status;
    vp.dst_blen = blen;
    vp.dst_L = dst_L;
    vp.dst_len_out = dst_len_out;
    vp.n_src = (uint32_t)n_src;
    vp.n_dst = (uint32_t)n_dst;
    sse::sse_reseal_verdict_kernel<<<grid, 256, 0, st>>>(vp);
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    CU_TRY(ctx, cudaGetLastError());
    memset(&q, 0, sizeof(q));
    q.plain_len = plen;
    q.blen = blen;
    q.shard_len = dst_L;
    q.nonces = dst_nonces;
    q.ks = ks + n_src;
    q.shards = dst_shards;
    q.stride = (uint32_t)stride;
    q.k = (uint32_t)ctx->k;
    q.m = (uint32_t)ctx->m;
    q.n = (uint32_t)n_dst;
    q.cmax = cmax;
    q.pieces = pieces;
    q.piece_start = piece_start;
    q.src_shards = src_shards;
    q.src_len = src_len;
    q.src_L = src_L;
    q.src_ks = src_keys ? ks : nullptr;
    q.crc_kind = crc_kind;
    q.crc_acc = cp.acc;
    rc = crc_kind ? sse_launch_chunks<sse::kReseal | sse::kCrc>(ctx, q, st) : sse_launch_chunks<sse::kReseal>(ctx, q, st);
    cp.final = 1;
    cp.status = nullptr;
    if (!rc && crc_kind) rc = sse_launch_crc_pass(ctx, cp, st);
    if (!rc)
        rc = run_uniform(ctx, kModeEncode, dst_shards, tot * stride, dst_shards + (size_t)ctx->k * stride, tot * stride,
                         nullptr, dst_L, stride, n_dst, st);
    if (!rc) rc = sse_launch_block_sums(ctx, dst_shards, blen, nullptr, nullptr, dst_hashes, stride, n_dst, st);
    if (!rc && dst_sums) rc = run_sums(ctx, dst_shards, nullptr, dst_L, stride, n_dst * tot, (int)tot, dst_sums, nullptr, st);
    return rc;
}

// The checks a HOST reseal makes before any GPU work: every source's L fits the stride and some piece names it, every
// destination has a well-formed piece list inside its sources' plaintext, and every L' fits the stride
int reseal_host_args_ok(garage_ec_ctx *ctx, const uint32_t *src_len, bool keyed, size_t n_src,
                        const garage_ec_piece *pieces, const uint32_t *piece_start, size_t stride, size_t n_dst)
{
    for (size_t i = 0; i < n_src; i++)
        if (code_shard_len(ctx, src_len[i]) > stride) return GARAGE_EC_E_INVALID;
    std::vector<uint8_t> named(n_src, 0);
    for (size_t d = 0; d < n_dst; d++) {
        if (piece_start[d + 1] <= piece_start[d]) return GARAGE_EC_E_INVALID;
        uint64_t Q = 0;
        for (uint32_t p = piece_start[d]; p < piece_start[d + 1]; p++) {
            const garage_ec_piece &x = pieces[p];
            if (x.src >= n_src || !x.len) return GARAGE_EC_E_INVALID;
            named[x.src] = 1;
            const int64_t P = keyed ? sse_plain_len(src_len[x.src]) : (int64_t)src_len[x.src];
            if (P >= 0 && (int64_t)x.offset + x.len > P) return GARAGE_EC_E_INVALID;  // P < 0: the source fails AUTH
            Q += x.len;
        }
        const uint64_t B = sse::sealed_len(Q);
        if (B > 0xffffffffull || code_shard_len(ctx, (uint32_t)B) > stride) return GARAGE_EC_E_INVALID;
    }
    for (size_t i = 0; i < n_src; i++)
        if (!named[i]) return GARAGE_EC_E_INVALID;  // a chunk uploads only the sources its pieces name
    return GARAGE_EC_OK;
}

// HOST reseal.  src_stripes != NULL: the gather form.  The pipeline chunks the destinations; a chunk uploads the
// distinct sources its pieces name (a source two chunks name is uploaded and proven by both), renumbers their pieces,
// and uploads only what garage_ec_open would upload of each: ciphertext.  Only roundup16(L') bytes of the k+m shards of the destinations that passed come down.
int reseal_host(garage_ec_ctx *ctx, const uint8_t *src_shards, const uint8_t *const *src_stripes,
                const uint8_t *src_present, const uint32_t *src_len, const uint8_t *src_hashes, const uint8_t *src_keys,
                size_t n_src, const garage_ec_piece *pieces, const uint32_t *piece_start, const uint8_t *dst_keys,
                const uint8_t *dst_nonces, uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums,
                uint32_t *dst_len_out, uint8_t *src_hash_bad, int32_t *src_status, int32_t *status,
                const uint8_t *crc_kind, uint32_t *crcs, size_t stride, size_t n_dst)
{
    const size_t k = ctx->k, tot = ctx->k + ctx->m;
    auto shard_at = [&](size_t i, size_t j) {
        return src_stripes ? src_stripes[i] + j * stride : src_shards + (i * tot + j) * stride;
    };
    // per destination: its own shards and those of the most distinct sources one destination names, so that a
    // chunk's sources and destinations fit the pipeline's chunk budget (or one destination's worth when that is more)
    std::vector<size_t> last(n_src, SIZE_MAX);
    size_t per_dst = 1;
    for (size_t d = 0; d < n_dst; d++) {
        size_t cnt = 0;
        for (uint32_t x = piece_start[d]; x < piece_start[d + 1]; x++)
            if (last[pieces[x].src] != d) {
                last[pieces[x].src] = d;
                cnt++;
            }
        per_dst = std::max(per_dst, cnt);
    }
    LaneKeyWipe wipe;  // outlives p: p's destructor runs wipe.wipe()
    HostPipeline p(ctx, n_dst, (1 + per_dst) * tot * stride);
    const size_t cs = p.cs, nch = (n_dst + cs - 1) / cs;
    std::vector<std::vector<uint32_t>> srcs(nch);
    last.assign(n_src, SIZE_MAX);
    size_t max_src = 1, max_pieces = 1;
    for (size_t c = 0; c < nch; c++) {
        const size_t d0 = c * cs, d1 = std::min(n_dst, d0 + cs);
        for (uint32_t x = piece_start[d0]; x < piece_start[d1]; x++)
            if (last[pieces[x].src] != c) {
                last[pieces[x].src] = c;
                srcs[c].push_back(pieces[x].src);
            }
        max_pieces = std::max<size_t>(max_pieces, piece_start[d1] - piece_start[d0]);
    }
    for (const auto &v : srcs) max_src = std::max(max_src, v.size());
    std::vector<uint32_t> local(n_src);
    std::vector<uint8_t> want(tot);
    for (size_t j = 0; j < tot; j++) want[j] = j < k;

    p.before_release = [&wipe] { wipe.wipe(); };
    SmallLayout sl;
    const ResealScratch sc(ctx, max_src, cs);
    // device small buffer: scratch | keys and nonces | the uploaded tables | the downloaded verdicts | hashes | sums;
    // the lane's pageable staging mirrors [o_present, o_dhash)
    const size_t o_scr = sl.take(sc.bytes), o_key = sl.take(max_src * 32 + cs * 40), o_present = sl.take(max_src * tot),
                 o_slen = sl.take(max_src * 4), o_shash = sl.take(max_src * 32), o_pieces = sl.take(max_pieces * 12),
                 o_pstart = sl.take((cs + 1) * 4), o_sbad = sl.take(max_src), o_sstatus = sl.take(max_src * 4),
                 o_dlen = sl.take(cs * 4), o_status = sl.take(cs * 4), o_dhash = sl.take(cs * 32),
                 o_dsums = sl.take(dst_sums ? cs * tot * 32 : 0), o_kind = sl.take(crc_kind ? cs : 0),
                 o_crcs = sl.take(crc_kind ? cs * 4 : 0);
    wipe.dev_off = o_scr;
    wipe.dev_bytes = o_present - o_scr;
    const size_t src_b = align_up(max_src * tot * stride, 256);
    int rc = p.reserve(src_b + cs * tot * stride, sl.bytes, o_dhash - o_present);
    if (rc) return rc;
    bool pinned = true;
    for (size_t i = 0; pinned && i < (src_stripes ? n_src : 1); i++) pinned = device_addressable_host(shard_at(i, 0));
    p.up.use_batch = pinned;
    p.down.use_batch = device_addressable_host(dst_shards);
    auto at = [](const HostChunk &ch, size_t o, size_t base) { return ch.host + (o - base); };
    const Retire retire = [&](const HostChunk &ch) -> int {
        memset(ch.L->h_key, 0, ch.L->h_key_cap);
        const std::vector<uint32_t> &S = srcs[ch.s0 / cs];
        const uint8_t *sbad = at(ch, o_sbad, o_present);
        const int32_t *sst = reinterpret_cast<const int32_t *>(at(ch, o_sstatus, o_present)),
                      *dst = reinterpret_cast<const int32_t *>(at(ch, o_status, o_present));
        const uint32_t *dlen = reinterpret_cast<const uint32_t *>(at(ch, o_dlen, o_present));
        for (size_t li = 0; li < S.size(); li++) {
            src_hash_bad[S[li]] = sbad[li];
            src_status[S[li]] = sst[li];
        }
        const uint8_t *d_dst = ch.L->d_buf + src_b;
        for (size_t q = 0; q < ch.cnt; q++) {
            const size_t d = ch.s0 + q;
            status[d] = dst[q];
            if (dst[q]) continue;
            dst_len_out[d] = dlen[q];
            const size_t bytes = align_up(code_shard_len(ctx, dlen[q]), 16);
            for (size_t j = 0; j < tot; j++) p.down.add(dst_shards + (d * tot + j) * stride, d_dst + (q * tot + j) * stride, bytes);
        }
        int r = p.down.flush(ctx, cudaMemcpyDeviceToHost, ch.L->stream);
        if (r) return r;
        CU_TRY(ctx, lane_wait(ctx, *ch.L));
        return GARAGE_EC_OK;
    };
    rc = p.run(
        [&](const HostChunk &ch) -> int {
            HostLane &L = *ch.L;
            wipe.use(&L);
            const size_t s0 = ch.s0, cnt = ch.cnt;
            const std::vector<uint32_t> &S = srcs[s0 / cs];
            uint8_t *d_src = L.d_buf, *d_dst = L.d_buf + src_b;
            int r = lane_key_staging(ctx, L, max_src * 32 + cs * 40);
            if (r) return r;
            uint8_t *h_present = at(ch, o_present, o_present), *h_shash = at(ch, o_shash, o_present);
            uint32_t *h_slen = reinterpret_cast<uint32_t *>(at(ch, o_slen, o_present)),
                     *h_pieces = reinterpret_cast<uint32_t *>(at(ch, o_pieces, o_present)),
                     *h_pstart = reinterpret_cast<uint32_t *>(at(ch, o_pstart, o_present));
            // H2D: the present data shards of each source and what the code's plan reads to rebuild the others
            for (size_t li = 0; li < S.size(); li++) {
                const size_t i = S[li];
                local[i] = (uint32_t)li;
                const uint8_t *pr = src_present + i * tot;
                memcpy(h_present + li * tot, pr, tot);
                h_slen[li] = src_len[i];
                memcpy(h_shash + li * 32, src_hashes + i * 32, 32);
                if (src_keys) memcpy(L.h_key + li * 32, src_keys + i * 32, 32);
                uint64_t hv = 0;
                const size_t len = code_shard_len(ctx, src_len[i]);
                const bool ok = stripe_read_plan(ctx, pr, want.data(), &hv);
                for (size_t j = 0; j < tot; j++) {
                    uint8_t *dp = d_src + (li * tot + j) * stride;
                    if (j < k && pr[j]) p.up.add(dp, shard_at(i, j), align_up(len, 16));
                    else if (ok && j >= k)
                        for_each_read_piece(ctx, hv, j, len, align_up(len, 16),
                                            [&](size_t off, size_t bytes) { p.up.add(dp + off, shard_at(i, j) + off, bytes); });
                }
            }
            const uint32_t pbase = piece_start[s0];
            for (size_t q = 0; q <= cnt; q++) h_pstart[q] = piece_start[s0 + q] - pbase;
            for (uint32_t x = pbase; x < piece_start[s0 + cnt]; x++) {
                h_pieces[3 * (x - pbase)] = local[pieces[x].src];
                h_pieces[3 * (x - pbase) + 1] = pieces[x].offset;
                h_pieces[3 * (x - pbase) + 2] = pieces[x].len;
            }
            memcpy(L.h_key + max_src * 32, dst_keys + s0 * 32, cnt * 32);
            memcpy(L.h_key + max_src * 32 + cs * 32, dst_nonces + s0 * 8, cnt * 8);
            r = p.up.flush(ctx, cudaMemcpyHostToDevice, L.stream);
            if (r) return r;
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_key, L.h_key, max_src * 32 + cs * 40, cudaMemcpyHostToDevice, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_present, ch.host, o_sbad - o_present, cudaMemcpyHostToDevice, L.stream));
            if (crc_kind)
                CU_TRY(ctx, cudaMemcpyAsync(L.d_small + o_kind, crc_kind + s0, cnt, cudaMemcpyHostToDevice, L.stream));
            auto u32 = [&](size_t o) { return reinterpret_cast<uint32_t *>(L.d_small + o); };
            r = run_reseal(ctx, d_src, L.d_small + o_present, u32(o_slen), L.d_small + o_shash,
                           src_keys ? L.d_small + o_key : nullptr, S.size(), u32(o_pieces), u32(o_pstart),
                           L.d_small + o_key + max_src * 32, L.d_small + o_key + max_src * 32 + cs * 32, d_dst,
                           L.d_small + o_dhash, dst_sums ? L.d_small + o_dsums : nullptr, u32(o_dlen), L.d_small + o_sbad,
                           reinterpret_cast<int32_t *>(u32(o_sstatus)), reinterpret_cast<int32_t *>(u32(o_status)),
                           crc_kind ? L.d_small + o_kind : nullptr, u32(o_crcs), stride, cnt, L.d_small + o_scr, L.stream);
            if (r) return r;
            CU_TRY(ctx, cudaMemsetAsync(L.d_small + o_scr, 0, wipe.dev_bytes, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(at(ch, o_sbad, o_present), L.d_small + o_sbad, o_dhash - o_sbad,
                                        cudaMemcpyDeviceToHost, L.stream));
            CU_TRY(ctx, cudaMemcpyAsync(dst_hashes + s0 * 32, L.d_small + o_dhash, cnt * 32, cudaMemcpyDeviceToHost, L.stream));
            if (dst_sums)
                CU_TRY(ctx, cudaMemcpyAsync(dst_sums + s0 * tot * 32, L.d_small + o_dsums, cnt * tot * 32,
                                            cudaMemcpyDeviceToHost, L.stream));
            if (crc_kind) CU_TRY(ctx, cudaMemcpyAsync(crcs + s0, u32(o_crcs), cnt * 4, cudaMemcpyDeviceToHost, L.stream));
            return GARAGE_EC_OK;
        },
        retire);
    if (!rc) rc = p.drain(retire);
    wipe.failed = rc != 0;
    if (rc) return rc;
    int worst = GARAGE_EC_OK;
    for (size_t d = 0; d < n_dst; d++) {
        if (status[d] == GARAGE_EC_E_UNRECOVERABLE) return GARAGE_EC_E_UNRECOVERABLE;
        if (status[d]) worst = status[d];
    }
    return worst;
}

int reseal_args(garage_ec_ctx *ctx, const void *src_shards, const uint8_t *src_present, const uint32_t *src_len,
                const uint8_t *src_hashes, size_t n_src, const garage_ec_piece *pieces, const uint32_t *piece_start,
                const uint8_t *dst_keys, const uint8_t *dst_nonces, const uint8_t *dst_shards, const uint8_t *dst_hashes,
                const uint32_t *dst_len_out, const uint8_t *src_hash_bad, const int32_t *src_status,
                const int32_t *status, const uint8_t *crc_kind, const uint32_t *crcs, size_t stride, size_t n_dst)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    int rc = check_geometry(ctx, stride, std::max(n_src, n_dst), ctx->k + ctx->m);
    if (rc) return rc;
    if (n_dst == 0) return GARAGE_EC_OK;
    if (!piece_start || !pieces || !dst_keys || !dst_nonces || !dst_shards || !dst_hashes || !dst_len_out || !status ||
        (crc_kind && !crcs))
        return GARAGE_EC_E_INVALID;
    if (n_src && (!src_shards || !src_present || !src_len || !src_hashes || !src_hash_bad || !src_status))
        return GARAGE_EC_E_INVALID;
    if (!aligned16(dst_shards)) return GARAGE_EC_E_ALIGN;
    return GARAGE_EC_OK;
}

}  // namespace
extern "C" {

int garage_ec_reseal_crc(garage_ec_ctx *ctx, uint8_t *src_shards, const uint8_t *src_present, const uint32_t *src_len,
                         const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src, const garage_ec_piece *pieces,
                         const uint32_t *piece_start, const uint8_t *dst_keys, const uint8_t *dst_nonces,
                         uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums, uint32_t *dst_len_out,
                         uint8_t *src_hash_bad, int32_t *src_status, int32_t *status, const uint8_t *crc_kind,
                         uint32_t *crcs, size_t stride, size_t n_dst, int mem_kind, void *cuda_stream)
{
    if (mem_kind != GARAGE_EC_MEM_HOST && mem_kind != GARAGE_EC_MEM_DEVICE) return GARAGE_EC_E_INVALID;
    int rc = reseal_args(ctx, src_shards, src_present, src_len, src_hashes, n_src, pieces, piece_start, dst_keys,
                         dst_nonces, dst_shards, dst_hashes, dst_len_out, src_hash_bad, src_status, status, crc_kind, crcs,
                         stride, n_dst);
    if (rc || n_dst == 0) return rc;
    if (n_src && !aligned16(src_shards)) return GARAGE_EC_E_ALIGN;
    if (mem_kind == GARAGE_EC_MEM_HOST) {
        rc = reseal_host_args_ok(ctx, src_len, src_keys != nullptr, n_src, pieces, piece_start, stride, n_dst);
        if (!rc) rc = crc_kinds_ok(crc_kind, n_dst);
        if (rc) return rc;
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        return reseal_host(ctx, src_shards, nullptr, src_present, src_len, src_hashes, src_keys, n_src, pieces,
                           piece_start, dst_keys, dst_nonces, dst_shards, dst_hashes, dst_sums, dst_len_out,
                           src_hash_bad, src_status, status, crc_kind, crcs, stride, n_dst);
    }
    for (const void *p : {(const void *)src_len, (const void *)pieces, (const void *)piece_start, (const void *)dst_len_out,
                          (const void *)src_status, (const void *)status, (const void *)crcs})
        if (reinterpret_cast<uintptr_t>(p) & 3) return GARAGE_EC_E_ALIGN;
    if ((reinterpret_cast<uintptr_t>(src_hashes) & 7) || (reinterpret_cast<uintptr_t>(dst_hashes) & 7) ||
        (reinterpret_cast<uintptr_t>(dst_sums) & 7))
        return GARAGE_EC_E_ALIGN;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const ResealScratch sc(ctx, n_src, n_dst);
    return with_stream_scratch(ctx, sc.bytes, st, [&](uint8_t *scratch) {
        const int r = run_reseal(ctx, src_shards, src_present, src_len, src_hashes, src_keys, n_src,
                                 reinterpret_cast<const uint32_t *>(pieces), piece_start, dst_keys, dst_nonces, dst_shards,
                                 dst_hashes, dst_sums, dst_len_out, src_hash_bad, src_status, status, crc_kind, crcs,
                                 stride, n_dst, scratch, st);
        const cudaError_t e = cudaMemsetAsync(scratch + sc.o_keys, 0, sc.keys_bytes, st);
        if (r) return r;
        return e == cudaSuccess ? GARAGE_EC_OK : set_cuda_error(ctx, e, "cudaMemsetAsync(key material)");
    });
}

int garage_ec_reseal(garage_ec_ctx *ctx, uint8_t *src_shards, const uint8_t *src_present, const uint32_t *src_len,
                     const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src, const garage_ec_piece *pieces,
                     const uint32_t *piece_start, const uint8_t *dst_keys, const uint8_t *dst_nonces,
                     uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums, uint32_t *dst_len_out,
                     uint8_t *src_hash_bad, int32_t *src_status, int32_t *status, size_t stride, size_t n_dst,
                     int mem_kind, void *cuda_stream)
{
    return garage_ec_reseal_crc(ctx, src_shards, src_present, src_len, src_hashes, src_keys, n_src, pieces, piece_start,
                                dst_keys, dst_nonces, dst_shards, dst_hashes, dst_sums, dst_len_out, src_hash_bad,
                                src_status, status, nullptr, nullptr, stride, n_dst, mem_kind, cuda_stream);
}

int garage_ec_reseal_stripes_crc(garage_ec_ctx *ctx, uint8_t *const *src_stripes, const uint8_t *src_present,
                                 const uint32_t *src_len, const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src,
                                 const garage_ec_piece *pieces, const uint32_t *piece_start, const uint8_t *dst_keys,
                                 const uint8_t *dst_nonces, uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums,
                                 uint32_t *dst_len_out, uint8_t *src_hash_bad, int32_t *src_status, int32_t *status,
                                 const uint8_t *crc_kind, uint32_t *crcs, size_t stride, size_t n_dst)
{
    int rc = reseal_args(ctx, src_stripes, src_present, src_len, src_hashes, n_src, pieces, piece_start, dst_keys,
                         dst_nonces, dst_shards, dst_hashes, dst_len_out, src_hash_bad, src_status, status, crc_kind, crcs,
                         stride, n_dst);
    if (rc || n_dst == 0) return rc;
    for (size_t i = 0; i < n_src; i++) {
        if (!src_stripes[i]) return GARAGE_EC_E_INVALID;
        if (!aligned16(src_stripes[i])) return GARAGE_EC_E_ALIGN;
    }
    rc = reseal_host_args_ok(ctx, src_len, src_keys != nullptr, n_src, pieces, piece_start, stride, n_dst);
    if (!rc) rc = crc_kinds_ok(crc_kind, n_dst);
    if (rc) return rc;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    return reseal_host(ctx, nullptr, src_stripes, src_present, src_len, src_hashes, src_keys, n_src, pieces, piece_start,
                       dst_keys, dst_nonces, dst_shards, dst_hashes, dst_sums, dst_len_out, src_hash_bad, src_status,
                       status, crc_kind, crcs, stride, n_dst);
}

int garage_ec_reseal_stripes(garage_ec_ctx *ctx, uint8_t *const *src_stripes, const uint8_t *src_present,
                             const uint32_t *src_len, const uint8_t *src_hashes, const uint8_t *src_keys, size_t n_src,
                             const garage_ec_piece *pieces, const uint32_t *piece_start, const uint8_t *dst_keys,
                             const uint8_t *dst_nonces, uint8_t *dst_shards, uint8_t *dst_hashes, uint8_t *dst_sums,
                             uint32_t *dst_len_out, uint8_t *src_hash_bad, int32_t *src_status, int32_t *status,
                             size_t stride, size_t n_dst)
{
    return garage_ec_reseal_stripes_crc(ctx, src_stripes, src_present, src_len, src_hashes, src_keys, n_src, pieces,
                                        piece_start, dst_keys, dst_nonces, dst_shards, dst_hashes, dst_sums, dst_len_out,
                                        src_hash_bad, src_status, status, nullptr, nullptr, stride, n_dst);
}

// ---- test hook -------------------------------------------------------------------------------
int garage_ec_debug_fail_after(garage_ec_ctx *ctx, long n_calls)
{
    if (!ctx) return GARAGE_EC_E_INVALID;
    ctx->fault_countdown.store(n_calls, std::memory_order_relaxed);
    return GARAGE_EC_OK;
}

}  // extern "C"
