// libb200aa.so -- C ABI (include/b200aa.h) over the sm_90a kernels.
// Build: see pyaudioanalysis_b200/build.py (nvcc -gencode arch=compute_90a,code=sm_90a).
// This file holds the short-term path (plan, kernel 0, kernel 1, host-buffer entry points) and the shared error state;
// the other kernel families have a .cu each (DESIGN.md §4).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/b200aa.h"
#include "common.cuh"
#include "entry.h"
#include "generic_kernel.cuh"
#include "fast_kernel.cuh"
#include "pair_kernel.cuh"
#include "slots.h"
#include "solo_kernel.cuh"
#include "tables.inl"

using namespace b200aa;

// the error state of every entry point in every file (entry.h)
thread_local std::string g_cuda_err;
std::atomic<int64_t> g_launches{0};

extern "C" int b200aa_abi_version(void) { return B200AA_ABI_VERSION; }
extern "C" int64_t b200aa_launch_count(void) { return g_launches.load(); }
extern "C" const char *b200aa_last_cuda_error(void) { return g_cuda_err.c_str(); }

extern "C" const char *b200aa_status_string(int s)
{
    switch (s) {
    case B200AA_OK: return "ok";
    case B200AA_ERR_INVALID: return "invalid argument";
    case B200AA_ERR_TOO_SHORT: return "need at least one array to concatenate";   // the reference's text
    case B200AA_ERR_CHROMA: return "chroma: semitone index >= num_fft (window too short for this sampling rate)";
    case B200AA_ERR_MEL_RANGE: return "mel filterbank: filter edge beyond num_fft";
    case B200AA_ERR_CUDA: return "CUDA error";
    case B200AA_ERR_UNSUPPORTED: return "window too large for the on-chip transform";
    case B200AA_ERR_NO_DEVICE: return "no sm_90 CUDA device";
    case B200AA_ERR_CAPTURE: return "this call cannot be captured; make it once outside capture first, or call it eagerly";
    default: return "unknown status";
    }
}

extern "C" int b200aa_device_ok(void)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return B200AA_ERR_NO_DEVICE; }
    cudaDeviceProp pr;
    if (cudaGetDeviceProperties(&pr, dev) != cudaSuccess) { cudaGetLastError(); return B200AA_ERR_NO_DEVICE; }
    return (pr.major == 9 && pr.minor == 0) ? B200AA_OK : B200AA_ERR_NO_DEVICE;
}

// ------------------------------------------------------------------------------------------------
// host tables / counts
// ------------------------------------------------------------------------------------------------
extern "C" int b200aa_host_table(int fs, int window, int which, double *h_out)
{
    if (!h_out || window < 2 || fs <= 0) return B200AA_ERR_INVALID;
    const int K = window / 2;
    std::vector<double> t;
    int rc = B200AA_OK;
    if (which == 0) rc = b200aa_host::build_mel(fs, K, t);
    else if (which == 1) rc = b200aa_host::build_chroma(fs, K, t);
    else if (which == 2) b200aa_host::build_dct(t);
    else return B200AA_ERR_INVALID;
    if (rc != B200AA_OK) return rc;
    std::memcpy(h_out, t.data(), t.size() * sizeof(double));
    return B200AA_OK;
}

extern "C" int64_t b200aa_num_frames(int64_t n, int w, int s)
{
    return (w < 1 || s < 1) ? 0 : rows::frames(n, w, s);
}
extern "C" int64_t b200aa_spectrogram_rows(int64_t n, int w, int s)
{
    return (w < 1 || s < 1) ? 0 : rows::spectrogram(n, w, s).R;
}
extern "C" int64_t b200aa_chromagram_rows(int64_t n, int w, int s)
{
    return (w < 1 || s < 1) ? 0 : rows::chromagram(n, w, s).R;
}

extern "C" int64_t b200aa_mid_windows(int64_t n_frames, int stepr) { return rows::windows_of(n_frames, stepr); }

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct Transform {           // the window's transform: packed real (even window) or complex, and its device twiddles
    int Nc = 0, packed = 0;
    std::vector<int> radix;
    b200aa_host::DeviceMemory tw, tw_post;      // float2 [Nc] each
};

// Device buffer that only grows, reused across calls (a cudaMalloc / cudaFree pair per call costs more than the kernels
// for a single clip)
struct GrowBuffer {
    b200aa_host::DeviceMemory p;
    size_t cap = 0;
    // at least `need` bytes: when it holds fewer, it is reallocated to `want` (>= need) bytes
    cudaError_t reserve(size_t need, size_t want)
    {
        if (cap >= need) return cudaSuccess;
        clear();
        const cudaError_t e = b200aa_host::device_alloc(want, p);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void *get() const { return p.get(); }
    void clear() { p.reset(); cap = 0; }
};

// the work-slot ring's event operations (csrc/slots.h) on CUDA events
struct CudaSlotOps {
    using Event = cudaEvent_t;
    using Stream = cudaStream_t;
    static int create(cudaEvent_t &e)
    {
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        return B200AA_OK;
    }
    static int record(cudaEvent_t e, cudaStream_t st)
    {
        CK(cudaEventRecord(e, st));
        return B200AA_OK;
    }
    static int wait(cudaStream_t st, cudaEvent_t e)
    {
        CK(cudaStreamWaitEvent(st, e, 0));
        return B200AA_OK;
    }
    static void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
};

struct b200aa_plan {
    int fs = 0, window = 0, step = 0, K = 0;
    int device = 0, sm_count = 0;
    int force_generic = 0;
    int fast_kind = 0;                  // 0 = none, else index of the specialised kernel
    int tables_status = B200AA_OK;      // B200AA_ERR_CHROMA / _MEL_RANGE when the reference cannot build its tables
    BlobLayout bl{};
    b200aa_host::DeviceMemory blob;     // int [bl.words]
    Transform transform;
    // workspace of the host-buffer entry points; calls serialise on host_mu
    std::mutex host_mu;
    GrowBuffer ws[4];
    FastTables fast{};                  // extra device tables of the specialised kernel
    PairTables pair{};                  // inter-pass twiddles of the warp-autonomous pair kernel (windows 32 * R)
    SoloTables solo{};                  // tables of the warp-autonomous per-frame kernel (windows 882 / 400 / 600)
    int prefer = -1;                    // -1 = automatic, 0 / 1 / 2 / 3 = generic / register-tiled CTA / pair / solo kernel only (testing, A/B)
    // ring of work counters (one per in-flight launch of a persistent kernel, csrc/slots.h).  A slot is in flight from
    // acquire until its launch is queued and has recorded the slot's event; it is never handed to a second launch in that
    // time, and the next user's stream waits on that event, so it runs after the launch that used the slot last.
    // A slot is kSlotBytes wide: the CTA / solo / generic kernels use its first word as their work counter, the pair kernel
    // the whole slot as its per-warp range descriptors (csrc/sched.cuh: 8 bytes per resident warp).
    static constexpr unsigned kSlots = SlotRing<CudaSlotOps>::kSlots;
    static constexpr size_t kSlotBytes = 64 * 1024;
    b200aa_host::DeviceMemory counters;
    SlotRing<CudaSlotOps> slots;
    static constexpr int kPipe = 3;     // streams of the chunked host pipeline, each with its own clips / records / features buffers
    cudaStream_t pipe_stream[kPipe] = {nullptr, nullptr, nullptr};
    GrowBuffer pipe_ws[kPipe][3];
    // tables of the float64 path, built by its first call (f64.cu)
    std::mutex f64_mu;
    std::shared_ptr<const F64Tables> f64;
    ~b200aa_plan()
    {
        for (cudaStream_t s : pipe_stream) if (s) cudaStreamDestroy(s);
    }
};

extern "C" int b200aa_plan_create(b200aa_plan **out, int fs, int window, int step)
{
    if (!out || fs <= 0 || window < 2 || step < 1) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(nullptr, "b200aa_plan_create", kWhyAllocates);
    int rc = b200aa_device_ok();
    if (rc != B200AA_OK) return rc;
    std::unique_ptr<b200aa_plan> pl(new b200aa_plan);
    pl->fs = fs; pl->window = window; pl->step = step; pl->K = window / 2;
    CK(cudaGetDevice(&pl->device));
    CK(cudaDeviceGetAttribute(&pl->sm_count, cudaDevAttrMultiProcessorCount, pl->device));
    // tables that only feature_extraction / chromagram need may be unbuildable (the reference raises
    // there too); spectrogram must still work, so remember the status instead of failing here.
    std::vector<int> h_blob;
    pl->tables_status = b200aa_host::build_blob(fs, pl->K, h_blob, pl->bl);
    CK(b200aa_host::upload(h_blob, pl->blob));
    Transform &t = pl->transform;
    t.packed = (window % 2 == 0) ? 1 : 0;
    t.Nc = t.packed ? window / 2 : window;
    t.radix = b200aa_host::radix_list(t.Nc);
    if (t.Nc == 1) t.radix.clear();
    if ((int)t.radix.size() > kMaxRadix) return B200AA_ERR_UNSUPPORTED;
    CK(b200aa_host::upload(b200aa_host::twiddles(t.Nc, t.Nc), t.tw));
    CK(b200aa_host::upload(b200aa_host::twiddles(t.Nc, window), t.tw_post));
    rc = fast_plan_init(window, &pl->fast, &pl->fast_kind);
    if (rc != B200AA_OK) return rc;
    int sl_ = 0, sr_ = 0;
    if ((pair_r_for_window(window) || solo_shape_for_window(window, &sl_, &sr_)) && pl->tables_status == B200AA_OK) {
        std::vector<double> mel, chr, dct;
        b200aa_host::build_mel(fs, pl->K, mel);
        b200aa_host::build_chroma(fs, pl->K, chr);
        b200aa_host::build_dct(dct);
        std::vector<int> pblob;
        PairBlobLayout pbl{};
        build_pair_blob(mel, chr, dct, pl->K, pblob, pbl);
        rc = pair_plan_init(window, pblob, pbl, &pl->pair);
        if (rc != B200AA_OK) return cuda_fail(cudaGetLastError(), "pair_plan_init");
        rc = solo_plan_init(window, pblob, pbl, &pl->solo);
        if (rc != B200AA_OK) return cuda_fail(cudaGetLastError(), "solo_plan_init");
    }
    CK(b200aa_host::device_alloc(b200aa_plan::kSlots * b200aa_plan::kSlotBytes, pl->counters));
    *out = pl.release();
    return B200AA_OK;
}

extern "C" void b200aa_plan_destroy(b200aa_plan *plan) { delete plan; }
// One launch of a persistent kernel: the constructor takes a work-counter slot of the plan's ring (status in rc, counter
// in ctr), finish() gets the launcher's status, counts the launch, maps the status and frees the slot.
// B200AA_ERR_UNSUPPORTED = the launcher declined the shape and launched nothing; the caller tries the next kernel.
// On a capturing stream the slot is the launch's own stream-ordered scratch instead (an allocation and a free node of the
// graph): the ring's events cannot be waited on or recorded across a capture, and a graph keeps its slot for every replay,
// so a ring slot would be handed to eager launches that run at the same time as a replay.  The launcher zeroes either
// slot on the stream before its kernel.
struct SlotLaunch {
    b200aa_plan *pl;
    cudaStream_t st;
    unsigned slot = 0;
    unsigned int *ctr = nullptr;
    int rc;
    bool captured = false;
    StreamScratch own;
    SlotLaunch(b200aa_plan *plan, cudaStream_t stream) : pl(plan), st(stream), own(stream)
    {
        if (stream_capturing(st)) {
            captured = true;
            rc = own.alloc(b200aa_plan::kSlotBytes);
            ctr = static_cast<unsigned int *>(own.get());
            return;
        }
        rc = pl->slots.acquire(st, slot);
        if (rc == B200AA_OK)
            ctr = reinterpret_cast<unsigned int *>(static_cast<unsigned char *>(pl->counters.get()) + size_t(slot) * b200aa_plan::kSlotBytes);
    }
    int finish(int launch_rc, const char *name)
    {
        const int r = launch_rc == B200AA_OK ? launched(name)
                                             : (launch_rc == B200AA_ERR_CUDA ? cuda_fail(cudaGetLastError(), name) : launch_rc);
        if (captured) return own.done(r);
        const int done = pl->slots.done(st, slot);    // after launched(): a failed record keeps its own message
        return r != B200AA_OK ? r : done;
    }
};

static bool use_pair(const b200aa_plan *pl) { return pl->pair.R && !pl->force_generic && (pl->prefer < 0 || pl->prefer == 2); }
static bool use_solo(const b200aa_plan *pl) { return pl->solo.L && !pl->force_generic && (pl->prefer < 0 || pl->prefer == 3); }
static bool use_fast(const b200aa_plan *pl) { return pl->fast_kind && !pl->force_generic && (pl->prefer < 0 || pl->prefer == 1); }
extern "C" int b200aa_plan_kernel_kind(const b200aa_plan *plan)
{
    if (!plan) return 0;
    return use_pair(plan) ? 2 : (use_solo(plan) ? 3 : (use_fast(plan) ? 1 : 0));
}
extern "C" int b200aa_plan_prefer_kernel(b200aa_plan *plan, int kind)
{
    if (!plan || kind < -1 || kind > 3) return B200AA_ERR_INVALID;
    plan->prefer = kind;
    return B200AA_OK;
}
static float *g_pair_dump = nullptr;
extern "C" int b200aa_debug_set_dump(float *d_rows)
{
    g_pair_dump = d_rows;
    return B200AA_OK;
}
extern "C" int b200aa_plan_force_generic(b200aa_plan *plan, int on)
{
    if (!plan) return 0;
    int prev = plan->force_generic;
    plan->force_generic = on ? 1 : 0;
    return prev;
}

// free the grow-only workspaces of the host-buffer entry points (they are re-allocated on demand)
extern "C" int b200aa_plan_trim(b200aa_plan *plan)
{
    if (!plan) return B200AA_ERR_INVALID;
    std::lock_guard<std::mutex> g(plan->host_mu);
    for (GrowBuffer &w : plan->ws) w.clear();
    for (auto &stream_ws : plan->pipe_ws)
        for (GrowBuffer &w : stream_ws) w.clear();
    return B200AA_OK;
}

// a plan's tables live on the device that was current when it was created
static int plan_device_check(const b200aa_plan *pl)
{
    int dev = -1;
    CK(cudaGetDevice(&dev));
    return dev == pl->device ? B200AA_OK : B200AA_ERR_INVALID;
}

int plan_f64(const b200aa_plan *plan, PlanF64 &out)
{
    out = PlanF64{plan->fs, plan->window, plan->step, plan->K, plan->sm_count, plan->tables_status, nullptr};
    return B200AA_OK;
}

int plan_f64_device(const b200aa_plan *plan) { return plan_device_check(plan); }

int plan_f64_tables(const b200aa_plan *plan, PlanF64 &out, cudaStream_t st, const char *entry)
{
    int rc = plan_device_check(plan);
    if (rc != B200AA_OK) return rc;
    b200aa_plan *pl = const_cast<b200aa_plan *>(plan);
    std::lock_guard<std::mutex> g(pl->f64_mu);
    if (!pl->f64) {         // the build allocates and copies synchronously
        if ((rc = refuse_capture(st, entry, "the plan's float64 tables are built by its first float64 call; make one "
                                            "outside capture first")) != B200AA_OK)
            return rc;
        if ((rc = f64_tables_build(pl->fs, pl->window, pl->tables_status, pl->f64)) != B200AA_OK) return rc;
    }
    out.tables = pl->f64.get();
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel 0: clip statistics  (signal / 2**15 + dc_normalize, ShortTermFeatures.py:567-570, :14-19)
// accumulators live in the output records: rsv[1..2] (8-byte aligned) = sum (int64 / double), lo/hi = min/max keys
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int float_key(float f)
{
    int b = __float_as_int(f);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float key_float(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

__global__ void stats_init_kernel(b200aa_clip_norm *nm, int64_t n)
{
    int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(&nm[i].rsv[1]);
    *acc = 0ull;
    reinterpret_cast<int *>(&nm[i].lo)[0] = 0x7fffffff;              // running min key
    reinterpret_cast<int *>(&nm[i].hi)[0] = int(0x80000000u);        // running max key
}

template <int DTYPE>
__global__ void __launch_bounds__(256) stats_accum_kernel(const void *sig, int64_t n_samples, int64_t clip_stride,
                                                           const int64_t *len, b200aa_clip_norm *nm, int chunks)
{
    const int64_t b = blockIdx.y;
    const int64_t L = len ? len[b] : n_samples;
    const int64_t per = (L + chunks - 1) / chunks;
    const int64_t s0 = blockIdx.x * per, s1 = min(L, s0 + per);
    long long isum = 0;
    double dsum = 0.0;
    int kmin = 0x7fffffff, kmax = int(0x80000000u);
    if (DTYPE == B200AA_DTYPE_I16) {
        const short *x = reinterpret_cast<const short *>(sig) + b * clip_stride;
        int mn = 32767, mx = -32768;
        int64_t i = s0 + threadIdx.x;
        // 16-byte vector body when the chunk start is aligned
        const bool al = ((reinterpret_cast<uintptr_t>(x + s0) & 15) == 0);
        if (al) {
            const int4 *v = reinterpret_cast<const int4 *>(x + s0);
            const int64_t nv = (s1 - s0) / 8;
            // four 16-byte loads in flight per thread (the kernel is a pure HBM stream: memory-level parallelism is all it needs)
            int64_t j = threadIdx.x;
            for (; j + 3 * int64_t(blockDim.x) < nv; j += 4 * int64_t(blockDim.x)) {
                int4 q[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) q[t] = __ldg(v + j + t * int64_t(blockDim.x));
                int acc = 0;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const int w4[4] = {q[t].x, q[t].y, q[t].z, q[t].w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int a0 = (short)(w4[u] & 0xffff), a1 = w4[u] >> 16;
                        acc += a0 + a1;
                        mn = min(mn, min(a0, a1));
                        mx = max(mx, max(a0, a1));
                    }
                }
                isum += acc;
            }
            for (; j < nv; j += blockDim.x) {
                int acc = 0;
                const int4 q = __ldg(v + j);
                const int w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int a0 = (short)(w4[u] & 0xffff), a1 = w4[u] >> 16;
                    acc += a0 + a1;
                    mn = min(mn, min(a0, a1));
                    mx = max(mx, max(a0, a1));
                }
                isum += acc;
            }
            i = s0 + nv * 8 + threadIdx.x;
        }
        for (; i < s1; i += blockDim.x) {
            const int a0 = x[i];
            isum += a0;
            mn = min(mn, a0);
            mx = max(mx, a0);
        }
        kmin = mn; kmax = mx;
    } else {
        const float *x = reinterpret_cast<const float *>(sig) + b * clip_stride;
        for (int64_t i = s0 + threadIdx.x; i < s1; i += blockDim.x) {
            const float v = x[i];
            dsum += double(v);
            const int k = float_key(v);
            kmin = min(kmin, k);
            kmax = max(kmax, k);
        }
    }
    // block reduce
    __shared__ long long s_i[8];
    __shared__ double s_d[8];
    __shared__ int s_mn[8], s_mx[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        isum += __shfl_xor_sync(0xffffffffu, isum, o);
        dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
        kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
        kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    }
    if (lane == 0) { s_i[warp] = isum; s_d[warp] = dsum; s_mn[warp] = kmin; s_mx[warp] = kmax; }
    __syncthreads();
    if (threadIdx.x == 0 && s1 > s0) {
        for (int w = 1; w < 8; ++w) { isum += s_i[w]; dsum += s_d[w]; kmin = min(kmin, s_mn[w]); kmax = max(kmax, s_mx[w]); }
        if (DTYPE == B200AA_DTYPE_I16)
            atomicAdd(reinterpret_cast<unsigned long long *>(&nm[b].rsv[1]), (unsigned long long)isum);
        else
            atomicAdd(reinterpret_cast<double *>(&nm[b].rsv[1]), dsum);
        atomicMin(reinterpret_cast<int *>(&nm[b].lo), kmin);
        atomicMax(reinterpret_cast<int *>(&nm[b].hi), kmax);
    }
}

template <int DTYPE>
__global__ void stats_finish_kernel(b200aa_clip_norm *nm, int64_t n, int64_t n_samples, const int64_t *len)
{
    int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (i >= n) return;
    const int64_t L = len ? len[i] : n_samples;
    b200aa_clip_norm r = nm[i];
    double mean, mn, mx;
    if (DTYPE == B200AA_DTYPE_I16) {
        const long long s = *reinterpret_cast<const long long *>(&nm[i].rsv[1]);
        mean = L > 0 ? double(s) / double(L) : 0.0;
        mn = double(*reinterpret_cast<const int *>(&r.lo));
        mx = double(*reinterpret_cast<const int *>(&r.hi));
    } else {
        const double s = *reinterpret_cast<const double *>(&nm[i].rsv[1]);
        mean = L > 0 ? s / double(L) : 0.0;
        mn = double(key_float(*reinterpret_cast<const int *>(&r.lo)));
        mx = double(key_float(*reinterpret_cast<const int *>(&r.hi)));
    }
    if (L <= 0) { mn = mx = 0.0; }
    // y = (x/2^15 - mean/2^15) / (max|x/2^15 - mean/2^15| + 1e-10)  ==  (x - mean) / (maxdev + 2^15 * 1e-10)
    const double maxdev = fmax(mx - mean, mean - mn);
    const double a = 1.0 / (maxdev + 32768.0 * 1e-10);
    double m, lo, hi;
    if (DTYPE == B200AA_DTYPE_I16) {
        m = nearbyint(mean);
        lo = floor(mean);
        hi = ceil(mean);
    } else {
        const float mf = float(mean);
        m = double(mf);
        if (double(mf) > mean) { hi = mf; lo = nextafterf(mf, -INFINITY); }
        else if (double(mf) < mean) { lo = mf; hi = nextafterf(mf, INFINITY); }
        else { lo = hi = mf; }
    }
    b200aa_clip_norm o;
    o.a = float(a);
    o.bp = float(a * (m - mean));
    o.m = float(m);
    o.lo = float(lo - m);
    o.hi = float(hi - m);
    o.rsv[0] = o.rsv[1] = o.rsv[2] = 0.f;
    nm[i] = o;
}

extern "C" int b200aa_clip_stats(const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                                 int64_t clip_stride, const int64_t *d_len, b200aa_clip_norm *d_norm, void *stream)
{
    NvtxRange nvtx_("b200aa_clip_stats");
    if (!d_sig || !d_norm || n_clips < 0 || n_samples < 0 || (dtype != 0 && dtype != 1)) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int tb = 256;
    auto accum = dtype == 0 ? stats_accum_kernel<0> : stats_accum_kernel<1>;
    auto finish = dtype == 0 ? stats_finish_kernel<0> : stats_finish_kernel<1>;
    stats_init_kernel<<<(unsigned)((n_clips + tb - 1) / tb), tb, 0, st>>>(d_norm, n_clips);
    CK_LAUNCH("stats_init_kernel");
    // enough CTAs to fill the machine, each reading >= 32 KiB
    int64_t want = (int64_t(sms) * 8 + n_clips - 1) / n_clips;
    const int64_t bytes = n_samples * (dtype == 0 ? 2 : 4);
    int64_t cap = (bytes + 32767) / 32768;
    int chunks = (int)std::max<int64_t>(1, std::min<int64_t>(want, cap));
    for (int64_t b0 = 0; b0 < n_clips; b0 += 32768) {
        const int64_t nb = std::min<int64_t>(32768, n_clips - b0);
        dim3 grid(chunks, (unsigned)nb);
        const size_t es = dtype == 0 ? 2 : 4;
        const void *sig = reinterpret_cast<const char *>(d_sig) + size_t(b0) * clip_stride * es;
        const int64_t *ln = d_len ? d_len + b0 : nullptr;
        accum<<<grid, 256, 0, st>>>(sig, n_samples, clip_stride, ln, d_norm + b0, chunks);
        CK_LAUNCH("stats_accum_kernel");
    }
    finish<<<(unsigned)((n_clips + tb - 1) / tb), tb, 0, st>>>(d_norm, n_clips, n_samples, d_len);
    CK_LAUNCH("stats_finish_kernel");
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel 1 launchers
// ------------------------------------------------------------------------------------------------
static void fill_common(StParams &p, const b200aa_plan *pl, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                        int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm *d_norm, float *d_out)
{
    const Transform &t = pl->transform;
    std::memset(&p, 0, sizeof(p));
    p.sig = d_sig; p.len = d_len; p.norm = d_norm; p.out = d_out;
    p.tw = static_cast<const float2 *>(t.tw.get()); p.tw_post = static_cast<const float2 *>(t.tw_post.get());
    p.blob = static_cast<const int *>(pl->blob.get()); p.bl = pl->bl;
    p.n_clips = n_clips; p.n_samples = n_samples; p.clip_stride = clip_stride;
    p.dtype = dtype; p.window = pl->window; p.step = pl->step; p.K = pl->K;
    p.Kp = (pl->K + 3) & ~3;
    p.Nc = t.Nc; p.packed = t.packed;
    p.nrad = (int)t.radix.size();
    for (int i = 0; i < p.nrad; ++i) p.radix[i] = t.radix[i];
}

// choose frames/group and launch the generic kernel
template <int MODE>
static int launch_generic(const b200aa_plan *pl, StParams &p, int64_t rows_max, cudaStream_t st)
{
    int G = generic_group(p.Nc, p.Kp, p.bl.words);
    const bool big = G < 1;            // one frame does not fit shared memory: window-sized arrays go to global memory
    if (big) G = 1;
    const size_t smem = generic_smem_bytes(G, p.Nc, p.Kp, p.bl.words, !big);
    if (big && p.Nc > (1 << 20)) return B200AA_ERR_UNSUPPORTED;      // 2^21-sample windows: beyond any use of the path
    p.G = G;
    // segments: long enough to amortise the 2-frame halo, short enough to balance the SMs
    int64_t seg = rows_max;
    if (MODE == kModeFeatures) {
        const int64_t slots = int64_t(pl->sm_count) * 2;
        int64_t per_clip = std::max<int64_t>(1, (slots * 12 + p.n_clips - 1) / p.n_clips);
        seg = std::max<int64_t>(G * 6 - 2, (rows_max + per_clip - 1) / per_clip);
        seg = std::min<int64_t>(seg, std::max<int64_t>(rows_max, 1));
    } else {
        seg = std::max<int64_t>(G * 4, (rows_max + 63) / 64);
    }
    p.seg_len = seg;
    p.segs_per_clip = std::max<int64_t>(1, (rows_max + seg - 1) / seg);
    p.n_items = p.segs_per_clip * p.n_clips;
    if (p.n_items == 0) return B200AA_OK;
    if (big) {
        auto kern = st_generic_kernel<MODE, true>;
        if constexpr (MODE != kModeFeatures) {
            if (p.len) kern = st_generic_kernel<MODE, true, true>;
        }
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
        const int64_t grid = std::min<int64_t>(p.n_items, int64_t(pl->sm_count) * 2);
        p.scratch_stride = generic_big_bytes(G, p.Nc, p.Kp);
        StreamScratch scratch(st);             // stream-ordered: safe across concurrent launches
        const int rc = scratch.alloc(p.scratch_stride * size_t(grid));
        if (rc != B200AA_OK) return rc;
        p.scratch = static_cast<unsigned char *>(scratch.get());
        kern<<<(unsigned)grid, kThreads, smem, st>>>(p);
        return scratch.done(launched("st_generic_kernel (large window)"));
    }
    auto kern = st_generic_kernel<MODE, false>;
    if constexpr (MODE != kModeFeatures) {
        if (p.len) kern = st_generic_kernel<MODE, false, true>;
    }
    int occ = 1;
    CK(resident_ctas(kern, kThreads, smem, 226 * 1024, occ));
    const int64_t grid = std::min<int64_t>(p.n_items, int64_t(pl->sm_count) * occ);
    kern<<<(unsigned)grid, kThreads, smem, st>>>(p);
    CK_LAUNCH("st_generic_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_st_features(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                  int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                  const b200aa_clip_norm *d_norm, int deltas, float *d_out, int64_t t_stride, void *stream)
{
    NvtxRange nvtx_("b200aa_st_features");
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || (dtype != 0 && dtype != 1) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    b200aa_plan *pl = const_cast<b200aa_plan *>(plan);
    // error order of the reference: mel bank (before the loop), no frames (:684), chroma (frame 0)
    if (pl->tables_status == B200AA_ERR_MEL_RANGE) return B200AA_ERR_MEL_RANGE;
    const int64_t T = rows::frames(n_samples, pl->window, pl->step);
    if (T == 0) return B200AA_ERR_TOO_SHORT;
    int rc = pl->tables_status;
    if (rc != B200AA_OK) return rc;
    if ((rc = plan_device_check(pl)) != B200AA_OK) return rc;
    if (t_stride < T) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    StParams p;
    fill_common(p, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    p.t_stride = t_stride; p.deltas = deltas ? 1 : 0; p.n_out = deltas ? 68 : 34;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (use_pair(pl)) {
        SlotLaunch sl(pl, st);
        if (sl.rc != B200AA_OK) return sl.rc;
        rc = sl.finish(pair_launch_features(pl->pair, p, pl->sm_count, T, reinterpret_cast<unsigned long long *>(sl.ctr),
                                            b200aa_plan::kSlotBytes, g_pair_dump, st), "pair kernel");
        if (rc != B200AA_ERR_UNSUPPORTED) return rc;
    }
    if (use_solo(pl)) {
        SlotLaunch sl(pl, st);
        if (sl.rc != B200AA_OK) return sl.rc;
        rc = sl.finish(solo_launch_mode<kModeFeatures>(pl->solo, p, pl->sm_count, T, sl.ctr, b200aa_plan::kSlotBytes, st), "solo kernel");
        if (rc != B200AA_ERR_UNSUPPORTED) return rc;
    }
    if (use_fast(pl)) {
        SlotLaunch sl(pl, st);
        if (sl.rc != B200AA_OK) return sl.rc;
        rc = sl.finish(fast_launch_mode<kModeFeatures>(pl->fast_kind, pl->fast, p, pl->sm_count, T, sl.ctr, st), "fast kernel");
        if (rc != B200AA_ERR_UNSUPPORTED) return rc;
    }
    return launch_generic<kModeFeatures>(pl, p, T, st);
}

// The plan's row kernel over every clip: the per-frame solo kernel, else the register-tiled CTA kernel (the pair kernel
// has no row mode), else the generic kernel.  p.len set: a ragged batch, every clip with its own rows (ragged_rows).
template <int MODE>
static int launch_rows(b200aa_plan *pl, StParams &p, cudaStream_t st)
{
    if (use_solo(pl)) {
        SlotLaunch sl(pl, st);
        if (sl.rc != B200AA_OK) return sl.rc;
        const int rc = sl.finish(solo_launch_mode<MODE>(pl->solo, p, pl->sm_count, p.rows_launch, sl.ctr, b200aa_plan::kSlotBytes, st), "solo kernel");
        if (rc != B200AA_ERR_UNSUPPORTED) return rc;
    }
    if (pl->fast_kind && !pl->force_generic && pl->prefer != 0 && pl->prefer != 3) {
        SlotLaunch sl(pl, st);
        if (sl.rc != B200AA_OK) return sl.rc;
        const int rc = sl.finish(fast_launch_mode<MODE>(pl->fast_kind, pl->fast, p, pl->sm_count, p.rows_launch, sl.ctr, st), "fast kernel");
        if (rc != B200AA_ERR_UNSUPPORTED) return rc;
    }
    return launch_generic<MODE>(pl, p, p.rows_launch, st);
}

// Every clipped chromagram frame of the batch in one launch of clipped_chroma_kernel: per_clip candidate rows per clip
static int launch_clipped(const b200aa_plan *pl, StParams p, int64_t per_clip, cudaStream_t st)
{
    constexpr size_t kSmemCap = 226 * 1024;        // the per-CTA opt-in maximum, less the static reserve
    p.n_items = p.n_clips * per_clip;
    const size_t bytes = clipped_bytes(p.window, p.K);
    if (bytes <= kSmemCap) {
        CK(cudaFuncSetAttribute(clipped_chroma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap));
        const int64_t grid = std::min<int64_t>(p.n_items, int64_t(1) << 30);
        clipped_chroma_kernel<false><<<(unsigned)grid, kThreads, bytes, st>>>(p, per_clip);
        CK_LAUNCH("clipped_chroma_kernel");
        return B200AA_OK;
    }
    // large windows: the arrays of every resident CTA in stream-ordered scratch, CTAs loop over the items
    const int64_t grid = std::min<int64_t>(p.n_items, int64_t(pl->sm_count) * 2);
    p.scratch_stride = align256(bytes);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(p.scratch_stride * size_t(grid));
    if (rc != B200AA_OK) return rc;
    p.scratch = static_cast<unsigned char *>(scratch.get());
    clipped_chroma_kernel<true><<<(unsigned)grid, kThreads, 0, st>>>(p, per_clip);
    return scratch.done(launched("clipped_chroma_kernel (large window)"));
}

// b200aa_spectrogram and b200aa_spectrogram_ragged (d_len set): the launch is sized by n_samples
static int spectrogram_launch(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                              int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm *d_norm, float *d_out,
                              void *stream)
{
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || (dtype != 0 && dtype != 1) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    b200aa_plan *pl = const_cast<b200aa_plan *>(plan);
    const rows::Rows r = rows::spectrogram(n_samples, pl->window, pl->step);
    if (r.refused) return B200AA_ERR_TOO_SHORT;     // np.zeros with a non-positive row count / empty result
    if (n_clips == 0) return B200AA_OK;
    const int rc = plan_device_check(pl);
    if (rc != B200AA_OK) return rc;
    StParams p;
    fill_common(p, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    p.rows_launch = r.R; p.rows_valid = r.n_full;
    return launch_rows<kModeSpectrogram>(pl, p, static_cast<cudaStream_t>(stream));
}

extern "C" int b200aa_spectrogram(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                  int64_t n_samples, int64_t clip_stride, const b200aa_clip_norm *d_norm,
                                  float *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_spectrogram");
    return spectrogram_launch(plan, d_sig, dtype, n_clips, n_samples, clip_stride, nullptr, d_norm, d_out, stream);
}

extern "C" int b200aa_spectrogram_ragged(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                         int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                         const b200aa_clip_norm *d_norm, float *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_spectrogram_ragged");
    if (!d_len) return B200AA_ERR_INVALID;
    return spectrogram_launch(plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream);
}

// b200aa_chromagram and b200aa_chromagram_ragged (d_len set): the row kernel writes the rows of full frames and zeros
// after them, then one launch transforms every clipped frame of the batch into its row
static int chromagram_launch(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips, int64_t n_samples,
                             int64_t clip_stride, const int64_t *d_len, const b200aa_clip_norm *d_norm, float *d_out,
                             void *stream)
{
    if (!plan || !d_sig || !d_norm || !d_out || n_clips < 0 || (dtype != 0 && dtype != 1) || clip_stride < n_samples)
        return B200AA_ERR_INVALID;
    b200aa_plan *pl = const_cast<b200aa_plan *>(plan);
    const int w = pl->window, s = pl->step;
    const rows::Rows r = rows::chromagram(n_samples, w, s);
    // a ragged batch is refused only when its width gives no rows: each clip's own refusal leaves its rows unwritten
    if (r.R <= 0 || (!d_len && n_samples - s - w < 0)) return B200AA_ERR_TOO_SHORT;
    int rc = pl->tables_status;
    if (rc == B200AA_ERR_CHROMA) return rc;
    if (n_clips == 0) return B200AA_OK;
    if (!d_len && r.refused) return B200AA_ERR_INVALID;     // a clipped frame shorter than K: the reference's scatter raises
    if ((rc = plan_device_check(pl)) != B200AA_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StParams p;
    fill_common(p, pl, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out);
    p.rows_launch = r.R; p.rows_valid = r.n_full;
    rc = launch_rows<kModeChromagram>(pl, p, st);
    if (rc != B200AA_OK) return rc;
    const int64_t per_clip = d_len ? rows::max_clipped(w, s) : r.n_it - r.n_full;
    return per_clip > 0 ? launch_clipped(pl, p, per_clip, st) : B200AA_OK;
}

extern "C" int b200aa_chromagram(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                 int64_t n_samples, int64_t clip_stride, const b200aa_clip_norm *d_norm,
                                 float *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_chromagram");
    return chromagram_launch(plan, d_sig, dtype, n_clips, n_samples, clip_stride, nullptr, d_norm, d_out, stream);
}

extern "C" int b200aa_chromagram_ragged(const b200aa_plan *plan, const void *d_sig, int dtype, int64_t n_clips,
                                        int64_t n_samples, int64_t clip_stride, const int64_t *d_len,
                                        const b200aa_clip_norm *d_norm, float *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_chromagram_ragged");
    if (!d_len) return B200AA_ERR_INVALID;
    return chromagram_launch(plan, d_sig, dtype, n_clips, n_samples, clip_stride, d_len, d_norm, d_out, stream);
}

// ------------------------------------------------------------------------------------------------
// host-buffer entry points
// ------------------------------------------------------------------------------------------------
// slot `slot` of the plan's workspace, grown to at least n bytes, with room to spare (caller holds host_mu);
// nullptr = cudaMalloc failed
static void *workspace(b200aa_plan *pl, int slot, size_t n)
{
    return pl->ws[slot].reserve(n, n + n / 4 + 4096) == cudaSuccess ? pl->ws[slot].get() : nullptr;
}

// One host-buffer call: takes the plan's workspace lock, uploads the clips (slot 0) and produces their normalisation
// records (slot 1); the entry points add their own kernels and downloads on the same (legacy default) stream.
struct HostCall {
    b200aa_plan *pl;
    std::unique_lock<std::mutex> hold;
    cudaStream_t st = nullptr;
    void *sig = nullptr;
    b200aa_clip_norm *norm = nullptr;
    explicit HostCall(const b200aa_plan *plan) : pl(const_cast<b200aa_plan *>(plan)), hold(pl->host_mu) {}
    int upload(const void *h_sig, int dtype, int64_t n_clips, int64_t n_samples)
    {
        int rc = plan_device_check(pl);
        if (rc != B200AA_OK) return rc;
        const size_t in_b = size_t(n_clips) * n_samples * (dtype == B200AA_DTYPE_I16 ? 2 : 4);
        sig = workspace(pl, 0, in_b);
        norm = static_cast<b200aa_clip_norm *>(workspace(pl, 1, sizeof(b200aa_clip_norm) * n_clips));
        if (!sig || !norm) return cuda_fail(cudaGetLastError(), "cudaMalloc");
        CK(cudaMemcpyAsync(sig, h_sig, in_b, cudaMemcpyHostToDevice, st));
        return b200aa_clip_stats(sig, dtype, n_clips, n_samples, n_samples, nullptr, norm, st);
    }
    float *result(int slot, size_t bytes) { return static_cast<float *>(workspace(pl, slot, bytes)); }
    int download(void *h_dst, const void *d_src, size_t bytes)
    {
        CK(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, st));
        return B200AA_OK;
    }
    int finish()
    {
        CK(cudaStreamSynchronize(st));
        return B200AA_OK;
    }
};

// Chunked, multi-stream form of b200aa_st_features_host for batches of many clips: every chunk's upload, kernels and
// download are queued on one of three streams, so the PCIe transfers of neighbouring chunks overlap the kernels (pinned
// host memory -- b200aa_host_alloc -- makes the copies truly asynchronous; pageable memory still works, the copies
// then serialise in the driver).
static int st_features_host_pipelined(b200aa_plan *pl, const void *h_sig, int dtype, int64_t n_clips, int64_t n_samples,
                                      int deltas, float *h_out, int64_t T, int64_t chunk)
{
    std::lock_guard<std::mutex> hold(pl->host_mu);
    int rc = plan_device_check(pl);
    if (rc != B200AA_OK) return rc;
    const size_t es = dtype == B200AA_DTYPE_I16 ? 2 : 4;
    const size_t F = deltas ? 68 : 34;
    const size_t need[3] = {size_t(chunk) * n_samples * es, sizeof(b200aa_clip_norm) * size_t(chunk), size_t(chunk) * F * T * 4};
    for (int k = 0; k < b200aa_plan::kPipe; ++k) {
        if (!pl->pipe_stream[k]) CK(cudaStreamCreateWithFlags(&pl->pipe_stream[k], cudaStreamNonBlocking));
        for (int j = 0; j < 3; ++j) CK(pl->pipe_ws[k][j].reserve(need[j], need[j]));
    }
    int64_t c = 0;
    for (int64_t a = 0; a < n_clips && rc == B200AA_OK; a += chunk, ++c) {
        const int k = int(c % b200aa_plan::kPipe);
        const int64_t n = std::min<int64_t>(chunk, n_clips - a);
        cudaStream_t st = pl->pipe_stream[k];      // stream order also protects the buffers: chunk c + kPipe waits for chunk c
        void *sig = pl->pipe_ws[k][0].get();
        b200aa_clip_norm *norm = static_cast<b200aa_clip_norm *>(pl->pipe_ws[k][1].get());
        float *out = static_cast<float *>(pl->pipe_ws[k][2].get());
        cudaError_t e = cudaMemcpyAsync(sig, static_cast<const char *>(h_sig) + size_t(a) * n_samples * es, size_t(n) * n_samples * es,
                                        cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMemcpyAsync (clips)"); break; }
        rc = b200aa_clip_stats(sig, dtype, n, n_samples, n_samples, nullptr, norm, st);
        if (rc != B200AA_OK) break;
        rc = b200aa_st_features(pl, sig, dtype, n, n_samples, n_samples, nullptr, norm, deltas, out, T, st);
        if (rc != B200AA_OK) break;
        e = cudaMemcpyAsync(h_out + size_t(a) * F * T, out, size_t(n) * F * T * 4, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync (features)");
    }
    for (int k = 0; k < b200aa_plan::kPipe; ++k) {         // drain every stream, also after an error
        const cudaError_t e = cudaStreamSynchronize(pl->pipe_stream[k]);
        if (e != cudaSuccess && rc == B200AA_OK) rc = cuda_fail(e, "cudaStreamSynchronize");
    }
    return rc;
}

extern "C" int b200aa_st_features_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_clips,
                                       int64_t n_samples, int deltas, float *h_out)
{
    NvtxRange nvtx_("b200aa_st_features_host");
    if (!plan || !h_sig || !h_out || n_clips < 1 || (dtype != 0 && dtype != 1)) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(nullptr, "b200aa_st_features_host", kWhyHostBuffer);
    if (plan->tables_status == B200AA_ERR_MEL_RANGE) return B200AA_ERR_MEL_RANGE;
    const int64_t T = rows::frames(n_samples, plan->window, plan->step);
    if (T == 0) return B200AA_ERR_TOO_SHORT;
    if (plan->tables_status != B200AA_OK) return plan->tables_status;
    {   // chunks of ~32 MB of samples; batches of fewer than two chunks take the single-stream path below
        const int64_t chunk = std::max<int64_t>(1, (int64_t(32) << 20) / (n_samples * (dtype == B200AA_DTYPE_I16 ? 2 : 4)));
        if (n_clips >= 2 * chunk)
            return st_features_host_pipelined(const_cast<b200aa_plan *>(plan), h_sig, dtype, n_clips, n_samples, deltas, h_out, T, chunk);
    }
    const size_t out_b = size_t(n_clips) * (deltas ? 68 : 34) * T * 4;
    HostCall hc(plan);
    int rc = hc.upload(h_sig, dtype, n_clips, n_samples);
    if (rc) return rc;
    float *out = hc.result(2, out_b);
    if (!out) return cuda_fail(cudaGetLastError(), "cudaMalloc");
    rc = b200aa_st_features(plan, hc.sig, dtype, n_clips, n_samples, n_samples, nullptr, hc.norm, deltas, out, T, hc.st);
    if (rc) return rc;
    if ((rc = hc.download(h_out, out, out_b))) return rc;
    return hc.finish();
}

extern "C" int b200aa_spectrogram_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_samples, float *h_out)
{
    if (!plan || !h_sig || !h_out || (dtype != 0 && dtype != 1)) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(nullptr, "b200aa_spectrogram_host", kWhyHostBuffer);
    const int64_t R = b200aa_spectrogram_rows(n_samples, plan->window, plan->step);
    if (R <= 0) return B200AA_ERR_TOO_SHORT;
    const size_t out_b = size_t(R) * plan->K * 4;
    HostCall hc(plan);
    int rc = hc.upload(h_sig, dtype, 1, n_samples);
    if (rc) return rc;
    float *out = hc.result(2, out_b);
    if (!out) return cuda_fail(cudaGetLastError(), "cudaMalloc");
    rc = b200aa_spectrogram(plan, hc.sig, dtype, 1, n_samples, n_samples, hc.norm, out, hc.st);
    if (rc) return rc;
    if ((rc = hc.download(h_out, out, out_b))) return rc;
    return hc.finish();
}

extern "C" int b200aa_chromagram_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_samples, float *h_out)
{
    if (!plan || !h_sig || !h_out || (dtype != 0 && dtype != 1)) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(nullptr, "b200aa_chromagram_host", kWhyHostBuffer);
    const int64_t R = b200aa_chromagram_rows(n_samples, plan->window, plan->step);
    if (R <= 0 || n_samples - plan->step - plan->window < 0) return B200AA_ERR_TOO_SHORT;
    if (plan->tables_status == B200AA_ERR_CHROMA) return B200AA_ERR_CHROMA;
    const size_t out_b = size_t(R) * 12 * 4;
    HostCall hc(plan);
    int rc = hc.upload(h_sig, dtype, 1, n_samples);
    if (rc) return rc;
    float *out = hc.result(2, out_b);
    if (!out) return cuda_fail(cudaGetLastError(), "cudaMalloc");
    rc = b200aa_chromagram(plan, hc.sig, dtype, 1, n_samples, n_samples, hc.norm, out, hc.st);
    if (rc) return rc;
    if ((rc = hc.download(h_out, out, out_b))) return rc;
    return hc.finish();
}

extern "C" int b200aa_mid_features_host(const b200aa_plan *plan, const void *h_sig, int dtype, int64_t n_samples,
                                        int ratio, int step_ratio, float *h_mid, float *h_st)
{
    NvtxRange nvtx_("b200aa_mid_features_host");
    if (!plan || !h_sig || !h_mid || step_ratio < 1 || (dtype != 0 && dtype != 1)) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(nullptr, "b200aa_mid_features_host", kWhyHostBuffer);
    if (plan->tables_status == B200AA_ERR_MEL_RANGE) return B200AA_ERR_MEL_RANGE;
    const int64_t T = rows::frames(n_samples, plan->window, plan->step);
    if (T == 0) return B200AA_ERR_TOO_SHORT;
    if (plan->tables_status != B200AA_OK) return plan->tables_status;
    const int64_t M = b200aa_mid_windows(T, step_ratio);
    const size_t st_b = size_t(68) * T * 4, mid_b = size_t(136) * M * 4;
    HostCall hc(plan);
    int rc = hc.upload(h_sig, dtype, 1, n_samples);
    if (rc) return rc;
    float *stf = hc.result(2, st_b), *mid = hc.result(3, mid_b);
    if (!stf || !mid) return cuda_fail(cudaGetLastError(), "cudaMalloc");
    rc = b200aa_st_features(plan, hc.sig, dtype, 1, n_samples, n_samples, nullptr, hc.norm, 1, stf, T, hc.st);
    if (rc) return rc;
    rc = b200aa_mid_pool(stf, 1, 68, T, T, ratio, step_ratio, mid, hc.st);
    if (rc) return rc;
    if ((rc = hc.download(h_mid, mid, mid_b))) return rc;
    if (h_st && (rc = hc.download(h_st, stf, st_b))) return rc;
    return hc.finish();
}

// ------------------------------------------------------------------------------------------------
// pinned host buffers (full-speed, truly asynchronous H2D / D2H copies for the host entry points)
// ------------------------------------------------------------------------------------------------
extern "C" int b200aa_host_alloc(void **h_out, size_t bytes)
{
    if (!h_out) return B200AA_ERR_INVALID;
    *h_out = nullptr;
    if (bytes == 0) return B200AA_OK;
    // pages are placed by the calling thread's NUMA policy: bind the thread to the GPU's node first
    CK(cudaHostAlloc(h_out, bytes, cudaHostAllocPortable));
    return B200AA_OK;
}
extern "C" int b200aa_host_free(void *h_ptr)
{
    if (h_ptr) CK(cudaFreeHost(h_ptr));
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// peer-mapped gather target (SURVEY 8e): rank 0 owns one [n_clips_total, F, T] buffer, every other rank of the
// box maps it (CUDA IPC over NVLink) and its feature kernel stores straight into its slice -- the gather is
// fused into the tile store, no collective kernel, no SMs on the root.
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == B200AA_IPC_HANDLE_BYTES, "handle size");
extern "C" int b200aa_peer_buffer_create(size_t bytes, void **d_out, unsigned char *handle_out)
{
    if (!d_out || !handle_out || bytes == 0) return B200AA_ERR_INVALID;
    CK(cudaMalloc(d_out, bytes));
    cudaIpcMemHandle_t h;
    const cudaError_t e = cudaIpcGetMemHandle(&h, *d_out);
    if (e != cudaSuccess) { cudaFree(*d_out); *d_out = nullptr; return cuda_fail(e, "cudaIpcGetMemHandle"); }
    std::memcpy(handle_out, &h, sizeof(h));
    return B200AA_OK;
}
extern "C" int b200aa_peer_buffer_open(const unsigned char *handle, void **d_out)
{
    if (!handle || !d_out) return B200AA_ERR_INVALID;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, sizeof(h));
    CK(cudaIpcOpenMemHandle(d_out, h, cudaIpcMemLazyEnablePeerAccess));
    return B200AA_OK;
}
extern "C" int b200aa_peer_copy(void *d_dst, const void *d_src, size_t bytes, void *stream)
{
    if (!d_dst || !d_src) return B200AA_ERR_INVALID;
    REFUSE_CAPTURE(stream, "b200aa_peer_copy", "peer copies are not captured; call it eagerly");
    if (bytes == 0) return B200AA_OK;
    // unified addressing: the copy engines move the block over NVLink, no SM on either side is involved
    CK(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    return B200AA_OK;
}
extern "C" int b200aa_peer_buffer_close(void *d_ptr, int owner)
{
    if (!d_ptr) return B200AA_OK;
    if (owner) CK(cudaFree(d_ptr));
    else CK(cudaIpcCloseMemHandle(d_ptr));
    return B200AA_OK;
}
