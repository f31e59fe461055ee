// libb200aa.so -- C ABI (include/b200aa.h) over the sm_90a kernels.
// Build: see pyaudioanalysis_b200/build.py (nvcc -gencode arch=compute_90a,code=sm_90a).
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>      // header-only NVTX 3: ranges around the entry points (visible in nsys / ncu timelines)

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200aa.h"
#include "beat.cuh"
#include "common.cuh"
#include "generic_kernel.cuh"
#include "hmm.cuh"
#include "knn.cuh"
#include "knn_cv.cuh"
#include "fast_kernel.cuh"
#include "pair_kernel.cuh"
#include "pcm.cuh"
#include "slots.h"
#include "solo_kernel.cuh"
#include "tables.inl"
#include "trees.cuh"

using namespace b200aa;

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_cuda_err;
static std::atomic<int64_t> g_launches{0};

static int cuda_fail(cudaError_t e, const char *what)
{
    g_cuda_err = std::string(what) + ": " + cudaGetErrorString(e);
    return B200AA_ERR_CUDA;
}
#define CK(call)                                                     \
    do {                                                             \
        cudaError_t e_ = (call);                                     \
        if (e_ != cudaSuccess) return cuda_fail(e_, #call);          \
    } while (0)
// every kernel launch ends here: count it (b200aa_launch_count), then report its launch error
static int launched(const char *name)
{
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? B200AA_OK : cuda_fail(e, name);
}
#define CK_LAUNCH(name)                                              \
    do {                                                             \
        const int rc_ = launched(name);                              \
        if (rc_ != B200AA_OK) return rc_;                            \
    } while (0)

// Stream-ordered device scratch of one entry point, bound to its scope: alloc() takes it with cudaMallocAsync, done(rc)
// frees it after everything queued on the stream and returns rc, else the free's error.  A scope left early (its error
// already reported) frees it in the destructor.
class StreamScratch {
  public:
    explicit StreamScratch(cudaStream_t st) : st_(st) {}
    StreamScratch(const StreamScratch &) = delete;
    StreamScratch &operator=(const StreamScratch &) = delete;
    ~StreamScratch() { release(); }
    int alloc(size_t bytes)
    {
        if (bytes) CK(cudaMallocAsync(&p_, bytes, st_));
        return B200AA_OK;
    }
    void *get() const { return p_; }
    int done(int rc)
    {
        const cudaError_t e = release();
        return (e != cudaSuccess && rc == B200AA_OK) ? cuda_fail(e, "cudaFreeAsync") : rc;
    }

  private:
    cudaError_t release()
    {
        const cudaError_t e = p_ ? cudaFreeAsync(p_, st_) : cudaSuccess;
        p_ = nullptr;
        return e;
    }
    cudaStream_t st_;
    void *p_ = nullptr;
};

struct NvtxRange {
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

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
// mid-term windows of a clip of n_frames frames: b200aa_mid_windows on the host, per clip of a ragged batch on the device
__host__ __device__ inline int64_t windows_of(int64_t n_frames, int stepr)
{
    return (stepr < 1 || n_frames <= 0) ? 0 : (n_frames + stepr - 1) / stepr;
}

extern "C" int64_t b200aa_mid_windows(int64_t n_frames, int stepr) { return windows_of(n_frames, stepr); }

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
    ~b200aa_plan()
    {
        for (cudaStream_t s : pipe_stream) if (s) cudaStreamDestroy(s);
    }
};

extern "C" int b200aa_plan_create(b200aa_plan **out, int fs, int window, int step)
{
    if (!out || fs <= 0 || window < 2 || step < 1) return B200AA_ERR_INVALID;
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
struct SlotLaunch {
    b200aa_plan *pl;
    cudaStream_t st;
    unsigned slot = 0;
    unsigned int *ctr = nullptr;
    int rc;
    SlotLaunch(b200aa_plan *plan, cudaStream_t stream) : pl(plan), st(stream)
    {
        rc = pl->slots.acquire(st, slot);
        if (rc == B200AA_OK)
            ctr = reinterpret_cast<unsigned int *>(static_cast<unsigned char *>(pl->counters.get()) + size_t(slot) * b200aa_plan::kSlotBytes);
    }
    int finish(int launch_rc, const char *name)
    {
        const int r = launch_rc == B200AA_OK ? launched(name)
                                             : (launch_rc == B200AA_ERR_CUDA ? cuda_fail(cudaGetLastError(), name) : launch_rc);
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
        if (dtype == 0) stats_accum_kernel<0><<<grid, 256, 0, st>>>(sig, n_samples, clip_stride, ln, d_norm + b0, chunks);
        else stats_accum_kernel<1><<<grid, 256, 0, st>>>(sig, n_samples, clip_stride, ln, d_norm + b0, chunks);
        CK_LAUNCH("stats_accum_kernel");
    }
    if (dtype == 0) stats_finish_kernel<0><<<(unsigned)((n_clips + tb - 1) / tb), tb, 0, st>>>(d_norm, n_clips, n_samples, d_len);
    else stats_finish_kernel<1><<<(unsigned)((n_clips + tb - 1) / tb), tb, 0, st>>>(d_norm, n_clips, n_samples, d_len);
    CK_LAUNCH("stats_finish_kernel");
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel 2: mid-term pooling (MidTermFeatures.py:110-126): one warp per (clip, feature row, window)
// ------------------------------------------------------------------------------------------------
// frames (nullable, int64 [n_clips]): clip b has T_b = clamp(frames[b], 0, t_stride) frames and M_b = windows_of(T_b)
// windows; warps of windows j >= M_b write nothing.  Without frames every clip has T frames.  A warp's sums depend only
// on (c0, c1, lane), so a clip pooled in a ragged batch gives bit for bit what it gives alone with T = T_b.  RAGGED is
// a template flag only so that the batch without counts keeps the code (and time) it had before counts existed.
template <bool RAGGED>
__global__ void __launch_bounds__(256) mid_pool_kernel(const float *st, int64_t n_clips, int F, int64_t T,
                                                        int64_t t_stride, const int64_t *frames, int ratio, int stepr,
                                                        int64_t M, float *mid)
{
    const int lane = threadIdx.x & 31;
    const int64_t wid = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t total = n_clips * F * M;
    if (wid >= total) return;
    const int64_t j = wid % M, bf = wid / M;
    const int64_t b = bf / F;
    const int f = int(bf - b * F);
    if (RAGGED) {
        T = min(max(frames[b], int64_t(0)), t_stride);
        if (j >= windows_of(T, stepr)) return;              // the whole warp: j is uniform across it
    }
    // window j is the Python slice row[c0 : min(c0 + ratio, T)] (:116-120): a negative end counts from the end of
    // the row (ratio < 0), an end before c0 gives an empty window; n = 0 makes mean and std 0 / 0 -> 0 below
    const int64_t c0 = j * stepr;
    int64_t c1 = min(T, c0 + ratio);
    if (c1 < 0) c1 = max(c1 + T, int64_t(0));
    const float *row = st + (size_t(b) * F + f) * t_stride;
    const int n = int(max(c1 - c0, int64_t(0)));
    double s = 0.0;
    for (int64_t c = c0 + lane; c < c1; c += 32) s += double(row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double mean = s / double(n);
    double v = 0.0;
    for (int64_t c = c0 + lane; c < c1; c += 32) { const double d = double(row[c]) - mean; v += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) {
        float mu = float(mean), sd = float(sqrt(v / double(n)));
        // np.nan_to_num (:126)
        if (isnan(mu)) mu = 0.f;
        if (isnan(sd)) sd = 0.f;
        if (isinf(mu)) mu = mu > 0 ? 3.4028234664e38f : -3.4028234664e38f;
        if (isinf(sd)) sd = 3.4028234664e38f;
        mid[(size_t(b) * 2 * F + f) * M + j] = mu;
        mid[(size_t(b) * 2 * F + F + f) * M + j] = sd;
    }
}

// d_mid's row stride is M = windows_of(T): with frames, T = t_stride, the longest any clip can have
static int mid_pool_launch(const float *d_st, int64_t n_clips, int n_feats, int64_t T, int64_t t_stride, const int64_t *d_frames,
                           int ratio, int step_ratio, float *d_mid, void *stream)
{
    const int64_t M = windows_of(T, step_ratio);
    const int64_t warps = n_clips * n_feats * M;
    if (warps == 0) return B200AA_OK;
    const int64_t blocks = (warps * 32 + 255) / 256;
    auto kernel = d_frames ? mid_pool_kernel<true> : mid_pool_kernel<false>;
    kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_st, n_clips, n_feats, T, t_stride, d_frames,
                                                                             ratio, step_ratio, M, d_mid);
    CK_LAUNCH("mid_pool_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_mid_pool(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                               int ratio, int step_ratio, float *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool");
    if (!d_st || !d_mid || n_clips < 0 || n_feats < 1 || n_frames < 1 || step_ratio < 1 || t_stride < n_frames)
        return B200AA_ERR_INVALID;
    return mid_pool_launch(d_st, n_clips, n_feats, n_frames, t_stride, nullptr, ratio, step_ratio, d_mid, stream);
}

extern "C" int b200aa_mid_pool_ragged(const float *d_st, int64_t n_clips, int n_feats, int64_t t_stride,
                                      const int64_t *d_frames, int ratio, int step_ratio, float *d_mid, void *stream)
{
    NvtxRange nvtx_("b200aa_mid_pool_ragged");
    if (!d_st || !d_frames || !d_mid || n_clips < 0 || n_feats < 1 || step_ratio < 1 || t_stride < 0)
        return B200AA_ERR_INVALID;
    return mid_pool_launch(d_st, n_clips, n_feats, t_stride, t_stride, d_frames, ratio, step_ratio, d_mid, stream);
}

// long-term average of the mid-term matrix: one warp per (clip, row), fp64 accumulation.  windows (nullable, int64
// [n_clips]): clip b averages its first M_b = clamp(windows[b], 0, M) columns (0 / 0 = NaN for none, as np.mean of an
// empty axis); the sum's order depends only on (M_b, lane), as in mid_pool_kernel.
__global__ void __launch_bounds__(256) long_term_mean_kernel(const float *mid, int64_t all_rows, int n_rows, int64_t M,
                                                             const int64_t *windows, float *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t wid = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (wid >= all_rows) return;
    const int64_t Mb = windows ? min(max(windows[wid / n_rows], int64_t(0)), M) : M;
    const float *row = mid + size_t(wid) * M;
    double s = 0.0;
    for (int64_t c = lane; c < Mb; c += 32) s += double(row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[wid] = float(s / double(Mb));
}

static int long_term_mean_launch(const float *d_mid, int64_t n_clips, int n_rows, int64_t m_stride, const int64_t *d_windows,
                                 float *d_out, void *stream)
{
    const int64_t rows = n_clips * n_rows;
    if (rows == 0) return B200AA_OK;
    const int64_t blocks = (rows * 32 + 255) / 256;
    long_term_mean_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_mid, rows, n_rows, m_stride,
                                                                                             d_windows, d_out);
    CK_LAUNCH("long_term_mean_kernel");
    return B200AA_OK;
}

extern "C" int b200aa_long_term_mean(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, float *d_out, void *stream)
{
    if (!d_mid || !d_out || n_clips < 0 || n_rows < 1 || n_windows < 1) return B200AA_ERR_INVALID;
    return long_term_mean_launch(d_mid, n_clips, n_rows, n_windows, nullptr, d_out, stream);
}

extern "C" int b200aa_long_term_mean_ragged(const float *d_mid, int64_t n_clips, int n_rows, int64_t m_stride,
                                            const int64_t *d_windows, float *d_out, void *stream)
{
    if (!d_mid || !d_windows || !d_out || n_clips < 0 || n_rows < 1 || m_stride < 0) return B200AA_ERR_INVALID;
    return long_term_mean_launch(d_mid, n_clips, n_rows, m_stride, d_windows, d_out, stream);
}

// per-clip counts of a ragged batch from its device lengths: one thread per clip
__global__ void __launch_bounds__(256) frame_counts_kernel(const int64_t *len, int64_t n_clips, int w, int s, int stepr,
                                                           int64_t *frames, int64_t *windows)
{
    const int64_t b = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (b >= n_clips) return;
    const int64_t T = rows::frames(len[b], w, s);
    frames[b] = T;
    if (windows) windows[b] = windows_of(T, stepr);
}

extern "C" int b200aa_frame_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int step_ratio,
                                   int64_t *d_frames, int64_t *d_windows, void *stream)
{
    if (!d_len || !d_frames || n_clips < 0 || window < 1 || step < 1 || (d_windows && step_ratio < 1))
        return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    const int64_t blocks = (n_clips + 255) / 256;
    frame_counts_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_len, n_clips, window, step,
                                                                                           step_ratio, d_frames, d_windows);
    CK_LAUNCH("frame_counts_kernel");
    return B200AA_OK;
}

// per-clip output rows of a ragged spectrogram (which = 0) / chromagram (1): R_b, or 0 where the single-clip entry point
// refuses the clip
__global__ void __launch_bounds__(256) row_counts_kernel(const int64_t *len, int64_t n_clips, int w, int s, int which, int64_t *out)
{
    const int64_t b = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (b >= n_clips) return;
    const rows::Rows r = which ? rows::chromagram(len[b], w, s) : rows::spectrogram(len[b], w, s);
    out[b] = r.refused ? 0 : r.R;
}

extern "C" int b200aa_row_counts(const int64_t *d_len, int64_t n_clips, int window, int step, int which, int64_t *d_rows,
                                 void *stream)
{
    if (!d_len || !d_rows || n_clips < 0 || window < 1 || step < 1 || (which != 0 && which != 1)) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    const int64_t blocks = (n_clips + 255) / 256;
    row_counts_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_len, n_clips, window, step, which, d_rows);
    CK_LAUNCH("row_counts_kernel");
    return B200AA_OK;
}

// (mid[b, f, j] - mean[f]) / std[f] -> out[b, j, f]: 32 x 32 tiles through shared memory, both sides coalesced
// (audioSegmentation.py:581-584: one column of the mid-term matrix at a time)
__global__ void normalize_windows_kernel(const float *__restrict__ mid, int n_rows, int64_t n_windows, const float *__restrict__ mean,
                                         const float *__restrict__ sd, float *__restrict__ out)
{
    __shared__ float tile[32][33];
    const int64_t b = blockIdx.z;
    const int64_t j0 = int64_t(blockIdx.x) * 32;
    const int f0 = blockIdx.y * 32;
    const float *src = mid + b * n_rows * n_windows;
    float *dst = out + b * n_rows * n_windows;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int f = f0 + r;
        const int64_t j = j0 + threadIdx.x;
        if (f < n_rows && j < n_windows) tile[r][threadIdx.x] = (src[int64_t(f) * n_windows + j] - mean[f]) / sd[f];
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t j = j0 + r;
        const int f = f0 + threadIdx.x;
        if (f < n_rows && j < n_windows) dst[j * n_rows + f] = tile[threadIdx.x][r];
    }
}

extern "C" int b200aa_normalize_windows(const float *d_mid, int64_t n_clips, int n_rows, int64_t n_windows, const float *d_mean,
                                        const float *d_std, float *d_out, void *stream)
{
    if (!d_mid || !d_out || !d_mean || !d_std || n_clips < 0 || n_rows < 1 || n_windows < 0) return B200AA_ERR_INVALID;
    if (n_clips == 0 || n_windows == 0) return B200AA_OK;
    if (n_clips > 65535 || (n_rows + 31) / 32 > 65535) return B200AA_ERR_UNSUPPORTED;
    const dim3 grid((unsigned)((n_windows + 31) / 32), (unsigned)((n_rows + 31) / 32), (unsigned)n_clips), block(32, 8);
    normalize_windows_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(d_mid, n_rows, n_windows, d_mean, d_std, d_out);
    CK_LAUNCH("normalize_windows_kernel");
    return B200AA_OK;
}

// ------------------------------------------------------------------------------------------------
// PCM WAV decode (csrc/pcm.cuh): raw data chunks of a byte arena -> the [B, N] int16 / float32 ragged batch
// ------------------------------------------------------------------------------------------------
extern "C" int b200aa_decode_pcm(const void *d_arena, int64_t arena_bytes, const b200aa_pcm_clip *h_clips, int64_t n_clips,
                                 int out_dtype, void *d_out, int64_t n_out, int64_t out_stride, void *stream)
{
    NvtxRange nvtx_("b200aa_decode_pcm");
    if (!d_arena || !h_clips || !d_out || arena_bytes < 0 || n_clips < 0 || n_out < 0 || out_stride < n_out ||
        (out_dtype != B200AA_DTYPE_I16 && out_dtype != B200AA_DTYPE_F32))
        return B200AA_ERR_INVALID;
    for (int64_t b = 0; b < n_clips; ++b) {
        const b200aa_pcm_clip &c = h_clips[b];
        const int64_t bytes = pcm::sample_bytes(c.format);
        if (bytes == 0 || (c.channels != 1 && c.channels != 2) || c.offset < 0 || c.offset % 16 || c.n_frames < 0 ||
            c.n_frames > n_out)
            return B200AA_ERR_INVALID;
        if (out_dtype == B200AA_DTYPE_I16 && (c.channels != 1 || (c.format != B200AA_PCM_U8 && c.format != B200AA_PCM_S16)))
            return B200AA_ERR_INVALID;
        const int64_t block = c.channels * bytes;
        if (c.offset > arena_bytes || c.n_frames > (arena_bytes - c.offset) / block ||
            (c.n_frames * block + 15) / 16 * 16 > arena_bytes - c.offset)      // the kernel reads whole 16-byte words
            return B200AA_ERR_INVALID;
    }
    if (n_clips == 0 || n_out == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t clip_bytes = size_t(n_clips) * sizeof(b200aa_pcm_clip);
    const int64_t tiles = (n_out + pcm::kTile - 1) / pcm::kTile;
    const int64_t items = n_clips * tiles;
    const unsigned grid = unsigned(std::min<int64_t>(items, int64_t(1) << 30));
    StreamScratch scratch(st);
    int rc = scratch.alloc(clip_bytes);
    if (rc != B200AA_OK) return rc;
    const b200aa_pcm_clip *d_clips = static_cast<const b200aa_pcm_clip *>(scratch.get());
    const cudaError_t e = cudaMemcpyAsync(scratch.get(), h_clips, clip_bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpyAsync");
    const unsigned char *arena = static_cast<const unsigned char *>(d_arena);
    if (out_dtype == B200AA_DTYPE_I16)
        pcm::decode_kernel<<<grid, pcm::kThreads, 0, st>>>(arena, d_clips, items, tiles, n_out, out_stride,
                                                           static_cast<int16_t *>(d_out));
    else
        pcm::decode_kernel<<<grid, pcm::kThreads, 0, st>>>(arena, d_clips, items, tiles, n_out, out_stride,
                                                           static_cast<float *>(d_out));
    return scratch.done(launched("pcm::decode_kernel"));
}

// ------------------------------------------------------------------------------------------------
// kernel 4: beat extraction (MidTermFeatures.py:18-84), bit for bit the host beat_extraction (csrc/beat.cuh)
// ------------------------------------------------------------------------------------------------
// One CTA of P = blockDim.x threads (a power of two, 32 .. 256) per (clip, beat row): threshold, chunked peak scan, and the
// distances between successive peaks counted into the row's integer histogram counts[row][d - 1], d = 1 .. min(mbt, T - 1).
__global__ void __launch_bounds__(256) beat_rows_kernel(const float *st, int F, int64_t n_frames, int64_t t_stride,
                                                        const int64_t *frames, int64_t b0, int64_t mbt, int nb, int chunk,
                                                        int nch_max, beat::Chunk *recs, unsigned *counts)
{
    __shared__ double part[256];
    const int64_t bl = blockIdx.x / beat::kRows;
    const int r = int(blockIdx.x - bl * beat::kRows);
    const int64_t b = b0 + bl;
    const int64_t T = frames ? min(max(frames[b], int64_t(0)), n_frames) : n_frames;
    const float *row = st + (size_t(b) * F + beat::row_index(r)) * t_stride;
    const int P = blockDim.x, k = threadIdx.x;
    auto v = [row](int64_t i) { return double(row[i]); };
    auto absdiff = [row](int64_t i) { return fabs(beat::dsub(double(row[i]), double(row[i + 1]))); };

    const int64_t n = T > 1 ? T - 1 : 0;
    int64_t off, len;
    beat::pairwise_part(n, __ffs(P) - 1, k, off, len);
    part[k] = beat::pairwise_sum(absdiff, off, len, n);
    __syncthreads();
    for (int s = 1; s < P; s <<= 1) {
        if ((k & (2 * s - 1)) == 0) part[k] = beat::dadd(part[k], part[k + s]);
        __syncthreads();
    }
    const double delta = beat::threshold(part[0], T);

    const int32_t nch = int32_t((T + chunk - 1) / chunk);
    beat::Chunk *rec = recs + (size_t(bl) * beat::kRows + r) * nch_max;
    if (nch > 1) {
        for (int32_t c = k; c < nch; c += P)                                 // speculative pass, every chunk from the fresh state
            rec[c] = beat::spec_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta);
        __syncthreads();
        if (k == 0) {                                                         // fix-up, serial over the chunks
            beat::State s = rec[0].s;
            int32_t last = rec[0].last;
            for (int32_t c = 1; c < nch; ++c) {
                const beat::Chunk spec = rec[c];
                rec[c].s = s;
                rec[c].last = last;
                beat::fixup_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta, spec, s, last);
            }
        }
        __syncthreads();
    }
    unsigned *cnt = counts + (size_t(bl) * beat::kRows + r) * nb;
    for (int32_t c = k; c < nch; c += P) {                                    // counting pass from the true entry states
        int32_t last = c ? rec[c].last : -1;
        beat::scan_chunk(v, c * chunk, int32_t(min(T, int64_t(c + 1) * chunk)), delta, c ? rec[c].s : beat::fresh(),
                         [&](int32_t p) {
                             if (last >= 0 && p - last >= 1 && p - last <= mbt) atomicAdd(cnt + (p - last - 1), 1u);
                             last = p;
                         });
    }
}

// One warp per clip: hist[k] = sum over the rows, in _BEAT_ROWS order, of counts[row][k] / T; its first maximum k, and its
// pairwise sum over all mbt bins (bins >= nb are zero).  d_out[b] = (60 / ((k + 1) * window), hist[k] / (sum + 1e-8)).
__global__ void __launch_bounds__(256) beat_finish_kernel(const int64_t *frames, int64_t n_frames, int64_t b0, int64_t n_slice,
                                                          double window, int64_t mbt, int nb, const unsigned *counts, double *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t bl = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    if (bl >= n_slice) return;
    const int64_t b = b0 + bl;
    const int64_t T = frames ? min(max(frames[b], int64_t(0)), n_frames) : n_frames;
    if (T == 0) {               // every bin is 0 / 0: np.argmax picks the first NaN, the ratio is NaN
        if (lane == 0) {
            out[2 * b] = beat::ddiv(60.0, beat::dmul(1.0, window));
            out[2 * b + 1] = __longlong_as_double(0x7ff8000000000000LL);
        }
        return;
    }
    const unsigned *cnt = counts + size_t(bl) * beat::kRows * nb;
    const double Td = double(T);
    auto hist = [cnt, nb, Td](int64_t k) {
        double h = 0.0;
        for (int r = 0; r < beat::kRows; ++r) h = beat::dadd(h, beat::ddiv(double(cnt[size_t(r) * nb + k]), Td));
        return h;
    };
    double bv = 0.0;            // every bin is >= 0: (0.0, 0) is the answer when all are zero
    int64_t bk = 0;
    for (int64_t k = lane; k < nb; k += 32) {
        const double h = hist(k);
        if (h > bv) { bv = h; bk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int64_t ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov > bv || (ov == bv && ok < bk)) { bv = ov; bk = ok; }
    }
    int64_t off, len;
    beat::pairwise_part(mbt, 5, lane, off, len);
    double s = beat::pairwise_sum(hist, off, len, nb);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_down_sync(0xffffffffu, s, o);
        if ((lane & (2 * o - 1)) == 0) s = beat::dadd(s, t);
    }
    if (lane == 0) {
        out[2 * b] = beat::ddiv(60.0, beat::dmul(double(bk + 1), window));
        out[2 * b + 1] = beat::ddiv(bv, beat::dadd(s, 0.00000001));
    }
}

extern "C" int b200aa_beat_extraction(const float *d_st, int64_t n_clips, int n_feats, int64_t n_frames, int64_t t_stride,
                                      const int64_t *d_frames, double window_size, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_beat_extraction");
    if (!d_st || !d_out || n_clips < 0 || n_feats < 19 || n_frames < 0 || n_frames > INT32_MAX - beat::kChunk ||
        t_stride < n_frames)
        return B200AA_ERR_INVALID;
    const double mbt_d = std::nearbyint(2.0 / window_size);               // Python's round(): half to even
    if (!(mbt_d >= 1.0) || mbt_d > double(INT32_MAX)) return B200AA_ERR_INVALID;
    if (n_clips == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t mbt = int64_t(mbt_d);
    const int nb = int(std::min<int64_t>(mbt, std::max<int64_t>(n_frames - 1, 0)));
    const int chunk = beat::kChunk;
    const int nch_max = int(std::max<int64_t>(1, (n_frames + chunk - 1) / chunk));
    int P = 32;
    while (P < nch_max && P < 256) P <<= 1;
    // scratch per clip: the rows' histograms and, for rows of more than one chunk, their chunk records; clips go in slices
    // whose scratch stays below 256 MiB
    const size_t rec_bytes = nch_max > 1 ? size_t(nch_max) * sizeof(beat::Chunk) : 0;
    const size_t per_clip = size_t(beat::kRows) * (size_t(nb) * sizeof(unsigned) + rec_bytes);
    const int64_t slice = std::max<int64_t>(1, std::min<int64_t>({n_clips, int64_t((size_t(256) << 20) / std::max<size_t>(per_clip, 1)),
                                                                   int64_t(INT32_MAX / beat::kRows)}));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(size_t(slice) * per_clip);
    if (rc != B200AA_OK) return rc;
    unsigned *counts = static_cast<unsigned *>(scratch.get());
    beat::Chunk *recs = reinterpret_cast<beat::Chunk *>(static_cast<char *>(scratch.get()) + size_t(slice) * beat::kRows * nb * sizeof(unsigned));
    for (int64_t b0 = 0; b0 < n_clips; b0 += slice) {
        const int64_t ns = std::min<int64_t>(slice, n_clips - b0);
        const cudaError_t e = nb ? cudaMemsetAsync(counts, 0, size_t(ns) * beat::kRows * nb * sizeof(unsigned), st) : cudaSuccess;
        if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync");
        beat_rows_kernel<<<(unsigned)(ns * beat::kRows), P, 0, st>>>(d_st, n_feats, n_frames, t_stride, d_frames, b0, mbt, nb, chunk,
                                                                     nch_max, recs, counts);
        CK_LAUNCH("beat_rows_kernel");
        beat_finish_kernel<<<(unsigned)((ns * 32 + 255) / 256), 256, 0, st>>>(d_frames, n_frames, b0, ns, window_size, mbt, nb,
                                                                               counts, d_out);
        CK_LAUNCH("beat_finish_kernel");
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernels 5 and 6: kNN classification (audioTrainTest.py:33-49), bit for bit the reference's Knn.classify per query
// (csrc/knn.cuh), and its cross-validation (audioTrainTest.py:576-771, csrc/knn_cv.cuh)
// ------------------------------------------------------------------------------------------------
// The distance and select kernels run a batch of problems (knn::Problem): `probs` on the device, one problem per grid z
// (distance) or y (select).  Kernel 5 passes NULL and its one problem by value in `one`.
//
// keys[q][i] = key_of(distance(query q, training row i)) for a 64-query x 64-row tile per CTA.  Both tiles are staged
// 16 features at a time, transposed to [feature][row]; each thread runs 4 x 4 independent chains (queries ty + 16a,
// rows tx + 16b), so the 136-long dependent DADD chain of one pair is hidden behind 15 others.
template <class Tq>
__global__ void __launch_bounds__(knn::kThreads, 3) knn_dist_kernel(const knn::Problem *__restrict__ probs, knn::Problem one,
                                                                 const double *__restrict__ feats, int F,
                                                                 const Tq *__restrict__ q, int64_t q_stride,
                                                                 uint64_t *__restrict__ keys)
{
    static_assert(knn::kQ == knn::kT && knn::kQ == 64 && knn::kThreads == 256, "tile shape");
    __shared__ double sq[knn::kF][knn::kQ + 1];
    __shared__ double sv[knn::kF][knn::kT + 1];
    const knn::Problem pb = probs ? probs[blockIdx.z] : one;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t t0 = int64_t(blockIdx.x) * knn::kT;
    const int64_t q0 = int64_t(blockIdx.y) * knn::kQ;
    const int64_t N = pb.N, n_slice = pb.n_q;
    if (t0 >= N || q0 >= n_slice) return;       // a tile past this problem: the grid covers the batch's largest
    feats += pb.train0 * F;
    q += pb.q0 * q_stride;
    keys += pb.key0;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int f0 = 0; f0 < F; f0 += knn::kF) {
        const int nf = min(knn::kF, F - f0);
        __syncthreads();
        for (int e = threadIdx.x; e < knn::kQ * knn::kF; e += knn::kThreads) {
            const int r = e / knn::kF, j = e % knn::kF;
            const int64_t qi = q0 + r, ti = t0 + r;
            sq[j][r] = (j < nf && qi < n_slice) ? double(q[qi * q_stride + f0 + j]) : 0.0;      // float32: widened exactly
            sv[j][r] = (j < nf && ti < N) ? feats[ti * F + f0 + j] : 0.0;
        }
        __syncthreads();
#pragma unroll 2
        for (int j = 0; j < nf; ++j) {
            double x[4], v[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) x[a] = sq[j][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 4; ++b) v[b] = sv[j][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = knn::dist_step(acc[a][b], x[a], v[b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int64_t qi = q0 + ty + 16 * a;
        if (qi >= n_slice) continue;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int64_t ti = t0 + tx + 16 * b;
            if (ti < N) keys[qi * N + ti] = knn::key_of(knn::dsqrt(acc[a][b]));
        }
    }
}

// One CTA per query: the k-th smallest key by radix select (8 passes of 256 bins over the keys sharing the prefix found so
// far), then one pass in training-index order that selects the keys below it and the first r equal to it, counting the
// selected entries' classes in shared memory, kVoteClasses classes per pass.  Kernel 5 (kCounts false) writes P[q][0..C)
// and the first maximum as ids[q]; kernel 6 writes the first maximum as pred[q] and counts it in the problem's confusion
// block, counts[id][truth][pred] (integer atomics: the counts do not depend on the order).
struct KnnVotes {
    int64_t *ids;
    double *P;
    int32_t *pred;
    const int32_t *truth;               // kernel 6: the class of each query row; outside [0, n_classes) it is not counted
    unsigned long long *counts;
    int n_classes;
};

template <bool kCounts>
__global__ void __launch_bounds__(knn::kThreads) knn_select_kernel(const knn::Problem *__restrict__ probs, knn::Problem one,
                                                                   const uint64_t *__restrict__ keys,
                                                                   const int32_t *__restrict__ slots, KnnVotes out)
{
    constexpr int kWarps = knn::kThreads / 32;
    __shared__ unsigned hist[knn::kBins];
    __shared__ unsigned votes[knn::kVoteClasses];
    __shared__ unsigned warp_eq[kWarps];
    __shared__ int64_t warp_best_c[kWarps], warp_best_i[kWarps];
    __shared__ uint64_t s_prefix;
    __shared__ int64_t s_rank;
    const knn::Problem pb = probs ? probs[blockIdx.y] : one;
    if (blockIdx.x >= pb.n_q) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t N = pb.N, k = pb.k;
    const int C = pb.C;
    const int64_t q = pb.out0 + blockIdx.x;
    const uint64_t *row = keys + pb.key0 + int64_t(blockIdx.x) * N;
    slots += pb.train0;

    uint64_t thr = knn::kAll;           // k >= N: every entry is selected
    int64_t r = 0;
    if (k < N) {
        uint64_t prefix = 0;
        int64_t rank = k;
        for (int shift = 64 - knn::kDigitBits; shift >= 0; shift -= knn::kDigitBits) {
            const uint64_t mask = knn::prefix_mask(shift);
            for (int b = tid; b < knn::kBins; b += knn::kThreads) hist[b] = 0;
            __syncthreads();
            for (int64_t i = tid; i < N; i += knn::kThreads) {
                const uint64_t key = row[i];
                if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & (knn::kBins - 1)], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                const int d = knn::select_digit(hist, rank);
                s_prefix = prefix | (uint64_t(d) << shift);
                s_rank = rank;
            }
            __syncthreads();
            prefix = s_prefix;
            rank = s_rank;
        }
        thr = prefix;
        r = rank;
    }

    int64_t best_c = -1, best_i = 0;    // thread 0: the first maximum over the classes done so far
    for (int c0 = 0; c0 < C; c0 += knn::kVoteClasses) {
        const int nc = min(knn::kVoteClasses, C - c0);
        for (int c = tid; c < knn::kVoteClasses; c += knn::kThreads) votes[c] = 0;
        __syncthreads();
        int64_t eq_done = 0;            // keys equal to thr at indices below this chunk
        for (int64_t base = 0; base < N; base += knn::kThreads) {
            const int64_t i = base + tid;
            const uint64_t key = i < N ? row[i] : 0;
            const bool eq = i < N && key == thr;
            const unsigned m = __ballot_sync(0xffffffffu, eq);
            if (lane == 0) warp_eq[warp] = __popc(m);
            __syncthreads();
            int64_t before = eq_done + __popc(m & ((1u << lane) - 1u)), total = 0;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) {
                if (w < warp) before += warp_eq[w];
                total += warp_eq[w];
            }
            if (i < N && knn::selected(key, thr, before, r)) {
                const int s = slots[i];
                if (s >= c0 && s < c0 + nc) atomicAdd(&votes[s - c0], 1u);
            }
            eq_done += total;
            __syncthreads();
        }
        int64_t bc = -1, bi = 0;
        for (int c = tid; c < nc; c += knn::kThreads) {
            if (!kCounts) out.P[q * C + c0 + c] = knn::vote(votes[c], k);
            if (bc < 0 || knn::better(votes[c], c0 + c, bc, bi)) { bc = votes[c]; bi = c0 + c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int64_t oc = __shfl_xor_sync(0xffffffffu, bc, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oc >= 0 && (bc < 0 || knn::better(oc, oi, bc, bi))) { bc = oc; bi = oi; }
        }
        if (lane == 0) { warp_best_c[warp] = bc; warp_best_i[warp] = bi; }
        __syncthreads();
        if (tid == 0)
            for (int w = 0; w < kWarps; ++w)
                if (warp_best_c[w] >= 0 && (best_c < 0 || knn::better(warp_best_c[w], warp_best_i[w], best_c, best_i))) {
                    best_c = warp_best_c[w];
                    best_i = warp_best_i[w];
                }
        __syncthreads();
    }
    if (tid == 0) {
        if (kCounts) {
            out.pred[q] = int32_t(best_i);
            const int32_t t = out.truth[pb.q0 + blockIdx.x];
            if (t >= 0 && t < out.n_classes)
                atomicAdd(&out.counts[(int64_t(pb.id) * out.n_classes + t) * out.n_classes + best_i], 1ull);
        } else {
            out.ids[q] = best_i;
        }
    }
}

extern "C" int b200aa_knn_classify(const double *d_feats, const int32_t *d_slots, int64_t n_train, int n_feats, int n_classes,
                                   int64_t k, const void *d_query, int dtype, int64_t n_query, int64_t q_stride, int64_t *d_ids,
                                   double *d_P, void *stream)
{
    NvtxRange nvtx_("b200aa_knn_classify");
    if (!d_feats || !d_slots || !d_query || !d_ids || !d_P || n_train < 1 || n_train > INT32_MAX || n_feats < 1 ||
        n_classes < 1 || k < 1 || n_query < 0 || q_stride < n_feats || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (n_query == 0) return B200AA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // scratch: one key per (query, training row); queries go in slices whose keys stay below 256 MiB
    const size_t row_bytes = size_t(n_train) * sizeof(uint64_t);
    const int64_t slice = std::max<int64_t>(1, std::min<int64_t>({n_query, int64_t((size_t(256) << 20) / row_bytes),
                                                                   int64_t(65535) * knn::kQ}));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(size_t(slice) * row_bytes);
    if (rc != B200AA_OK) return rc;
    uint64_t *keys = static_cast<uint64_t *>(scratch.get());
    for (int64_t q0 = 0; q0 < n_query; q0 += slice) {
        const int64_t ns = std::min<int64_t>(slice, n_query - q0);
        const knn::Problem one{0, n_train, 0, ns, 0, q0, k, 0, 0, n_classes, 0};
        const dim3 grid((unsigned)((n_train + knn::kT - 1) / knn::kT), (unsigned)((ns + knn::kQ - 1) / knn::kQ));
        if (dtype == B200AA_DTYPE_F32)
            knn_dist_kernel<<<grid, knn::kThreads, 0, st>>>(nullptr, one, d_feats, n_feats,
                                                            static_cast<const float *>(d_query) + q0 * q_stride, q_stride, keys);
        else
            knn_dist_kernel<<<grid, knn::kThreads, 0, st>>>(nullptr, one, d_feats, n_feats,
                                                            static_cast<const double *>(d_query) + q0 * q_stride, q_stride, keys);
        CK_LAUNCH("knn_dist_kernel");
        KnnVotes out{};
        out.ids = d_ids;
        out.P = d_P;
        knn_select_kernel<false><<<(unsigned)ns, knn::kThreads, 0, st>>>(nullptr, one, keys, d_slots, out);
        CK_LAUNCH("knn_select_kernel");
    }
    return scratch.done(B200AA_OK);
}

// Kernel 6, first step of a slice: per (problem, column) StandardScaler().fit over the problem's training rows in the
// split's order, then its training and query rows standardised into the slice's matrices, the training rows' slots and
// the query rows' classes.  One thread per column: each fit is a sequential chain, as scikit-learn sums it.
__global__ void __launch_bounds__(knn::kFitThreads) knn_cv_gather_kernel(const knn::Problem *__restrict__ probs,
                                                                         const double *__restrict__ X, const int32_t *__restrict__ y,
                                                                         int F, const int32_t *__restrict__ train_idx,
                                                                         const int32_t *__restrict__ test_idx,
                                                                         double *__restrict__ train, double *__restrict__ query,
                                                                         int32_t *__restrict__ slots, int32_t *__restrict__ truth)
{
    const knn::Problem pb = probs[blockIdx.y];
    const int32_t *tr = train_idx + pb.src_train, *te = test_idx + pb.src_test;
    if (blockIdx.x == 0) {
        for (int64_t i = threadIdx.x; i < pb.N; i += knn::kFitThreads) slots[pb.train0 + i] = knn::split_slot(y[tr[i]], pb.C);
        for (int64_t i = threadIdx.x; i < pb.n_q; i += knn::kFitThreads) truth[pb.q0 + i] = y[te[i]];
    }
    const int j = blockIdx.x * knn::kFitThreads + threadIdx.x;
    if (j >= F) return;
    const knn::Scale s = knn::scaler_fit([&](int64_t i) { return X[int64_t(tr[i]) * F + j]; }, pb.N);
    for (int64_t i = 0; i < pb.N; ++i) train[(pb.train0 + i) * F + j] = knn::standardise(X[int64_t(tr[i]) * F + j], s);
    for (int64_t i = 0; i < pb.n_q; ++i) query[(pb.q0 + i) * F + j] = knn::standardise(X[int64_t(te[i]) * F + j], s);
}

// The host half of kernel 6: validates the splits, cuts them into work items (a problem, or a range of its test rows when
// one problem's scratch passes the bound) and packs the items into slices whose scratch stays under kSliceBytes.
namespace {
constexpr size_t kSliceBytes = size_t(256) << 20;
constexpr int64_t kMaxItems = 65535;    // grid z of the distance kernel, grid y of the select kernel

struct CvSlice {
    int64_t first, end;                 // items [first, end)
    int64_t train_rows, query_rows, keys, max_N, max_q;
};

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }
}  // namespace

extern "C" int b200aa_knn_cross_validate(const double *d_X, const int32_t *d_y, int64_t n, int n_feats, int n_classes,
                                         int64_t n_problems, const int64_t *h_train_off, const int32_t *h_train_idx,
                                         const int64_t *h_test_off, const int32_t *h_test_idx, const int64_t *h_k,
                                         const int32_t *h_classes, int32_t *d_pred, int64_t *d_counts, void *stream)
{
    NvtxRange nvtx_("b200aa_knn_cross_validate");
    if (!d_X || !d_y || !h_train_off || !h_train_idx || !h_test_off || !h_test_idx || !h_k || !h_classes || !d_pred ||
        !d_counts || n < 1 || n > INT32_MAX || n_feats < 1 || n_classes < 1 || n_problems < 0 || h_train_off[0] != 0 ||
        h_test_off[0] != 0)
        return B200AA_ERR_INVALID;
    for (int64_t p = 0; p < n_problems; ++p)
        if (h_train_off[p + 1] - h_train_off[p] < 1 || h_test_off[p + 1] - h_test_off[p] < 1 || h_k[p] < 1 ||
            h_classes[p] < 1 || h_classes[p] > n_classes)
            return B200AA_ERR_INVALID;
    const int64_t n_train_all = h_train_off[n_problems], n_test_all = h_test_off[n_problems];
    for (int64_t i = 0; i < n_train_all; ++i)
        if (h_train_idx[i] < 0 || h_train_idx[i] >= n) return B200AA_ERR_INVALID;
    for (int64_t i = 0; i < n_test_all; ++i)
        if (h_test_idx[i] < 0 || h_test_idx[i] >= n) return B200AA_ERR_INVALID;
    if (n_problems == 0) return B200AA_OK;

    // work items and slices: per item its standardised rows, slots / classes and keys
    const size_t row = size_t(n_feats) * sizeof(double) + sizeof(int32_t);
    std::vector<knn::Problem> items;
    std::vector<CvSlice> slices;
    CvSlice cur{0, 0, 0, 0, 0, 0, 0};
    size_t cur_bytes = 0;
    for (int64_t p = 0; p < n_problems; ++p) {
        const int64_t N = h_train_off[p + 1] - h_train_off[p], T = h_test_off[p + 1] - h_test_off[p];
        const size_t fixed = size_t(N) * row, per_q = row + size_t(N) * sizeof(uint64_t);
        const int64_t fit = fixed < kSliceBytes ? int64_t((kSliceBytes - fixed) / per_q) : 0;
        const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>({T, fit, int64_t(65535) * knn::kQ}));
        for (int64_t a = 0; a < T; a += chunk) {
            const int64_t nq = std::min(chunk, T - a);
            const size_t bytes = fixed + size_t(nq) * per_q;
            if (cur.end > cur.first && (cur_bytes + bytes > kSliceBytes || cur.end - cur.first == kMaxItems)) {
                slices.push_back(cur);
                cur = CvSlice{cur.end, cur.end, 0, 0, 0, 0, 0};
                cur_bytes = 0;
            }
            items.push_back(knn::Problem{cur.train_rows, N, cur.query_rows, nq, cur.keys, h_test_off[p] + a, h_k[p],
                                         h_train_off[p], h_test_off[p] + a, h_classes[p], int32_t(p)});
            cur.end++;
            cur.train_rows += N;
            cur.query_rows += nq;
            cur.keys += N * nq;
            cur.max_N = std::max(cur.max_N, N);
            cur.max_q = std::max(cur.max_q, nq);
            cur_bytes += bytes;
        }
    }
    slices.push_back(cur);

    // scratch: [items | training indices | test indices] uploaded once, then one slice's matrices, slots, classes, keys
    size_t train_b = 0, query_b = 0, slots_b = 0, truth_b = 0, keys_b = 0;
    for (const CvSlice &s : slices) {
        train_b = std::max(train_b, align256(size_t(s.train_rows) * n_feats * sizeof(double)));
        query_b = std::max(query_b, align256(size_t(s.query_rows) * n_feats * sizeof(double)));
        slots_b = std::max(slots_b, align256(size_t(s.train_rows) * sizeof(int32_t)));
        truth_b = std::max(truth_b, align256(size_t(s.query_rows) * sizeof(int32_t)));
        keys_b = std::max(keys_b, align256(size_t(s.keys) * sizeof(uint64_t)));
    }
    const size_t items_b = align256(items.size() * sizeof(knn::Problem));
    const size_t tr_b = align256(size_t(n_train_all) * sizeof(int32_t)), te_b = size_t(n_test_all) * sizeof(int32_t);
    std::vector<char> blob(items_b + tr_b + te_b);
    std::memcpy(blob.data(), items.data(), items.size() * sizeof(knn::Problem));
    std::memcpy(blob.data() + items_b, h_train_idx, size_t(n_train_all) * sizeof(int32_t));
    std::memcpy(blob.data() + items_b + tr_b, h_test_idx, te_b);

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t head_b = align256(blob.size());
    StreamScratch scratch(st);
    const int rc = scratch.alloc(head_b + train_b + query_b + slots_b + truth_b + keys_b);
    if (rc != B200AA_OK) return rc;
    char *base = static_cast<char *>(scratch.get());
    const knn::Problem *d_items = reinterpret_cast<const knn::Problem *>(base);
    const int32_t *d_tr = reinterpret_cast<const int32_t *>(base + items_b);
    const int32_t *d_te = reinterpret_cast<const int32_t *>(base + items_b + tr_b);
    double *train = reinterpret_cast<double *>(base + head_b);
    double *query = reinterpret_cast<double *>(base + head_b + train_b);
    int32_t *slots = reinterpret_cast<int32_t *>(base + head_b + train_b + query_b);
    int32_t *truth = reinterpret_cast<int32_t *>(base + head_b + train_b + query_b + slots_b);
    uint64_t *keys = reinterpret_cast<uint64_t *>(base + head_b + train_b + query_b + slots_b + truth_b);
    CK(cudaMemcpyAsync(base, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_counts, 0, size_t(n_problems) * n_classes * n_classes * sizeof(int64_t), st));

    KnnVotes out{};
    out.pred = d_pred;
    out.truth = truth;
    out.counts = reinterpret_cast<unsigned long long *>(d_counts);
    out.n_classes = n_classes;
    const knn::Problem none{};
    for (const CvSlice &s : slices) {
        const unsigned n_items = unsigned(s.end - s.first);
        const knn::Problem *probs = d_items + s.first;
        knn_cv_gather_kernel<<<dim3((n_feats + knn::kFitThreads - 1) / knn::kFitThreads, n_items), knn::kFitThreads, 0, st>>>(
            probs, d_X, d_y, n_feats, d_tr, d_te, train, query, slots, truth);
        CK_LAUNCH("knn_cv_gather_kernel");
        const dim3 grid((unsigned)((s.max_N + knn::kT - 1) / knn::kT), (unsigned)((s.max_q + knn::kQ - 1) / knn::kQ), n_items);
        knn_dist_kernel<<<grid, knn::kThreads, 0, st>>>(probs, none, train, n_feats, static_cast<const double *>(query),
                                                        int64_t(n_feats), keys);
        CK_LAUNCH("knn_dist_kernel");
        knn_select_kernel<true><<<dim3((unsigned)s.max_q, n_items), knn::kThreads, 0, st>>>(probs, none, keys, slots, out);
        CK_LAUNCH("knn_select_kernel");
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernel 7: HMM segmentation (audioSegmentation.py:287-344, :471-492), bit for bit the NumPy restatement (csrc/hmm.cuh)
// ------------------------------------------------------------------------------------------------
// One thread per (class, feature): the class's windows in the concatenated order, a sequential chain (pairwise for F == 1).
// col[i] is the element offset of window i's feature 0; out is [4, C, F]: sum, mean, ssq, std.
template <class T>
__global__ void __launch_bounds__(128) hmm_stats_kernel(const T *__restrict__ mid, int F, int64_t m_stride,
                                                        const int64_t *__restrict__ col, const int64_t *__restrict__ class_off,
                                                        int C, double *__restrict__ out)
{
    const int64_t w = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    if (w >= int64_t(C) * F) return;
    const int c = int(w / F), f = int(w - int64_t(c) * F);
    const int64_t a = class_off[c], n = class_off[c + 1] - a;
    const T *row = mid + int64_t(f) * m_stride;
    const int64_t *ix = col + a;
    const hmm::ClassStats s = hmm::class_stats([&](int64_t i) { return double(row[ix[i]]); }, n, F == 1);
    const int64_t cf = int64_t(C) * F;
    out[w] = s.sum;
    out[cf + w] = s.mean;
    out[2 * cf + w] = s.ssq;
    out[3 * cf + w] = s.std;
}

// One thread per (clip, window, state), consecutive threads on consecutive windows of one (clip, state): e[row, state] of the
// slice, row = the clip's first row + window.  clips[2b] = the clip's window count, clips[2b + 1] its first global row.
// A non-finite feature of a valid window raises bad[b].
__global__ void __launch_bounds__(128) hmm_emission_kernel(const float *__restrict__ mid, int F, int64_t m_stride,
                                                           const int64_t *__restrict__ clips, int64_t b0, int64_t row_base,
                                                           int C, const double *__restrict__ mu, const double *__restrict__ var,
                                                           const double *__restrict__ konst, double *__restrict__ e,
                                                           int32_t *__restrict__ bad)
{
    const int64_t b = b0 + blockIdx.z;
    const int j = blockIdx.y;
    const int64_t t = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
    const int64_t n = clips[2 * b];
    if (t >= n) return;
    const float *x = mid + size_t(b) * F * m_stride + t;
    auto xf = [&](int64_t f) { return double(x[f * m_stride]); };
    if (j == 0) {
        bool finite = true;
        for (int f = 0; f < F; ++f) finite &= isfinite(x[int64_t(f) * m_stride]);
        if (!finite) bad[b] = 1;
    }
    e[(clips[2 * b + 1] - row_base + t) * C + j] =
        hmm::emission(xf, mu + size_t(j) * F, var + size_t(j) * F, F, konst[j], n == 1);
}

// One warp per clip: the forward pass serial in t, lanes on states j, j + 32, ...; delta_{t-1} and delta_t in shared memory,
// the backpointers in the slice's scratch; then lane 0 backtracks.  ids[b, t] for t < n, zero up to m_stride; a refused clip
// (bad[b]) is not written.
__global__ void __launch_bounds__(32) hmm_viterbi_kernel(const int64_t *__restrict__ clips, int64_t b0, int64_t row_base, int C,
                                                         int64_t m_stride, const double *__restrict__ log_start,
                                                         const double *__restrict__ log_trans, const double *__restrict__ e,
                                                         int32_t *__restrict__ bp, const int32_t *__restrict__ bad,
                                                         int32_t *__restrict__ ids)
{
    extern __shared__ double delta[];
    const int64_t b = b0 + blockIdx.x;
    if (bad[b]) return;
    const int64_t n = clips[2 * b], r0 = clips[2 * b + 1] - row_base;
    const int lane = threadIdx.x;
    const double *eb = e + r0 * C;
    int32_t *bpb = bp + r0 * C;
    double *cur = delta, *prev = delta + C;
    for (int j = lane; j < C; j += 32) cur[j] = hmm::dadd(log_start[j], eb[j]);
    for (int64_t t = 1; t < n; ++t) {
        double *tmp = prev;
        prev = cur;
        cur = tmp;
        __syncwarp();
        for (int j = lane; j < C; j += 32) {
            int32_t p;
            cur[j] = hmm::step([prev](int32_t i) { return prev[i]; }, [log_trans, C, j](int32_t i) { return log_trans[int64_t(i) * C + j]; },
                               C, eb[t * C + j], p);
            bpb[t * C + j] = p;
        }
    }
    __syncwarp();
    int32_t *out = ids + size_t(b) * m_stride;
    if (lane == 0) {
        int32_t s = hmm::last_state([cur](int32_t i) { return cur[i]; }, C);
        out[n - 1] = s;
        for (int64_t t = n - 1; t > 0; --t) {
            s = bpb[t * C + s];
            out[t - 1] = s;
        }
    }
    for (int64_t t = n + lane; t < m_stride; t += 32) out[t] = 0;
}

namespace {
constexpr size_t kHmmSliceBytes = size_t(256) << 20;

bool hmm_counts_ok(const int64_t *h_n, int64_t n_clips, int64_t m_stride, int64_t lo)
{
    for (int64_t b = 0; b < n_clips; ++b)
        if (h_n[b] < lo || h_n[b] > m_stride) return false;
    return true;
}
}  // namespace

extern "C" int b200aa_hmm_statistics(const void *d_mid, int dtype, int64_t n_clips, int n_feats, int64_t m_stride,
                                     const int64_t *h_n_windows, int n_classes, const int64_t *h_class_off,
                                     const int64_t *h_idx, double *d_out, void *stream)
{
    NvtxRange nvtx_("b200aa_hmm_statistics");
    if (!d_mid || !h_n_windows || !h_class_off || !h_idx || !d_out || n_clips < 1 || n_feats < 1 || m_stride < 1 ||
        n_classes < 1 || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64) || h_class_off[0] != 0 ||
        !hmm_counts_ok(h_n_windows, n_clips, m_stride, 0))
        return B200AA_ERR_INVALID;
    std::vector<int64_t> first(size_t(n_clips) + 1, 0);              // first concatenated window of each clip
    for (int64_t b = 0; b < n_clips; ++b) first[b + 1] = first[b] + h_n_windows[b];
    for (int c = 0; c < n_classes; ++c)
        if (h_class_off[c + 1] < h_class_off[c]) return B200AA_ERR_INVALID;
    const int64_t n_idx = h_class_off[n_classes];
    // [class offsets | element offset of each listed window's feature 0]
    std::vector<int64_t> head(size_t(n_classes) + 1 + size_t(n_idx));
    std::memcpy(head.data(), h_class_off, (size_t(n_classes) + 1) * sizeof(int64_t));
    for (int64_t i = 0; i < n_idx; ++i) {
        const int64_t g = h_idx[i];
        if (g < 0 || g >= first[n_clips]) return B200AA_ERR_INVALID;
        const int64_t b = int64_t(std::upper_bound(first.begin(), first.end(), g) - first.begin()) - 1;
        head[n_classes + 1 + i] = b * n_feats * m_stride + (g - first[b]);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamScratch scratch(st);
    const int rc = scratch.alloc(head.size() * sizeof(int64_t));
    if (rc != B200AA_OK) return rc;
    int64_t *d_head = static_cast<int64_t *>(scratch.get());
    CK(cudaMemcpyAsync(d_head, head.data(), head.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const int64_t threads = int64_t(n_classes) * n_feats;
    const unsigned blocks = unsigned((threads + 127) / 128);
    if (dtype == B200AA_DTYPE_F32)
        hmm_stats_kernel<<<blocks, 128, 0, st>>>(static_cast<const float *>(d_mid), n_feats, m_stride, d_head + n_classes + 1,
                                                 d_head, n_classes, d_out);
    else
        hmm_stats_kernel<<<blocks, 128, 0, st>>>(static_cast<const double *>(d_mid), n_feats, m_stride, d_head + n_classes + 1,
                                                 d_head, n_classes, d_out);
    CK_LAUNCH("hmm_stats_kernel");
    return scratch.done(B200AA_OK);
}

extern "C" int b200aa_hmm_decode(const float *d_mid, int64_t n_clips, int n_feats, int64_t m_stride, const int64_t *h_n_windows,
                                 int n_states, const double *d_log_start, const double *d_log_trans, const double *d_means,
                                 const double *d_vars, const double *d_const, int32_t *d_ids, int32_t *d_bad, void *stream)
{
    NvtxRange nvtx_("b200aa_hmm_decode");
    if (!d_mid || !h_n_windows || !d_log_start || !d_log_trans || !d_means || !d_vars || !d_const || !d_ids || !d_bad ||
        n_clips < 1 || n_feats < 1 || m_stride < 1 || n_states < 1 || n_states > hmm::kMaxStates ||
        !hmm_counts_ok(h_n_windows, n_clips, m_stride, 1))
        return B200AA_ERR_INVALID;
    // per clip (window count, first global row); slices of whole clips whose e + backpointers stay under kHmmSliceBytes
    // (a clip larger than that on its own is a slice of its own), at most 65535 clips (grid z)
    const size_t row_bytes = size_t(n_states) * (sizeof(double) + sizeof(int32_t));
    std::vector<int64_t> clips(2 * size_t(n_clips));
    std::vector<int64_t> cuts{0};
    int64_t rows = 0, slice_rows = 0, max_rows = 0;
    for (int64_t b = 0; b < n_clips; ++b) {
        const int64_t n = h_n_windows[b];
        if (b > cuts.back() && ((slice_rows + n) * row_bytes > kHmmSliceBytes || b - cuts.back() == 65535)) {
            cuts.push_back(b);
            slice_rows = 0;
        }
        clips[2 * b] = n;
        clips[2 * b + 1] = rows;
        rows += n;
        slice_rows += n;
        max_rows = std::max(max_rows, slice_rows);
    }
    cuts.push_back(n_clips);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = 2 * size_t(n_states) * sizeof(double);
    const size_t clips_b = align256(clips.size() * sizeof(int64_t)), e_b = align256(size_t(max_rows) * n_states * sizeof(double));
    StreamScratch scratch(st);
    const int rc = scratch.alloc(clips_b + e_b + size_t(max_rows) * n_states * sizeof(int32_t));
    if (rc != B200AA_OK) return rc;
    char *base = static_cast<char *>(scratch.get());
    const int64_t *d_clips = reinterpret_cast<const int64_t *>(base);
    double *e = reinterpret_cast<double *>(base + clips_b);
    int32_t *bp = reinterpret_cast<int32_t *>(base + clips_b + e_b);
    CK(cudaMemcpyAsync(base, clips.data(), clips.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_bad, 0, size_t(n_clips) * sizeof(int32_t), st));
    for (size_t s = 0; s + 1 < cuts.size(); ++s) {
        const int64_t b0 = cuts[s], b1 = cuts[s + 1];
        int64_t max_n = 0;
        for (int64_t b = b0; b < b1; ++b) max_n = std::max(max_n, h_n_windows[b]);
        const int64_t row_base = clips[2 * b0 + 1];
        hmm_emission_kernel<<<dim3(unsigned((max_n + 127) / 128), unsigned(n_states), unsigned(b1 - b0)), 128, 0, st>>>(
            d_mid, n_feats, m_stride, d_clips, b0, row_base, n_states, d_means, d_vars, d_const, e, d_bad);
        CK_LAUNCH("hmm_emission_kernel");
        hmm_viterbi_kernel<<<unsigned(b1 - b0), 32, smem, st>>>(d_clips, b0, row_base, n_states, m_stride, d_log_start,
                                                               d_log_trans, e, bp, d_bad, d_ids);
        CK_LAUNCH("hmm_viterbi_kernel");
    }
    return scratch.done(B200AA_OK);
}

// ------------------------------------------------------------------------------------------------
// kernel 8: tree-ensemble classification, bit for bit scikit-learn's predict / predict_proba (csrc/trees.cuh)
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(b200aa_tree_node) == sizeof(trees::Node), "node layout of the C ABI");

struct b200aa_trees {
    int device;
    int64_t n_nodes, n_leaves;
    int n_trees, n_classes, n_feats, mode, allow_nan;
    void *blob;                         // [nodes | roots | values | init] on `device`
    const trees::Node *nodes;
    const int32_t *roots;
    const double *values, *init;
};

namespace {
constexpr int kTreeWarps = 4;           // warps per CTA of trees_kernel, one query row per warp at a time
}  // namespace

// One warp per query row (grid-stride).  The row, cast to float32, goes to shared memory; lane j walks tree t0 + j of
// each block of 32 trees and leaves its leaf row in shared memory; then lane c adds class c's leaf values of the block in
// tree order, so every class sum is the sequential sum over the trees.  Per warp: [x: F floats | 32 leaves | C sums].
template <class Tq>
__global__ void __launch_bounds__(kTreeWarps * 32) trees_kernel(const trees::Node *__restrict__ nodes,
                                                               const int32_t *__restrict__ roots, int n_trees,
                                                               const double *__restrict__ values,
                                                               const double *__restrict__ init, int mode, int C, int F,
                                                               bool allow_nan, const Tq *__restrict__ q, int64_t n,
                                                               int64_t stride, int64_t *__restrict__ ids,
                                                               double *__restrict__ scores, int32_t *__restrict__ bad)
{
    extern __shared__ __align__(16) unsigned char trees_smem[];
    const int w = threadIdx.x / 32, lane = threadIdx.x % 32;
    const size_t per = trees::warp_bytes(F, C);
    float *x = reinterpret_cast<float *>(trees_smem + w * per);
    int32_t *leaf = reinterpret_cast<int32_t *>(x + F);
    double *acc = reinterpret_cast<double *>(trees_smem + w * per + per - size_t(C) * sizeof(double));
    for (int64_t row = int64_t(blockIdx.x) * kTreeWarps + w; row < n; row += int64_t(gridDim.x) * kTreeWarps) {
        bool b = false;
        for (int j = lane; j < F; j += 32) x[j] = trees::cast(q[row * stride + j], allow_nan, b);
        b = __any_sync(0xffffffffu, b);
        for (int c = lane; c < C; c += 32) acc[c] = init ? init[c] : 0.0;
        __syncwarp();
        for (int t0 = 0; t0 < n_trees; t0 += 32) {
            const int nt = min(32, n_trees - t0);
            if (lane < nt) leaf[lane] = trees::walk(nodes, roots[t0 + lane], x);
            __syncwarp();
            for (int c = lane; c < C; c += 32) {
                double a = acc[c];
                for (int j = 0; j < nt; ++j) {
                    const int tc = trees::tree_class(mode, t0 + j, C);
                    if (tc < 0) a = trees::dadd(a, values[int64_t(leaf[j]) * C + c]);
                    else if (tc == c) a = trees::dadd(a, values[leaf[j]]);
                }
                acc[c] = a;
            }
            __syncwarp();
        }
        double best = 0.0, s0 = 0.0;
        int bi = -1;
        for (int c = lane; c < C; c += 32) {
            const double s = trees::finish(mode, acc[c], n_trees);
            scores[row * C + c] = s;
            if (c == 0) s0 = s;
            if (bi < 0 || trees::better(s, c, best, bi)) { best = s; bi = c; }
        }
        for (int off = 16; off > 0; off >>= 1) {
            const double ob = __shfl_down_sync(0xffffffffu, best, off);
            const int oi = __shfl_down_sync(0xffffffffu, bi, off);
            if (oi >= 0 && (bi < 0 || trees::better(ob, oi, best, bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            ids[row] = trees::class_id(mode, C, s0, bi);
            bad[row] = b ? 1 : 0;
        }
        __syncwarp();
    }
}

extern "C" int b200aa_trees_create(b200aa_trees **out, const b200aa_tree_node *h_nodes, int64_t n_nodes,
                                   const int32_t *h_roots, int n_trees, const double *h_values, int64_t n_leaves,
                                   int n_classes, int n_feats, int mode, const double *h_init, int allow_nan)
{
    if (!out) return B200AA_ERR_INVALID;
    *out = nullptr;
    if (!h_nodes || !h_roots || !h_values || n_nodes < 1 || n_nodes > INT32_MAX || n_trees < 1 || n_leaves < 1 ||
        n_leaves > INT32_MAX || n_classes < 1 || n_feats < 1 || (mode != trees::kForestMean && mode != trees::kBoostSum) ||
        (mode == trees::kBoostSum && !h_init))
        return B200AA_ERR_INVALID;
    if (h_roots[0] != 0) return B200AA_ERR_INVALID;
    // every tree a contiguous node range whose children come after their parent inside it: walks stay in the range and end
    for (int t = 0; t < n_trees; ++t) {
        const int64_t lo = h_roots[t], hi = t + 1 < n_trees ? h_roots[t + 1] : n_nodes;
        if (hi <= lo || hi > n_nodes) return B200AA_ERR_INVALID;
        for (int64_t i = lo; i < hi; ++i) {
            const b200aa_tree_node &nd = h_nodes[i];
            if (nd.left < 0) {
                if (nd.right < 0 || nd.right >= n_leaves) return B200AA_ERR_INVALID;
            } else {
                const int f = nd.feature & trees::kFeatureMask;
                if (nd.left <= i || nd.left >= hi || nd.right <= i || nd.right >= hi || f >= n_feats) return B200AA_ERR_INVALID;
            }
        }
    }
    if (trees::warp_bytes(n_feats, n_classes) * kTreeWarps > 48 * 1024) return B200AA_ERR_UNSUPPORTED;
    const size_t vals = size_t(n_leaves) * (mode == trees::kForestMean ? size_t(n_classes) : 1);
    const size_t nodes_b = align256(size_t(n_nodes) * sizeof(trees::Node)), roots_b = align256(size_t(n_trees) * sizeof(int32_t));
    const bool has_init = mode == trees::kBoostSum;         // a forest's sums start at 0: h_init is not read
    const size_t values_b = align256(vals * sizeof(double)), init_b = has_init ? size_t(n_classes) * sizeof(double) : 0;
    std::unique_ptr<b200aa_trees> m(new b200aa_trees{});
    CK(cudaGetDevice(&m->device));
    CK(cudaMalloc(&m->blob, nodes_b + roots_b + values_b + init_b));
    char *base = static_cast<char *>(m->blob);
    // The upload goes through a stream of its own and is waited for, so the model is on the device when create returns:
    // a copy from pageable memory may return before its DMA lands, and a caller's non-blocking stream is not ordered
    // after the legacy default stream.
    cudaStream_t up = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemcpyAsync(base, h_nodes, size_t(n_nodes) * sizeof(trees::Node), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(base + nodes_b, h_roots, size_t(n_trees) * sizeof(int32_t), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(base + nodes_b + roots_b, h_values, vals * sizeof(double), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess && has_init)
        e = cudaMemcpyAsync(base + nodes_b + roots_b + values_b, h_init, init_b, cudaMemcpyHostToDevice, up);
    if (up) {
        const cudaError_t es = cudaStreamSynchronize(up);
        if (e == cudaSuccess) e = es;
        cudaStreamDestroy(up);
    }
    if (e != cudaSuccess) {
        cudaFree(m->blob);
        return cuda_fail(e, "upload (tree ensemble)");
    }
    m->n_nodes = n_nodes;
    m->n_leaves = n_leaves;
    m->n_trees = n_trees;
    m->n_classes = n_classes;
    m->n_feats = n_feats;
    m->mode = mode;
    m->allow_nan = allow_nan ? 1 : 0;
    m->nodes = reinterpret_cast<const trees::Node *>(base);
    m->roots = reinterpret_cast<const int32_t *>(base + nodes_b);
    m->values = reinterpret_cast<const double *>(base + nodes_b + roots_b);
    m->init = has_init ? reinterpret_cast<const double *>(base + nodes_b + roots_b + values_b) : nullptr;
    *out = m.release();
    return B200AA_OK;
}

extern "C" int b200aa_trees_destroy(b200aa_trees *model)
{
    if (!model) return B200AA_OK;
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e == cudaSuccess && cur != model->device) e = cudaSetDevice(model->device);
    // work queued on any stream may still read the model
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaFree(model->blob);
    if (cur != model->device) cudaSetDevice(cur);
    delete model;
    return e == cudaSuccess ? B200AA_OK : cuda_fail(e, "cudaFree (tree ensemble)");
}

extern "C" int b200aa_trees_classify(const b200aa_trees *model, const void *d_query, int dtype, int64_t n_query,
                                     int n_feats, int64_t q_stride, int64_t *d_ids, double *d_scores, int32_t *d_bad,
                                     void *stream)
{
    NvtxRange nvtx_("b200aa_trees_classify");
    if (!model || !d_query || !d_ids || !d_scores || !d_bad || n_query < 0 || n_feats != model->n_feats ||
        q_stride < n_feats || (dtype != B200AA_DTYPE_F32 && dtype != B200AA_DTYPE_F64))
        return B200AA_ERR_INVALID;
    if (n_query == 0) return B200AA_OK;
    int cur = 0;
    CK(cudaGetDevice(&cur));
    if (cur != model->device) return B200AA_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = trees::warp_bytes(model->n_feats, model->n_classes) * kTreeWarps;
    const unsigned blocks = unsigned(std::min<int64_t>((n_query + kTreeWarps - 1) / kTreeWarps, INT32_MAX));
    if (dtype == B200AA_DTYPE_F32)
        trees_kernel<<<blocks, kTreeWarps * 32, smem, st>>>(model->nodes, model->roots, model->n_trees, model->values,
                                                            model->init, model->mode, model->n_classes, model->n_feats,
                                                            model->allow_nan != 0, static_cast<const float *>(d_query),
                                                            n_query, q_stride, d_ids, d_scores, d_bad);
    else
        trees_kernel<<<blocks, kTreeWarps * 32, smem, st>>>(model->nodes, model->roots, model->n_trees, model->values,
                                                            model->init, model->mode, model->n_classes, model->n_feats,
                                                            model->allow_nan != 0, static_cast<const double *>(d_query),
                                                            n_query, q_stride, d_ids, d_scores, d_bad);
    CK_LAUNCH("trees_kernel");
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
    p.scratch_stride = (bytes + 255) & ~size_t(255);
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
