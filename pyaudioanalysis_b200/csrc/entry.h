// Host-side plumbing of every C ABI entry point of libb200aa.so: CUDA error reporting and the launch count, the capture
// guard, stream-ordered scratch, NVTX ranges, scratch alignment and slicing, and the float32 / float64 dispatch of a launch.
// g_cuda_err and g_launches are defined once, in b200aa.cu, so that b200aa_last_cuda_error() and b200aa_launch_count()
// see every file's entry points.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>      // header-only NVTX 3: ranges around the entry points (visible in nsys / ncu timelines)

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>

#include "../../include/b200aa.h"

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
extern thread_local std::string g_cuda_err;
extern std::atomic<int64_t> g_launches;

inline int cuda_fail(cudaError_t e, const char *what)
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
inline int launched(const char *name)
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

// ------------------------------------------------------------------------------------------------
// CUDA graph capture (include/b200aa.h)
// ------------------------------------------------------------------------------------------------
// True when `st` is capturing a graph, or is the legacy default stream while a blocking stream captures (any use of it
// would invalidate that capture).  The query is legal in every capture mode.  A query that fails otherwise (no device, a
// bad stream) answers false and clears its error, so the call goes on to meet that error where it met it before.
inline bool stream_capturing(cudaStream_t st)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(st, &cs);
    if (e != cudaSuccess) cudaGetLastError();
    return e == cudaErrorStreamCaptureImplicit || (e == cudaSuccess && cs != cudaStreamCaptureStatusNone);
}

// The guard of an entry point that cannot be captured: B200AA_ERR_CAPTURE, with "entry: why" as the thread's error text,
// when `st` is capturing, before any other CUDA call
inline int refuse_capture(cudaStream_t st, const char *entry, const char *why)
{
    if (!stream_capturing(st)) return B200AA_OK;
    g_cuda_err = std::string(entry) + ": " + why;
    return B200AA_ERR_CAPTURE;
}
#define REFUSE_CAPTURE(stream, entry, why)                                                   \
    do {                                                                                     \
        const int rc_ = refuse_capture(static_cast<cudaStream_t>(stream), entry, why);      \
        if (rc_ != B200AA_OK) return rc_;                                                    \
    } while (0)
// reasons of the refusals
constexpr const char *kWhyHostArrays = "copies host arrays to the device, which a graph would read after they are freed; "
                                       "call it eagerly";
constexpr const char *kWhyHostBuffer = "host-buffer entry points allocate, copy and synchronise; call them eagerly";
constexpr const char *kWhyAllocates = "allocates and uploads device tables; make this call outside capture first";

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

// ------------------------------------------------------------------------------------------------
// scratch layout and dispatch
// ------------------------------------------------------------------------------------------------
// Bound on one slice of an entry point's stream-ordered scratch: work larger than this is cut into slices run in turn.
constexpr size_t kScratchSliceBytes = size_t(256) << 20;

inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// The regions of one block of scratch, in order from offset `at`, each padded to a multiple of 256 bytes: add() returns a
// region's byte offset, bytes() the end of the last.  One layout places both the host image of a head and the device block
// it is uploaded to, so the two cannot disagree.
class Layout {
  public:
    explicit Layout(size_t at = 0) : end_(at) {}
    size_t add(size_t bytes)
    {
        const size_t at = end_;
        end_ += align256(bytes);
        return at;
    }
    size_t bytes() const { return end_; }
    template <class T>
    static T *at(void *base, size_t offset)
    {
        return reinterpret_cast<T *>(static_cast<char *>(base) + offset);
    }

  private:
    size_t end_;
};

// f(float{}) for B200AA_DTYPE_F32, f(double{}) for B200AA_DTYPE_F64 (the caller has checked dtype): a launch over either
// element type written once
template <class F>
auto with_real_type(int dtype, F f)
{
    return dtype == B200AA_DTYPE_F32 ? f(float{}) : f(double{});
}

// ------------------------------------------------------------------------------------------------
// a plan as the float64 path (f64.cu) sees it
// ------------------------------------------------------------------------------------------------
struct F64Tables;                               // the plan's float64 device tables (f64.cu)
struct PlanF64 {
    int fs, window, step, K, sm_count, tables_status;
    const F64Tables *tables;                    // set by plan_f64_tables
};
// the plan's shape (b200aa.cu)
int plan_f64(const b200aa_plan *plan, PlanF64 &out);
// B200AA_OK when the current device is the plan's (b200aa.cu)
int plan_f64_device(const b200aa_plan *plan);
// the same after the device check, with the float64 tables, built on the plan's first float64 call (b200aa.cu); that
// build cannot be captured: B200AA_ERR_CAPTURE (as `entry`) when st is capturing and the tables are not built yet
int plan_f64_tables(const b200aa_plan *plan, PlanF64 &out, cudaStream_t st, const char *entry);
// builds them (f64.cu); tables_status: the plan's, the feature tables are only built when it is B200AA_OK
int f64_tables_build(int fs, int window, int tables_status, std::shared_ptr<const F64Tables> &out);
