// Minimal CUDA execution-model emulator for CPU-only kernel-logic tests.
//
// TEST INFRASTRUCTURE ONLY (think compute-sanitizer, not a backend): tests/emul/build.py compiles
// the library's .cu sources with g++ against this header into tests/emul/_build/libdplonk_emul.so
// so that indexing, shared-memory exchange, barriers and the host-side task logic can be debugged
// on a box without a GPU.  The shipped library (distributed_plonk_b200/_build/libdplonk.so) is
// nvcc-only, never includes this file, and the Python package refuses to load anything else.
//
// Model: one CUDA block at a time; blockDim threads are real std::threads; __syncthreads is a
// std::barrier; `__shared__` is plain `static` storage (one block alive at a time); dynamic shared
// memory is a per-launch heap buffer; "device" memory is host memory.
#pragma once
#include <atomic>
#include <barrier>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <thread>
#include <vector>

#define DP_EMUL_ACTIVE 1

struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint4 { uint32_t x, y, z, w; };
struct alignas(8) uint2 { uint32_t x, y; };
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

namespace dp_emul {
inline thread_local dim3 t_threadIdx, t_blockIdx, t_blockDim, t_gridDim;
inline thread_local std::barrier<> *t_block_barrier = nullptr;
inline thread_local unsigned char *t_dyn_smem = nullptr;
struct WarpXchg {
    std::barrier<> bar;
    uint64_t slot[32];
    unsigned char blob[32][256];  // whole-struct exchange (one barrier pair per struct, not per word)
    explicit WarpXchg(int n) : bar(n) {}
};
inline thread_local WarpXchg *t_warp = nullptr;
inline thread_local unsigned t_lane = 0;

inline void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()> &body) {
    const unsigned nthreads = block.x * block.y * block.z;
    const unsigned nwarps = (nthreads + 31) / 32;
    std::barrier<> bar(nthreads);
    std::vector<std::unique_ptr<WarpXchg>> warps;
    for (unsigned w = 0; w < nwarps; w++) {
        unsigned n = (w + 1) * 32 <= nthreads ? 32 : nthreads - w * 32;
        warps.emplace_back(new WarpXchg((int)n));
    }
    std::vector<unsigned char> dyn(smem + 64);
    unsigned char *dyn_aligned = (unsigned char *)(((uintptr_t)dyn.data() + 63) & ~(uintptr_t)63);
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < nthreads; t++) {
        pool.emplace_back([&, t] {
            t_blockDim = block;
            t_gridDim = grid;
            t_threadIdx = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
            t_block_barrier = &bar;
            t_dyn_smem = dyn_aligned;
            t_warp = warps[t / 32].get();
            t_lane = t % 32;
            for (unsigned bz = 0; bz < grid.z; bz++)
                for (unsigned by = 0; by < grid.y; by++)
                    for (unsigned bx = 0; bx < grid.x; bx++) {
                        t_blockIdx = dim3(bx, by, bz);
                        body();
                        bar.arrive_and_wait();  // next block reuses the static __shared__ storage
                    }
        });
    }
    for (auto &th : pool) th.join();
}
}  // namespace dp_emul

#define threadIdx (dp_emul::t_threadIdx)
#define blockIdx (dp_emul::t_blockIdx)
#define blockDim (dp_emul::t_blockDim)
#define gridDim (dp_emul::t_gridDim)
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __shared__ static
#define __constant__ static
#define __restrict__
#define __launch_bounds__(...)
#define __align__(n) alignas(n)

inline void __syncthreads() { dp_emul::t_block_barrier->arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { dp_emul::t_warp->bar.arrive_and_wait(); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __threadfence_block() { std::atomic_thread_fence(std::memory_order_seq_cst); }

template <class T>
inline T dp_emul_shfl(T v, unsigned src_lane) {
    static_assert(sizeof(T) <= 8, "shuffle payload");
    auto *w = dp_emul::t_warp;
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    w->slot[dp_emul::t_lane] = raw;
    w->bar.arrive_and_wait();
    uint64_t got = w->slot[src_lane & 31];
    w->bar.arrive_and_wait();
    T out;
    memcpy(&out, &got, sizeof(T));
    return out;
}
// struct-granular shuffle used by kernels under DP_EMUL to keep barrier counts (thread switches) low
template <class T>
inline T dp_emul_shfl_struct(const T &v, unsigned src_lane) {
    static_assert(sizeof(T) <= 256, "shuffle blob");
    auto *w = dp_emul::t_warp;
    memcpy(w->blob[dp_emul::t_lane], &v, sizeof(T));
    w->bar.arrive_and_wait();
    T out;
    memcpy(&out, w->blob[src_lane & 31], sizeof(T));
    w->bar.arrive_and_wait();
    return out;
}
template <class T> inline T __shfl_sync(unsigned, T v, int src) { return dp_emul_shfl(v, (unsigned)src); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) { return dp_emul_shfl(v, dp_emul::t_lane ^ (unsigned)m); }
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d) {
    unsigned s = dp_emul::t_lane + d;
    return dp_emul_shfl(v, s < 32 ? s : dp_emul::t_lane);
}
inline unsigned __ballot_sync(unsigned, int pred) {
    unsigned bit = pred ? (1u << dp_emul::t_lane) : 0u, acc = 0;
    for (int l = 0; l < 32; l++) acc |= dp_emul_shfl(bit, (unsigned)l);
    return acc;
}
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __clz(int v) { return v == 0 ? 32 : __builtin_clz((unsigned)v); }
inline unsigned __brev(unsigned v) {
    unsigned r = 0;
    for (int i = 0; i < 32; i++) r |= ((v >> i) & 1u) << (31 - i);
    return r;
}
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) {
    sh &= 31;
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
}

inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline int atomicAdd(int *p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) {
    return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST);
}
inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
inline unsigned atomicMax(unsigned *p, unsigned v) {
    unsigned old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
inline unsigned long long atomicMin(unsigned long long *p, unsigned long long v) {
    unsigned long long old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old > v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
template <class T> inline T __ldg(const T *p) { return *p; }

// ------------------------------------------------------------------ runtime API subset
typedef int cudaError_t;
typedef struct dp_emul_stream *cudaStream_t;
typedef struct dp_emul_event *cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { int multiProcessorCount; size_t totalGlobalMem; char name[256]; int major, minor; };

#if defined(DP_EMUL_ASYNC)
// ---- asynchronous streams (tests/emul/build.py --async): every stream is a worker thread with a FIFO
// of closures, events carry record / completion generations, kernels of all streams run one at a time
// (static __shared__ storage) but in whatever order the streams' dependencies allow, with a random delay
// before every operation.  A missing cudaStreamWaitEvent / synchronize in the library shows up as a wrong
// result here instead of only under unlucky timing on a GPU.  Pageable-memory semantics: the source of a
// host-to-device copy is captured when the copy is issued; device-to-host copies land when the stream
// gets there.
#include <condition_variable>
#include <deque>
#include <mutex>
#include <random>
#include <set>
namespace dp_emul {
inline std::mutex g_device;                 // one kernel at a time
inline std::mutex g_registry;
inline std::set<dp_emul_stream *> g_streams;
inline unsigned jitter_us() {
    static const unsigned v = [] {
        const char *e = getenv("DP_EMUL_JITTER_US");
        return e ? (unsigned)atoi(e) : 200u;
    }();
    return v;
}
// adversarial schedule: DP_EMUL_SLOW="i:us" delays every operation of the streams whose creation index is
// i mod 5 by `us` microseconds (a context creates compute, copy-in, copy-out, tail, sort in that order), so an
// operation that should have waited for that stream and does not is practically certain to run too early
inline std::atomic<unsigned> g_stream_counter{0};
inline unsigned slow_us(unsigned index) {
    static const std::pair<int, unsigned> cfg = [] {
        const char *e = getenv("DP_EMUL_SLOW");
        int i = -1;
        unsigned us = 0;
        if (e && sscanf(e, "%d:%u", &i, &us) != 2) i = -1;
        return std::make_pair(i, us);
    }();
    return cfg.first >= 0 && (int)(index % 5) == cfg.first ? cfg.second : 0u;
}
}  // namespace dp_emul
struct dp_emul_stream {
    std::mutex m;
    std::condition_variable cv;
    std::deque<std::function<void()>> q;
    uint64_t enq = 0, done = 0;
    bool stop = false;
    unsigned index = dp_emul::g_stream_counter++;
    std::thread worker;
    dp_emul_stream() : worker([this] { run(); }) {}
    void run() {
        std::minstd_rand rng((unsigned)(uintptr_t)this);
        for (;;) {
            std::function<void()> f;
            {
                std::unique_lock<std::mutex> l(m);
                cv.wait(l, [&] { return stop || !q.empty(); });
                if (q.empty()) return;
                f = std::move(q.front());
                q.pop_front();
            }
            if (dp_emul::jitter_us()) std::this_thread::sleep_for(std::chrono::microseconds(rng() % dp_emul::jitter_us()));
            if (dp_emul::slow_us(index)) std::this_thread::sleep_for(std::chrono::microseconds(dp_emul::slow_us(index)));
            f();
            {
                std::lock_guard<std::mutex> l(m);
                done++;
            }
            cv.notify_all();
        }
    }
    void push(std::function<void()> f) {
        {
            std::lock_guard<std::mutex> l(m);
            q.push_back(std::move(f));
            enq++;
        }
        cv.notify_all();
    }
    void sync() {
        std::unique_lock<std::mutex> l(m);
        cv.wait(l, [&] { return done == enq; });
    }
    ~dp_emul_stream() {
        {
            std::lock_guard<std::mutex> l(m);
            stop = true;
        }
        cv.notify_all();
        worker.join();
    }
};
struct dp_emul_event_state {
    std::mutex m;
    std::condition_variable cv;
    uint64_t recorded = 0, completed = 0;
    std::chrono::steady_clock::time_point t;
};
struct dp_emul_event { std::shared_ptr<dp_emul_event_state> st = std::make_shared<dp_emul_event_state>(); };
namespace dp_emul {
inline void run_on(cudaStream_t s, std::function<void()> f) {
    if (s) s->push(std::move(f));
    else f();
}
inline void sync_all() {
    std::vector<dp_emul_stream *> all;
    {
        std::lock_guard<std::mutex> l(g_registry);
        all.assign(g_streams.begin(), g_streams.end());
    }
    for (dp_emul_stream *s : all) s->sync();
}
inline void launch_on(cudaStream_t s, dim3 grid, dim3 block, size_t smem, std::function<void()> body) {
    run_on(s, [=] {
        std::lock_guard<std::mutex> g(g_device);
        launch(grid, block, smem, body);
    });
}
}  // namespace dp_emul
#else
struct dp_emul_event { std::chrono::steady_clock::time_point t; };
namespace dp_emul {
inline void launch_on(cudaStream_t, dim3 grid, dim3 block, size_t smem, const std::function<void()> &body) { launch(grid, block, smem, body); }
}  // namespace dp_emul
#endif

inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 8; return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    memset(p, 0, sizeof *p);
    p->multiProcessorCount = 4;
    p->totalGlobalMem = (size_t)8 << 30;
    snprintf(p->name, sizeof p->name, "cpu-emulator");
    p->major = 9;
    p->minor = 0;
    return cudaSuccess;
}
inline cudaError_t cudaMalloc(void **p, size_t n) {
    *p = aligned_alloc(256, (n + 255) & ~(size_t)255);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
template <class T> inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
#if defined(DP_EMUL_ASYNC)
inline cudaError_t cudaFree(void *p) { dp_emul::sync_all(); free(p); return cudaSuccess; }  // cudaFree synchronises the device
#else
inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
#endif
inline cudaError_t cudaMallocHost(void **p, size_t n) { return cudaMalloc(p, n); }
template <class T> inline cudaError_t cudaMallocHost(T **p, size_t n) { return cudaMalloc((void **)p, n); }
inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new dp_emul_event; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = new dp_emul_event; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }  // queued closures hold the shared state
#if defined(DP_EMUL_ASYNC)
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind kind, cudaStream_t st = nullptr) {
    if (kind == cudaMemcpyHostToDevice && st) {  // pageable source: staged when the copy is issued
        auto buf = std::make_shared<std::vector<unsigned char>>((const unsigned char *)s, (const unsigned char *)s + n);
        st->push([=] { memcpy(d, buf->data(), n); });
    } else {
        dp_emul::run_on(st, [=] { memmove(d, s, n); });
    }
    return cudaSuccess;
}
inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h,
                                     cudaMemcpyKind kind, cudaStream_t st = nullptr) {
    if (kind == cudaMemcpyHostToDevice && st) {  // pageable source: staged when the copy is issued
        auto buf = std::make_shared<std::vector<unsigned char>>(w * h);
        for (size_t i = 0; i < h; i++) memcpy(buf->data() + i * w, (const char *)s + i * sp, w);
        st->push([=] {
            for (size_t i = 0; i < h; i++) memcpy((char *)d + i * dp, buf->data() + i * w, w);
        });
        return cudaSuccess;
    }
    dp_emul::run_on(st, [=] {
        for (size_t i = 0; i < h; i++) memmove((char *)d + i * dp, (const char *)s + i * sp, w);
    });
    return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st = nullptr) {
    dp_emul::run_on(st, [=] { memset(d, v, n); });
    return cudaSuccess;
}
inline cudaError_t cudaMemset2DAsync(void *d, size_t pitch, int v, size_t w, size_t h, cudaStream_t st = nullptr) {
    dp_emul::run_on(st, [=] {
        for (size_t i = 0; i < h; i++) memset((char *)d + i * pitch, v, w);
    });
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) {
    *s = new dp_emul_stream;
    std::lock_guard<std::mutex> l(dp_emul::g_registry);
    dp_emul::g_streams.insert(*s);
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreate(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, 0); }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) {
    if (!s) return cudaSuccess;
    s->sync();
    {
        std::lock_guard<std::mutex> l(dp_emul::g_registry);
        dp_emul::g_streams.erase(s);
    }
    delete s;
    return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t s) {
    if (s) s->sync();
    return cudaSuccess;
}
inline cudaError_t cudaDeviceSynchronize() { dp_emul::sync_all(); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr) {
    auto st = e->st;
    uint64_t gen;
    {
        std::lock_guard<std::mutex> l(st->m);
        gen = ++st->recorded;
    }
    dp_emul::run_on(s, [st, gen] {
        {
            std::lock_guard<std::mutex> l(st->m);
            if (st->completed < gen) st->completed = gen;
            st->t = std::chrono::steady_clock::now();
        }
        st->cv.notify_all();
    });
    return cudaSuccess;
}
inline cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned = 0) {
    auto st = e->st;
    uint64_t gen;
    {
        std::lock_guard<std::mutex> l(st->m);
        gen = st->recorded;  // the most recent record at the time of the call; never recorded: no-op
    }
    dp_emul::run_on(s, [st, gen] {
        std::unique_lock<std::mutex> l(st->m);
        st->cv.wait(l, [&] { return st->completed >= gen; });
    });
    return cudaSuccess;
}
inline cudaError_t cudaEventSynchronize(cudaEvent_t e) {
    auto st = e->st;
    std::unique_lock<std::mutex> l(st->m);
    st->cv.wait(l, [&] { return st->completed >= st->recorded; });
    return cudaSuccess;
}
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->st->t - a->st->t).count();
    return cudaSuccess;
}
#else
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) {
    memmove(d, s, n);
    return cudaSuccess;
}
inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h,
                                     cudaMemcpyKind, cudaStream_t = nullptr) {
    for (size_t i = 0; i < h; i++) memmove((char *)d + i * dp, (const char *)s + i * sp, w);
    return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemset2DAsync(void *d, size_t pitch, int v, size_t w, size_t h, cudaStream_t = nullptr) {
    for (size_t i = 0; i < h; i++) memset((char *)d + i * pitch, v, w);
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) {
    e->t = std::chrono::steady_clock::now();
    return cudaSuccess;
}
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
    return cudaSuccess;
}
#endif
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated error"; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
// CUDA IPC: all emulated "devices" live in this process, so a handle is just the pointer
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) {
    memset(h, 0, sizeof *h);
    memcpy(h->reserved, &p, sizeof p);
    return cudaSuccess;
}
inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) {
    memcpy(p, h.reserved, sizeof *p);
    return cudaSuccess;
}
inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
inline cudaError_t cudaMemGetInfo(size_t *f, size_t *t) { *f = *t = (size_t)8 << 30; return cudaSuccess; }
