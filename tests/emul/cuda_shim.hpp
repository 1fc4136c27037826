// cuda_shim.hpp -- TEST INFRASTRUCTURE ONLY.  A small CUDA-on-CPU emulation that lets the HOST PIPELINE of libbdepth
// (sambamba_b200/csrc/bdepth.cu) and its kernels (kernels.cuh, mates.cuh, filter.cuh, inflate_core.cuh) be compiled with
// g++ (-DBDEPTH_EMULATE) into tests/emul/libbdepth_emul.so, so that launch plumbing written without access to a GPU can
// be exercised on the CPU against the oracle.  It is never part of the product: libbdepth.so is built by nvcc from the
// same sources without this file, and the product path still fails with BDEPTH_ERR_CUDA when there is no device.
//
//   * device memory = host memory; streams are synchronous (every operation completes before the call returns, which
//     satisfies any stream / event ordering); events carry wall-clock stamps;
//   * a kernel launch runs the grid block after block; the threads of a block are ucontext fibers on one OS thread,
//     scheduled round-robin; warp collectives (__ballot_sync, __shfl_*, __reduce_*, __all_sync) and __syncthreads are
//     rendezvous points between fibers, so kernels written for lock-step warps run unchanged;
//   * __shared__ is a static (one block runs at a time), dynamic shared memory is a per-launch buffer;
//   * atomics are plain read-modify-writes (one fiber runs at a time).
// What it cannot show: memory-model races, alignment faults, cp.async / inline PTX paths (K1 takes its host branch),
// performance.  Those stay with the GPU tests.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <functional>
#include <vector>

// ------------------------------------------------------------------------------------------------ language
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define BD_NOINLINE __attribute__((noinline))
#define __launch_bounds__(...)
#define __restrict__
#define __shared__ static thread_local      // (ranks are threads of one process under the emulation: every rank thread runs its own blocks)
#define BD_HD inline
#define BD_HD_COLD inline

struct uint3_ { unsigned x, y, z; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }

namespace emu {
struct Warp { uint32_t arrived = 0, departed = 0, exited = 0; uint64_t slot[32]; };
struct Fiber { ucontext_t ctx; char* stack = nullptr; bool done = false; unsigned tid = 0; };
struct BlockCtx {
    dim3 grid, block; unsigned bx = 0; std::vector<Warp> warps; std::vector<Fiber> fibers; ucontext_t sched; unsigned cur = 0;
    unsigned sync_arrived = 0, sync_gen = 0, alive = 0; void* dyn = nullptr; std::function<void()> body;
};
extern thread_local BlockCtx* g_blk;
void yield();
uint64_t collective(unsigned mask, uint64_t v, int op, int arg);   // op: 0 ballot, 1 shfl idx, 2 shfl xor, 3 shfl up, 4 or, 5 min, 6 all
void syncthreads();
void run_grid(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);
template <class F> struct Bound {
    dim3 g, b; size_t s; F f;
    template <class... A> void operator()(A... a) { run_grid(g, b, s, [&] { f(a...); }); }
};
template <class F> Bound<F> bind(dim3 g, dim3 b, size_t s, void*, F f) { return Bound<F>{g, b, s, f}; }
struct Idx { unsigned x, y, z; };
}  // namespace emu
#define threadIdx (emu::Idx{emu::g_blk->fibers[emu::g_blk->cur].tid, 0u, 0u})
#define blockIdx (emu::Idx{emu::g_blk->bx, 0u, 0u})
#define blockDim (emu::g_blk->block)
#define gridDim (emu::g_blk->grid)
#define BD_LAUNCH(g, b, s, st, ...) emu::bind(dim3((unsigned)(g)), dim3((unsigned)(b)), (size_t)(s), (void*)(st), __VA_ARGS__)
#define BD_DYN_SMEM(T, name) T* name = (T*)emu::g_blk->dyn

// ------------------------------------------------------------------------------------------------ device intrinsics
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (s & 31)); }
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline uint32_t __brev(uint32_t x) { x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1); x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2); x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4); x = ((x >> 8) & 0x00FF00FFu) | ((x & 0x00FF00FFu) << 8); return (x >> 16) | (x << 16); }
static inline float __uint_as_float(uint32_t b) { float f; memcpy(&f, &b, 4); return f; }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)(uintptr_t)p; }
static inline void __syncthreads() { emu::syncthreads(); }
static inline void __syncwarp(unsigned m = 0xFFFFFFFFu) { (void)emu::collective(m, 0, 0, 0); }
static inline unsigned __ballot_sync(unsigned m, int p) { return (unsigned)emu::collective(m, p ? 1 : 0, 0, 0); }
static inline int __all_sync(unsigned m, int p) { return (int)emu::collective(m, p ? 1 : 0, 6, 0); }
static inline uint32_t __reduce_or_sync(unsigned m, uint32_t v) { return (uint32_t)emu::collective(m, v, 4, 0); }
static inline uint32_t __reduce_min_sync(unsigned m, uint32_t v) { return (uint32_t)emu::collective(m, v, 5, 0); }
template <class T> static inline T __shfl_sync(unsigned m, T v, int lane) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); b = emu::collective(m, b, 1, lane); T r; memcpy(&r, &b, sizeof(T)); return r; }
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int x) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); b = emu::collective(m, b, 2, x); T r; memcpy(&r, &b, sizeof(T)); return r; }
template <class T> static inline T __shfl_up_sync(unsigned m, T v, unsigned d) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); b = emu::collective(m, b, 3, (int)d); T r; memcpy(&r, &b, sizeof(T)); return r; }
template <class T, class U> static inline T atomicAdd(T* p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicMin(T* p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMax(T* p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicOr(T* p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicExch(T* p, U v) { T o = *p; *p = (T)v; return o; }
using std::max; using std::min;
static inline int max(int a, int b) { return a > b ? a : b; }
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }

// ------------------------------------------------------------------------------------------------ runtime
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
typedef struct emu_stream* cudaStream_t;
struct emu_event { double t = 0; };
typedef emu_event* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocMapped = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9, cudaSharedmemCarveoutMaxShared = 100 };
static inline const char* cudaGetErrorString(cudaError_t e) { return e ? "emulated CUDA error" : "no error"; }
static inline const char* cudaGetErrorName(cudaError_t e) { return e ? "cudaErrorEmulated" : "cudaSuccess"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 8; return cudaSuccess; }       // eight pretend devices: ranks are threads (NCCL stand-in below)
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaMemGetInfo(size_t* f, size_t* t) { *f = (size_t)32 << 30; *t = (size_t)64 << 30; return cudaSuccess; }
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = calloc(n + 512, 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }       // + slack: device buffers are readable a little past their end (kernels.cuh ldu32)
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = calloc(n + 64, 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMallocHost(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaHostGetDevicePointer(void** d, void* h, unsigned) { *d = h; return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t) { return cudaMemcpy(d, s, n, k); }
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t) { for (size_t i = 0; i < h; i++) memmove((char*)d + i * dp, (const char*)s + i * sp, w); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { return cudaMemset(d, v, n); }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)calloc(1, 8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emu_event(); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
enum { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 132; return cudaSuccess; }      // an H100 SXM's SM count

// ------------------------------------------------------------------------------------------------ NCCL stand-in
// Ranks are THREADS of one process under emulation (the tests start one thread per rank; ctypes releases the GIL).  The
// collectives the library uses (all-gather, all-reduce sum, grouped send/recv) are rendezvous between those threads,
// matched by the 128-byte unique id.  Calls are blocking, which satisfies any stream ordering.
int emu_ncclGetUniqueId(void* uid128);
int emu_ncclCommInitRank(void** comm, int world, const void* uid128, int rank);
int emu_ncclCommDestroy(void* comm);
int emu_ncclAllGather(const void* send, void* recv, size_t count, int dtype, void* comm, cudaStream_t);
int emu_ncclAllReduce(const void* send, void* recv, size_t count, int dtype, int op, void* comm, cudaStream_t);
int emu_ncclSend(const void* send, size_t count, int dtype, int peer, void* comm, cudaStream_t);
int emu_ncclRecv(void* recv, size_t count, int dtype, int peer, void* comm, cudaStream_t);
int emu_ncclGroupStart();
int emu_ncclGroupEnd();
const char* emu_ncclGetErrorString(int);
