// TEST INFRASTRUCTURE.  A small CPU emulation of the CUDA execution model, just big enough to run edyn_b200/csrc/*.cu
// unmodified in logic on a machine without a GPU (tests/emu/build.py rewrites the launch syntax and the seven inline-PTX
// lines, nothing else).  One OS thread; the threads of a block are ucontext fibers scheduled round-robin:
//   * __syncthreads: a fiber parks until every live fiber of the block has arrived;
//   * warp collectives (*_sync): a lane parks until every live lane named in the mask has arrived at the same operation;
//   * __activemask() answers "this lane alone" -- the kernels use it only to aggregate atomics, where any grouping is valid;
//   * blocks of an ordinary launch run one after the other (they never wait for each other); the three cooperative,
//     persistent kernels are launched with ONE block (they are grid-stride, so that is a legal grid), which turns the grid
//     barrier into a block barrier and keeps the ticket dataflow inside one scheduler; every poll yields;
//   * streams are synchronous, graphs are "not supported" (the library then launches plainly), cub is two std algorithms.
// It says nothing about memory ordering, occupancy or speed.  It executes the same C++ the GPU executes, on the same data
// layout, through the same C ABI -- so logic errors show up here, hardware-level ones do not.
#pragma once
#include <ucontext.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define EMU_NOINLINE __attribute__((noinline))      // build.py rewrites __noinline__ (libstdc++ uses that token inside its own attributes)
#define __launch_bounds__(...)
#define __shared__ static
#define __constant__ static const
#define __restrict__

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {} };
struct alignas(8) float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float3 make_float3(float x, float y, float z) { return {x, y, z}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
inline uint2 make_uint2(unsigned x, unsigned y) { return {x, y}; }
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return {x, y, z, w}; }

// ------------------------------------------------------------------------------------------------ fibers
namespace emu {
enum wait_kind { W_NONE, W_BARRIER, W_WARP };
enum op_kind { OP_SHFL, OP_BALLOT, OP_ANY, OP_ALL, OP_MATCH32, OP_MATCH64, OP_RMAX, OP_RMIN, OP_SYNC };
struct Fiber {
    ucontext_t ctx;
    uint3 tid;
    bool done = false;
    wait_kind wait = W_NONE;
    // pending warp collective
    bool pending = false, resolved = false;
    op_kind op; unsigned mask; unsigned long long val; int arg; unsigned long long result;
};
struct Block {
    std::vector<Fiber> fibers;
    uint3 bid; dim3 bdim, gdim;
    ucontext_t sched;
    void *dyn_smem = nullptr;
};
extern Block *g_block;
extern Fiber *g_cur;
inline void yield() { swapcontext(&g_cur->ctx, &g_block->sched); }
inline void *dynamic_smem() { return g_block->dyn_smem; }
void run_grid(dim3 grid, dim3 block, size_t smem, void (*entry)(void *), void *closure);
unsigned long long collective(op_kind op, unsigned mask, unsigned long long val, int arg);

template<typename K, typename... A>
void launch(K kernel, dim3 grid, dim3 block, size_t smem, A... args) {
    auto body = [&]() { kernel(args...); };
    using B = decltype(body);
    run_grid(grid, block, smem, [](void *p) { (*static_cast<B *>(p))(); }, &body);
}
}  // namespace emu

#define threadIdx (emu::g_cur->tid)
#define blockIdx (emu::g_block->bid)
#define blockDim (emu::g_block->bdim)
#define gridDim (emu::g_block->gdim)
#define EMU_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch(kernel, dim3(grid), dim3(block), size_t(smem), ##__VA_ARGS__)

inline void __syncthreads() { emu::g_cur->wait = emu::W_BARRIER; emu::yield(); }
inline void __threadfence() {}
inline void __nanosleep(unsigned) { emu::yield(); }
inline unsigned __activemask() { return 1u << (threadIdx.x & 31u); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::collective(emu::OP_SYNC, mask, 0, 0); }

// ---- warp collectives
template<typename T> inline T emu_bits_to(unsigned long long v) { T t; std::memcpy(&t, &v, sizeof(T)); return t; }
template<typename T> inline unsigned long long emu_bits_of(T t) { unsigned long long v = 0; std::memcpy(&v, &t, sizeof(T)); return v; }
// arg encodes the source: 0x000 | lane (idx), 0x100 | delta (up), 0x200 | delta (down), 0x300 | lanemask (xor)
template<typename T> inline T __shfl_sync(unsigned m, T v, int src) { return emu_bits_to<T>(emu::collective(emu::OP_SHFL, m, emu_bits_of(v), 0x000 | (src & 31))); }
template<typename T> inline T __shfl_up_sync(unsigned m, T v, unsigned d) { return emu_bits_to<T>(emu::collective(emu::OP_SHFL, m, emu_bits_of(v), 0x100 | int(d))); }
template<typename T> inline T __shfl_down_sync(unsigned m, T v, unsigned d) { return emu_bits_to<T>(emu::collective(emu::OP_SHFL, m, emu_bits_of(v), 0x200 | int(d))); }
template<typename T> inline T __shfl_xor_sync(unsigned m, T v, int x) { return emu_bits_to<T>(emu::collective(emu::OP_SHFL, m, emu_bits_of(v), 0x300 | (x & 31))); }
inline unsigned __ballot_sync(unsigned m, int p) { return unsigned(emu::collective(emu::OP_BALLOT, m, p ? 1 : 0, 0)); }
inline int __any_sync(unsigned m, int p) { return int(emu::collective(emu::OP_ANY, m, p ? 1 : 0, 0)); }
inline int __all_sync(unsigned m, int p) { return int(emu::collective(emu::OP_ALL, m, p ? 1 : 0, 0)); }
inline unsigned __match_any_sync(unsigned m, unsigned v) { return unsigned(emu::collective(emu::OP_MATCH32, m, v, 0)); }
inline unsigned __match_any_sync(unsigned m, unsigned long long v) { return unsigned(emu::collective(emu::OP_MATCH64, m, v, 0)); }
inline unsigned __reduce_max_sync(unsigned m, unsigned v) { return unsigned(emu::collective(emu::OP_RMAX, m, v, 0)); }
inline unsigned __reduce_min_sync(unsigned m, unsigned v) { return unsigned(emu::collective(emu::OP_RMIN, m, v, 0)); }
// the int overloads compare signed (k_cell_extent reduces cell coordinates): flipping the sign bit maps int order onto unsigned order
inline int __reduce_max_sync(unsigned m, int v) { return int(__reduce_max_sync(m, unsigned(v) ^ 0x80000000u) ^ 0x80000000u); }
inline int __reduce_min_sync(unsigned m, int v) { return int(__reduce_min_sync(m, unsigned(v) ^ 0x80000000u) ^ 0x80000000u); }

// ---- scalar intrinsics
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline int __float_as_int(float f) { int u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline float __int_as_float(int u) { float f; std::memcpy(&f, &u, 4); return f; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __ffsll(long long v) { return __builtin_ffsll(v); }
inline int __clz(int v) { return v ? __builtin_clz(unsigned(v)) : 32; }
template<typename T> inline T __ldcg(const T *p) { return *p; }
template<typename T> inline T __ldcs(const T *p) { return *p; }
template<typename T> inline T __ldg(const T *p) { return *p; }

// ---- atomics (one OS thread: plain read-modify-write)
template<typename T, typename V> inline T atomicAdd(T *p, V v) { T o = *p; *p = T(o + T(v)); return o; }
template<typename T, typename V> inline T atomicSub(T *p, V v) { T o = *p; *p = T(o - T(v)); return o; }
template<typename T, typename V> inline T atomicOr(T *p, V v) { T o = *p; *p = T(o | T(v)); return o; }
template<typename T, typename V> inline T atomicAnd(T *p, V v) { T o = *p; *p = T(o & T(v)); return o; }
template<typename T, typename V> inline T atomicMax(T *p, V v) { T o = *p; if (T(v) > o) *p = T(v); return o; }
template<typename T, typename V> inline T atomicMin(T *p, V v) { T o = *p; if (T(v) < o) *p = T(v); return o; }
template<typename T, typename V> inline T atomicExch(T *p, V v) { T o = *p; *p = T(v); return o; }
template<typename T, typename C, typename V> inline T atomicCAS(T *p, C c, V v) { T o = *p; if (o == T(c)) *p = T(v); return o; }

// ---- min / max with CUDA's mixed-type convenience
template<typename A, typename B, typename = std::enable_if_t<std::is_arithmetic_v<A> && std::is_arithmetic_v<B>>>
inline std::common_type_t<A, B> min(A a, B b) { using C = std::common_type_t<A, B>; return C(a) < C(b) ? C(a) : C(b); }
template<typename A, typename B, typename = std::enable_if_t<std::is_arithmetic_v<A> && std::is_arithmetic_v<B>>>
inline std::common_type_t<A, B> max(A a, B b) { using C = std::common_type_t<A, B>; return C(a) > C(b) ? C(a) : C(b); }
inline void sincosf_emu(float x, float *s, float *c) { *s = sinf(x); *c = cosf(x); }

// ------------------------------------------------------------------------------------------------ runtime API
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorNotSupported = 801, cudaErrorMemoryAllocation = 2, cudaErrorNotReady = 600 };
typedef struct emu_stream *cudaStream_t;
typedef struct emu_event { std::chrono::steady_clock::time_point t; } *cudaEvent_t;
typedef struct emu_graph *cudaGraph_t;
typedef struct emu_graph_exec *cudaGraphExec_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyHostToHost, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaStreamCaptureModeThreadLocal = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaGraphExecUpdateResult { cudaGraphExecUpdateSuccess = 0, cudaGraphExecUpdateError = 1 };
struct cudaGraphExecUpdateResultInfo { cudaGraphExecUpdateResult result; };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; int cooperativeLaunch; int major, minor; size_t totalGlobalMem; };

inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : (e == cudaErrorNotSupported ? "not supported by the CPU emulation" : "emulated CUDA error"); }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { std::memset(p, 0, sizeof(*p)); std::strcpy(p->name, "CPU emulation (tests/emu)"); p->multiProcessorCount = 2; p->cooperativeLaunch = 1; p->major = 9; return cudaSuccess; }
template<typename T> inline cudaError_t cudaMalloc(T **p, size_t bytes) { *p = static_cast<T *>(std::aligned_alloc(256, (bytes + 255) / 256 * 256 + 256)); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void *p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemset(void *d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = reinterpret_cast<cudaStream_t>(new int(0)); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete reinterpret_cast<int *>(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new emu_event{std::chrono::steady_clock::now()}; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count(); return cudaSuccess; }
template<typename K> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, K, int, size_t) { *n = 1; return cudaSuccess; }
template<typename K> inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }
// graphs: refused, so the library falls back to plain launches
inline cudaError_t cudaStreamBeginCapture(cudaStream_t, int) { return cudaErrorNotSupported; }
inline cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t *g) { *g = nullptr; return cudaErrorNotSupported; }
inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t *, cudaGraph_t, unsigned long long = 0) { return cudaErrorNotSupported; }
inline cudaError_t cudaGraphExecUpdate(cudaGraphExec_t, cudaGraph_t, cudaGraphExecUpdateResultInfo *) { return cudaErrorNotSupported; }
inline cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
