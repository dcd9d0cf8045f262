// cuda_runtime.h -- TEST STUB (tests/emul): lets the DEVICE code of this repository
// (manatee_b200/csrc/*.cuh, untouched) be compiled by g++ and executed on the CPU under a
// SIMT emulator, so that the very source the GPU runs -- device functions AND __global__
// kernels -- can be fuzzed against the oracle on a machine without a GPU.
//   * every CUDA thread is a fiber (ucontext); fibers are switched at every *_sync intrinsic,
//     __syncthreads() and grid sync, never in between, so one legal interleaving is executed;
//   * warp intrinsics exchange through a per-warp buffer, __shared__ is one per-process
//     instance (CTAs of a launch run one after the other; a cooperative launch is emulated
//     with a single CTA), global memory is ordinary memory.
// This is test infrastructure only: nothing under tests/ is part of the product, which has no
// CPU path (mtz_open fails with MTZ_ENOGPU without an sm_90 device).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>
#include <functional>

#define MTZ_HOST_EMUL 1
#define __CUDACC__ 1
#define __device__
#define __host__
#define __global__
#define __shared__ thread_local      /* static storage shared by all fibers of the thread */
#define __forceinline__ inline
#define __launch_bounds__(...)

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r = { x, y, z, w }; return r; }
static inline uint2 make_uint2(uint32_t x, uint32_t y) { uint2 r = { x, y }; return r; }

namespace emu {
// launch `grid` CTAs of `block` threads (block % 32 == 0) one CTA after the other; the body
// is the kernel call.  cooperative = all CTAs alive at once is NOT supported: use grid = 1.
void launch(unsigned grid, unsigned block, const std::function<void()> &kernel);
void run_warp(const std::function<void(int)> &body);     // 1 CTA of 1 warp, body(lane)
void barrier_warp();
void barrier_cta();
unsigned tid();          // threadIdx.x of the running fiber
unsigned cta();          // blockIdx.x
unsigned ncta();         // gridDim.x
unsigned nthr();         // blockDim.x
uint64_t *xchg();        // the running fiber's warp exchange buffer (32 slots)
static inline int lane() { return (int)(tid() & 31u); }
unsigned long long syncs();
}

struct emu_tid_t { operator unsigned() const { return emu::tid(); } };
struct emu_cta_t { operator unsigned() const { return emu::cta(); } };
struct emu_nct_t { operator unsigned() const { return emu::ncta(); } };
struct emu_nth_t { operator unsigned() const { return emu::nthr(); } };
struct emu_threadIdx_t { emu_tid_t x; unsigned y = 0, z = 0; };
struct emu_blockIdx_t { emu_cta_t x; unsigned y = 0, z = 0; };
struct emu_gridDim_t { emu_nct_t x; unsigned y = 1, z = 1; };
struct emu_blockDim_t { emu_nth_t x; unsigned y = 1, z = 1; };
static emu_threadIdx_t threadIdx;
static emu_blockIdx_t blockIdx;
static emu_gridDim_t gridDim;
static emu_blockDim_t blockDim;

template <class T> static inline T min(T a, T b) { return a < b ? a : b; }
template <class T> static inline T max(T a, T b) { return a > b ? a : b; }

static inline void __syncwarp(unsigned = 0xffffffffu) { emu::barrier_warp(); }
static inline void __syncthreads() { emu::barrier_cta(); }

template <class T> static inline T emu_xchg(T v, int src)
{
	uint64_t raw = 0;
	memcpy(&raw, &v, sizeof(T));
	emu::xchg()[emu::lane()] = raw;
	emu::barrier_warp();
	raw = emu::xchg()[src & 31];
	emu::barrier_warp();
	T r;
	memcpy(&r, &raw, sizeof(T));
	return r;
}
template <class T> static inline T __shfl_sync(unsigned, T v, int src, int = 32) { return emu_xchg(v, src); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return emu_xchg(v, emu::lane() ^ m); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32)
{
	const int l = emu::lane();
	return emu_xchg(v, l >= (int)d ? l - (int)d : l);
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int = 32)
{
	const int l = emu::lane();
	return emu_xchg(v, l + (int)d < 32 ? l + (int)d : l);
}
static inline unsigned __ballot_sync(unsigned, int pred)
{
	emu::xchg()[emu::lane()] = pred ? 1u : 0u;
	emu::barrier_warp();
	unsigned r = 0;
	for (int i = 0; i < 32; i++) r |= (unsigned)(emu::xchg()[i] & 1u) << i;
	emu::barrier_warp();
	return r;
}
static inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0u; }
static inline int __all_sync(unsigned m, int pred) { return __ballot_sync(m, pred) == 0xffffffffu; }
template <class T> static inline unsigned __match_any_sync(unsigned, T v)
{
	uint64_t raw = 0;
	memcpy(&raw, &v, sizeof(T));
	emu::xchg()[emu::lane()] = raw;
	emu::barrier_warp();
	unsigned r = 0;
	for (int i = 0; i < 32; i++) if (emu::xchg()[i] == raw) r |= 1u << i;
	emu::barrier_warp();
	return r;
}
static inline unsigned __activemask() { return 0xffffffffu; }

template <class T> static inline T __ldg(const T *p) { return *p; }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh)
{
	const uint64_t v = ((uint64_t)hi << 32) | lo;
	return (uint32_t)(v >> (sh & 31u));
}
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline long long clock64() { return 0; }

// fibers never run concurrently: plain read-modify-write is atomic enough
template <class T, class V> static inline T atomicXor(T *p, V v) { T o = *p; *p = o ^ (T)v; return o; }
template <class T, class V> static inline T atomicOr(T *p, V v) { T o = *p; *p = o | (T)v; return o; }
template <class T, class V> static inline T atomicAnd(T *p, V v) { T o = *p; *p = o & (T)v; return o; }
template <class T, class V> static inline T atomicAdd(T *p, V v) { T o = *p; *p = o + (T)v; return o; }
template <class T, class V> static inline T atomicMin(T *p, V v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class V> static inline T atomicMax(T *p, V v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }

#include "fake_runtime.h"
