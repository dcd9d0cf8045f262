// fake_runtime.h -- TEST STUB (tests/emul): the slice of the CUDA runtime API that
// manatee_b200/csrc/mtz_lib.cu uses, implemented on the host so that the WHOLE library --
// streaming engine, batching, device API, every launch site -- can be compiled by g++ (launch
// sites rewritten by tests/emul/make_emul_lib.py) and run on the SIMT emulator.
//   * "Device" and pinned memory are host memory that ends at a guard page: an out-of-bounds
//     access by a kernel or by the host code is a SIGSEGV (the CPU stand-in for memcheck).
//   * Streams are FIFOs of deferred operations and events are real dependencies.  By default
//     every operation runs when it is enqueued (synchronous, deterministic, fast).  With
//     MTZ_EMUL_ASYNC=<seed> operations are only executed when something waits for them, and the
//     next stream to make progress is chosen at random among those whose head is not blocked on
//     an event: any ordering the stream/event graph allows can happen, so a MISSING dependency
//     between streams shows up as wrong bytes on the CPU (a synchronous fake would hide it).
// Included at the end of tests/emul/cuda_runtime.h.  Test infrastructure only.
#pragma once
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>
#include <deque>
#include <functional>
#include <mutex>
#include <vector>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNotReady = 600 };
struct emu_stream_;
struct emu_event_;
typedef emu_stream_ *cudaStream_t;
typedef emu_event_ *cudaEvent_t;
struct dim3 { unsigned x, y, z; dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {} };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaHostAllocDefault = 0, cudaHostAllocPortable = 1, cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
struct cudaDeviceProp { char name[256]; int major, minor, multiProcessorCount; size_t totalGlobalMem; };
#define CUDART_CB
typedef void (*cudaHostFn_t)(void *);

// ------------------------------------------------------------------ streams and events
struct emu_event_ { unsigned long long recorded = 0, completed = 0; int dev = 0; };
struct emu_op {
	std::function<void()> fn;                 // work (may be empty)
	emu_event_ *wait_ev = nullptr; unsigned long long wait_seq = 0;
	emu_event_ *rec_ev = nullptr; unsigned long long rec_seq = 0;
};
struct emu_stream_ { std::deque<emu_op> q; bool busy = false; int dev = 0; };

namespace emurt {
struct State {
	std::recursive_mutex mu;
	std::vector<emu_stream_ *> streams;
	emu_stream_ null_stream;
	bool async = false;
	unsigned long long rng = 88172645463325252ull;
	State()
	{
		const char *e = getenv("MTZ_EMUL_ASYNC");
		if (e && *e && strcmp(e, "0") != 0) { async = true; rng ^= strtoull(e, nullptr, 10) * 0x9E3779B97F4A7C15ull; }
		streams.push_back(&null_stream);
	}
	unsigned long long next() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; }
};
inline State &S() { static State s; return s; }
inline emu_stream_ *str(cudaStream_t st) { return st ? st : &S().null_stream; }

// execute ONE runnable operation (random stream); false when nothing can run right now
inline bool step()
{
	State &s = S();
	std::unique_lock<std::recursive_mutex> lk(s.mu);
	std::vector<emu_stream_ *> ok;
	for (emu_stream_ *st : s.streams) {
		if (st->busy || st->q.empty()) continue;
		const emu_op &o = st->q.front();
		if (o.wait_ev && o.wait_ev->completed < o.wait_seq) continue;
		ok.push_back(st);
	}
	if (ok.empty()) return false;
	emu_stream_ *st = ok[s.next() % ok.size()];
	emu_op o = std::move(st->q.front());
	st->q.pop_front();
	st->busy = true;
	lk.unlock();
	if (o.fn) o.fn();
	lk.lock();
	if (o.rec_ev && o.rec_ev->completed < o.rec_seq) o.rec_ev->completed = o.rec_seq;
	st->busy = false;
	return true;
}
template <class P> inline void drain_until(P done)
{
	for (;;) {
		{
			std::lock_guard<std::recursive_mutex> g(S().mu);
			if (done()) return;
		}
		if (!step()) {
			std::lock_guard<std::recursive_mutex> g(S().mu);
			if (done()) return;
			// another thread is executing the operation we need, or it is not enqueued yet
			usleep(50);
		}
	}
}
inline int &cur_dev();
// everything enqueued on the CURRENT device (what cudaDeviceSynchronize / a blocking cudaMemcpy /
// cudaFree wait for): another device's stream may be sitting in a collective that waits for us
inline void drain_all()
{
	const int dev = cur_dev();
	drain_until([dev] {
		for (emu_stream_ *st : S().streams) if (st->dev == dev && (st->busy || !st->q.empty())) return false;
		return true;
	});
}
inline void enqueue(cudaStream_t st_, emu_op &&o)
{
	State &s = S();
	emu_stream_ *st = str(st_);
	if (!s.async) {
		// synchronous mode: the operation runs HERE, on the enqueuing thread, as soon as what it
		// waits for has completed.  (Handing it to whichever thread happens to drain next would let
		// one rank's thread block inside another rank's blocking collective -- tests/emul/nccl.h.)
		emu_event_ *wev = o.wait_ev; const unsigned long long wseq = o.wait_seq;
		drain_until([st, wev, wseq] { return !st->busy && st->q.empty() && (wev == nullptr || wev->completed >= wseq); });
		{
			std::lock_guard<std::recursive_mutex> g(s.mu);
			st->busy = true;
		}
		if (o.fn) o.fn();
		std::lock_guard<std::recursive_mutex> g(s.mu);
		if (o.rec_ev && o.rec_ev->completed < o.rec_seq) o.rec_ev->completed = o.rec_seq;
		st->busy = false;
		return;
	}
	{
		std::lock_guard<std::recursive_mutex> g(s.mu);
		st->q.push_back(std::move(o));
	}
}
inline void run(cudaStream_t st, std::function<void()> fn) { emu_op o; o.fn = std::move(fn); enqueue(st, std::move(o)); }
} // namespace emurt

// Device discipline, as the real runtime enforces it: a kernel launch or an event record needs the
// stream's device to be the CURRENT device of the calling thread (else error 400, "invalid
// resource handle", reported by the next cudaGetLastError like a failed launch is).
enum { cudaErrorInvalidResourceHandle = 400 };
namespace emurt {
inline int &cur_dev() { static thread_local int d = 0; return d; }
inline cudaError_t &sticky() { static thread_local cudaError_t e = cudaSuccess; return e; }
}
static inline const char *cudaGetErrorString(cudaError_t e)
{
	return e == cudaSuccess ? "no error" : e == cudaErrorInvalidResourceHandle ? "invalid resource handle" : "emulated CUDA error";
}
static inline cudaError_t cudaGetLastError() { cudaError_t e = emurt::sticky(); emurt::sticky() = cudaSuccess; return e; }
// MTZ_EMUL_DEVICES=<n>: a box of n identical emulated GPUs (device memory is host memory, so a
// "peer copy" is a copy; what the multi-device tests exercise is the library's ordering)
static inline cudaError_t cudaGetDeviceCount(int *n)
{
	const char *e = getenv("MTZ_EMUL_DEVICES");
	*n = getenv("MTZ_EMUL_NO_DEVICE") ? 0 : (e && atoi(e) > 0 ? atoi(e) : 1);
	return cudaSuccess;
}
static inline cudaError_t cudaDeviceCanAccessPeer(int *can, int, int) { *can = 1; return cudaSuccess; }
static inline cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { emurt::cur_dev() = d; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { emurt::drain_all(); return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int)
{
	memset(p, 0, sizeof *p);
	strcpy(p->name, "SIMT emulator (tests/emul)");
	p->major = 9; p->minor = 0;
	p->multiProcessorCount = 2;                 // small grids: the emulator runs CTAs one by one
	p->totalGlobalMem = (size_t)8 << 30;
	return cudaSuccess;
}

// guard-page allocation: [p, p+bytes rounded to 16) then an inaccessible page
static inline void *emu_dev_alloc(size_t bytes)
{
	const size_t page = (size_t)sysconf(_SC_PAGESIZE);
	const size_t body = (bytes + 15) & ~(size_t)15;
	const size_t npages = (body + page - 1) / page + 2;
	uint8_t *m = (uint8_t *)mmap(nullptr, npages * page + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
	if (m == MAP_FAILED) return nullptr;
	uint8_t *end = m + (npages - 1) * page;
	uint8_t *p = end - body;
	memset(m + page, 0xA5, (size_t)(p - (m + page)));
	// device memory is not zeroed: junk at both ends (touching every page of a multi-GiB slot
	// would cost minutes; the untouched middle stays lazily-mapped zero pages)
	{
		const size_t edge = body < ((size_t)2 << 20) ? body : ((size_t)1 << 20);
		memset(p, 0xCD, edge);
		memset(p + body - edge, 0xCD, edge);
	}
	((size_t *)m)[0] = npages * page + page;     // bookkeeping in the leading page
	mprotect(end, page, PROT_NONE);
	memcpy(p - sizeof(void *), &m, sizeof(void *));   // mapping start, just below the block
	return p;
}
static inline void emu_dev_free(void *p)
{
	if (p == nullptr) return;
	emurt::drain_all();                          // cudaFree synchronises
	uint8_t *m;
	memcpy(&m, (uint8_t *)p - sizeof(void *), sizeof(void *));
	munmap(m, ((size_t *)m)[0]);
}
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t bytes)
{
	*p = (T *)emu_dev_alloc(bytes ? bytes : 1);
	return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void *p) { emu_dev_free(p); return cudaSuccess; }
template <class T> static inline cudaError_t cudaHostAlloc(T **p, size_t bytes, unsigned)
{
	*p = (T *)emu_dev_alloc(bytes ? bytes : 1);
	return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFreeHost(void *p) { emu_dev_free(p); return cudaSuccess; }

static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { emurt::drain_all(); memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { emurt::drain_all(); memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t st = nullptr)
{
	emurt::run(st, [d, s, n] { memmove(d, s, n); });
	return cudaSuccess;
}
static inline cudaError_t cudaMemcpyPeerAsync(void *d, int, const void *s, int, size_t n, cudaStream_t st = nullptr)
{
	emurt::run(st, [d, s, n] { memmove(d, s, n); });
	return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st = nullptr)
{
	emurt::run(st, [d, v, n] { memset(d, v, n); });
	return cudaSuccess;
}

static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned)
{
	*s = new emu_stream_();
	(*s)->dev = emurt::cur_dev();
	std::lock_guard<std::recursive_mutex> g(emurt::S().mu);
	emurt::S().streams.push_back(*s);
	return cudaSuccess;
}
static inline cudaError_t cudaDeviceGetStreamPriorityRange(int *least, int *greatest)
{
	*least = 0; *greatest = -5;
	return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned flags, int)
{
	return cudaStreamCreateWithFlags(s, flags);
}
static inline cudaError_t cudaStreamSynchronize(cudaStream_t st_)
{
	emu_stream_ *st = emurt::str(st_);
	emurt::drain_until([st] { return !st->busy && st->q.empty(); });
	return cudaSuccess;
}
static inline cudaError_t cudaStreamDestroy(cudaStream_t st)
{
	cudaStreamSynchronize(st);
	std::lock_guard<std::recursive_mutex> g(emurt::S().mu);
	auto &v = emurt::S().streams;
	for (size_t i = 0; i < v.size(); i++) if (v[i] == st) { v.erase(v.begin() + (long)i); break; }
	delete st;
	return cudaSuccess;
}
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new emu_event_(); (*e)->dev = emurt::cur_dev(); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t st = nullptr)
{
	if (st != nullptr && (st->dev != e->dev || st->dev != emurt::cur_dev())) return cudaErrorInvalidResourceHandle;
	emu_op o;
	{
		std::lock_guard<std::recursive_mutex> g(emurt::S().mu);
		o.rec_ev = e; o.rec_seq = ++e->recorded;
	}
	emurt::enqueue(st, std::move(o));
	return cudaSuccess;
}
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t st, cudaEvent_t e, unsigned = 0)
{
	emu_op o;
	{
		std::lock_guard<std::recursive_mutex> g(emurt::S().mu);
		if (e->recorded == 0) return cudaSuccess;             // never recorded: no dependency
		o.wait_ev = e; o.wait_seq = e->recorded;              // the record that is current NOW
	}
	emurt::enqueue(st, std::move(o));
	return cudaSuccess;
}
static inline cudaError_t cudaEventSynchronize(cudaEvent_t e)
{
	unsigned long long want;
	{ std::lock_guard<std::recursive_mutex> g(emurt::S().mu); want = e->recorded; }
	emurt::drain_until([e, want] { return e->completed >= want; });
	return cudaSuccess;
}
static inline cudaError_t cudaEventQuery(cudaEvent_t e)
{
	emurt::step();                                           // a poller must make the device progress
	std::lock_guard<std::recursive_mutex> g(emurt::S().mu);
	return e->completed >= e->recorded ? cudaSuccess : cudaErrorNotReady;
}
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { cudaEventSynchronize(e); delete e; return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b)
{
	cudaEventSynchronize(a); cudaEventSynchronize(b);
	*ms = 0.001f;
	return cudaSuccess;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
static inline cudaError_t cudaLaunchHostFunc(cudaStream_t st, cudaHostFn_t fn, void *ud)
{
	emurt::run(st, [fn, ud] { fn(ud); });
	return cudaSuccess;
}
// defined at the end of the generated translation unit, where the one cooperative kernel is visible
static cudaError_t cudaLaunchCooperativeKernel(const void *f, dim3 grid, dim3 block, void **args, size_t smem,
    cudaStream_t st);

namespace emu {
// a launch site `k<<<g, b, smem, st>>>(args)` becomes
//     emu::launch_site(g, b, st, [=] { k(args); })
// the arguments are captured BY VALUE when the launch is enqueued, like a real launch does
template <class G, class B, class F> static inline void launch_site(G g, B b, cudaStream_t st, const F &f)
{
	const unsigned grid = (unsigned)g, block = (unsigned)b;
	if (st != nullptr && st->dev != emurt::cur_dev()) { emurt::sticky() = cudaErrorInvalidResourceHandle; return; }
	std::function<void()> k(f);
	emurt::run(st, [grid, block, k] { launch(grid, block, k); });
}
}
