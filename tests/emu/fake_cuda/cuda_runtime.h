// Host stand-in for <cuda_runtime.h> (tests/emu): compiles the .cuh kernels with g++ and runs them on the CPU.
//
// Execution model -- a small SIMT emulator, enough for this repo's kernels:
//   * a CTA is a group of OS threads, one per WARP; the 32 lanes of a warp are user-level fibers (ucontext) of that
//     thread.  A lane runs until it reaches a warp collective (__syncwarp, __ballot_sync, __shfl*_sync,
//     __match_any_sync), a CTA barrier (__syncthreads, bar.sync) or a spin-wait hook (mbarrier wait, __nanosleep); the
//     warp's scheduler then runs the next lane.  When every live lane waits at a collective the values are exchanged
//     and all lanes resume.  Warps of a CTA really run concurrently, so shared-memory locks and atomics between warps
//     are exercised; CTAs of a grid run one after another.
//   * shared memory: `__shared__` arrays become function-local statics, dynamic shared memory is a per-CTA buffer.
//   * mbarrier + 1-D bulk TMA: the copy is accounted on the barrier (expect-tx / complete-tx / phase parity) and performed
//     either by the issuing lane at once or -- PGEMB_EMU_TMA=late -- only when somebody polls that barrier: the two
//     extreme legal hardware schedules.  Under "late" a consumer that reads a ring without waiting for its barrier sees
//     the 0xAA fill instead of data, and a wait on the wrong barrier / parity never completes.
//   * arithmetic: the _rn intrinsics are plain IEEE operations (compile with -ffp-contract=off, no fast-math).
// It checks LOGIC (indexing, protocols, summation order), not memory-model races inside a warp and not speed.
// Test infrastructure only; never part of the product build.
#pragma once
#define PGEMB_HOST_EMULATION 1

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <pthread.h>
#include <sched.h>
#include <time.h>
#include <thread>
#include <ucontext.h>
#include <vector>

#define __host__
#define __device__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

struct dim3
{
	unsigned x = 1, y = 1, z = 1;
	dim3() {}
	dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }

namespace emu {

constexpr size_t kLaneStack = 192 * 1024;
enum State { RUNNABLE, AT_COLL, DONE };
enum Kind { K_WARP, K_CTA_BAR, K_CTA_OR };
struct PendingCopy { void *dst; const void *src; uint32_t bytes; uint64_t *bar; };

struct Cta
{
	std::vector<PendingCopy> pending;  // PGEMB_EMU_TMA=late: bulk copies issued but not yet performed (guarded by g_mbar_mu)
	pthread_barrier_t bars[16];
	unsigned		  nwarps = 0;
	unsigned		  or_acc[2] = {0, 0};  // __syncthreads_or accumulators, double-buffered by phase
	unsigned char	 *dyn_smem = nullptr;
	dim3			  block_idx;
};

struct Lane
{
	ucontext_t ctx;
	char	  *stack = nullptr;
	State	   st = RUNNABLE;
	uint64_t   xchg = 0;
	int		   site = 0;  // source line of the collective this lane waits at
	dim3	   tid;
	std::vector<PendingCopy> cp_pending;  // this thread's cp.async pieces that have not landed yet (late schedule)
};

struct Warp
{
	ucontext_t			  sched;
	Lane				  lane[32];
	int					  cur = 0;
	Cta					 *cta = nullptr;
	int					  kind = K_WARP, bar_id = 0, or_phase = 0;
	uint64_t			  snap[32];
	bool				  present[32];
	std::function<void()> body;
};

extern thread_local Warp *tl_warp;
extern dim3				   g_block_dim, g_grid_dim;
extern pthread_mutex_t	   g_mbar_mu;
extern int				   g_jitter;	// PGEMB_EMU_JITTER != 0: warps pause at random around atomics (perturbs the interleaving of slots)
extern int				   g_tma_late;	// set from PGEMB_EMU_TMA at every launch
extern int				   g_tma_unwaited;	// copies still pending when their CTA exited (late schedule), since load
extern int				   g_launch_error;	// error of the last launch the runtime refused, until cudaGetLastError() reads it
// dynamic shared memory a CTA may opt in to on the H100 (227 KB): a larger cudaFuncSetAttribute or launch fails, as on the device
constexpr size_t		   kMaxDynamicSmem = 232448;

inline Warp &W() { return *tl_warp; }
inline Lane &L() { return tl_warp->lane[tl_warp->cur]; }
inline int	 lane_index() { return tl_warp->cur; }

inline void collective(int kind, uint64_t v, int bar_id = 0, int site = 0)
{
	Warp &w = W();
	Lane &l = w.lane[w.cur];
	l.xchg = v;
	l.site = site;
	l.st = AT_COLL;
	w.kind = kind;
	w.bar_id = bar_id;
	swapcontext(&l.ctx, &w.sched);
}
// spin-wait hook: let the other lanes of the warp (and the other warps' threads) run
inline void yield()
{
	Warp &w = W();
	Lane &l = w.lane[w.cur];
	swapcontext(&l.ctx, &w.sched);
}
// interleaving stress: called around every atomic; a warp's thread gives up the core (or sleeps a little) at random so that
// lock hand-overs, work stealing and table updates of different warps meet in many orders
inline void jitter()
{
	if (!g_jitter) return;
	static thread_local uint32_t r = 0;
	if (r == 0) r = (uint32_t) (uintptr_t) &r * 2654435761u | 1u;
	r ^= r << 13;
	r ^= r >> 17;
	r ^= r << 5;
	if ((r & 7u) == 0u) sched_yield();
	if ((r & 127u) == 1u)
	{
		struct timespec ts = {0, (long) (20000 + (r >> 20))};
		nanosleep(&ts, nullptr);
	}
}
inline unsigned char *dynamic_smem() { return W().cta->dyn_smem; }

void run_warp(Warp &w);	 // scheduler loop (emu_runtime.cpp)

// Run kernel body `fn` (called once per CUDA thread) over a grid; blocks are executed one after another.
void launch(dim3 grid, unsigned block_threads, size_t dyn_smem_bytes, const std::function<void()> &fn);

}  // namespace emu

#define threadIdx (emu::L().tid)
#define blockIdx (emu::W().cta->block_idx)
#define blockDim (emu::g_block_dim)
#define gridDim (emu::g_grid_dim)

// ---- barriers and warp collectives ------------------------------------------------------------------
static inline void __syncthreads(int site = __builtin_LINE()) { emu::collective(emu::K_CTA_BAR, 0, 0, site); }
static inline int  __syncthreads_or(int pred, int site = __builtin_LINE())
{
	emu::collective(emu::K_CTA_OR, pred ? 1u : 0u, 0, site);
	return (int) emu::W().snap[emu::W().cur];  // the scheduler stores the CTA-wide result in every lane's slot
}
static inline void __syncwarp(unsigned = 0xffffffffu, int site = __builtin_LINE()) { emu::collective(emu::K_WARP, 0, 0, site); }
static inline unsigned __ballot_sync(unsigned, int pred, int site = __builtin_LINE())
{
	emu::collective(emu::K_WARP, pred ? 1u : 0u, 0, site);
	const emu::Warp &w = emu::W();
	unsigned		 r = 0;
	for (int i = 0; i < 32; i++)
		if (w.present[i] && w.snap[i]) r |= 1u << i;
	return r;
}
template <typename T> static inline T __shfl_sync(unsigned, T v, int src, int width = 32, int site = __builtin_LINE())
{
	uint64_t b = 0;
	memcpy(&b, &v, sizeof(T));
	emu::collective(emu::K_WARP, b, 0, site);
	const emu::Warp &w = emu::W();
	const int		 base = w.cur / width * width;
	T				 out;
	memcpy(&out, &w.snap[base + ((src % width) + width) % width], sizeof(T));
	return out;
}
template <typename T> static inline T __shfl_xor_sync(unsigned, T v, int lanemask, int width = 32, int site = __builtin_LINE())
{
	uint64_t b = 0;
	memcpy(&b, &v, sizeof(T));
	emu::collective(emu::K_WARP, b, 0, site);
	const emu::Warp &w = emu::W();
	int				 s = w.cur ^ lanemask;
	if (s / width != w.cur / width) s = w.cur;
	T out;
	memcpy(&out, &w.snap[s], sizeof(T));
	return out;
}
static inline int __any_sync(unsigned m, int pred, int site = __builtin_LINE()) { return __ballot_sync(m, pred, site) != 0u; }
static inline unsigned __match_any_sync(unsigned, unsigned v, int site = __builtin_LINE())
{
	emu::collective(emu::K_WARP, v, 0, site);
	const emu::Warp &w = emu::W();
	unsigned		 r = 0;
	for (int i = 0; i < 32; i++)
		if (w.present[i] && (unsigned) w.snap[i] == v) r |= 1u << i;
	return r;
}
static inline void coop_bar(int id, uint32_t, int site = __builtin_LINE()) { emu::collective(emu::K_CTA_BAR, 0, id, site); }

// ---- bit tricks, conversions, arithmetic ------------------------------------------------------------
static inline int	   __popc(unsigned v) { return __builtin_popcount(v); }
static inline int	   __ffs(unsigned v) { return __builtin_ffs((int) v); }
static inline int	   __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int	   __clz(unsigned v) { return v ? __builtin_clz(v) : 32; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float	   __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float	   __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline float	   __fadd_rn(float a, float b) { return a + b; }
static inline float	   __fsub_rn(float a, float b) { return a - b; }
static inline float	   __fmul_rn(float a, float b) { return a * b; }
static inline float	   __fsqrt_rn(float a) { return sqrtf(a); }
static inline double   __dsqrt_rn(double a) { return sqrt(a); }
static inline double   __ddiv_rn(double a, double b) { return a / b; }
static inline float	   __double2float_rn(double a) { return (float) a; }
using std::max;
using std::min;

// ---- memory -----------------------------------------------------------------------------------------
template <typename T> static inline T __ldg(const T *p) { return *p; }
template <typename T> static inline T __ldcg(const T *p) { return *reinterpret_cast<const volatile T *>(p); }
static inline void					  __threadfence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void					  __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __nanosleep(unsigned)
{
	sched_yield();
	emu::yield();
}
static inline unsigned atomicAdd(unsigned *p, unsigned v) { emu::jitter(); return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicOr(unsigned *p, unsigned v) { emu::jitter(); return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicXor(unsigned *p, unsigned v) { emu::jitter(); return __atomic_fetch_xor(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicMin(unsigned *p, unsigned v)
{
	unsigned old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
	while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
	return old;
}
static inline unsigned atomicCAS(unsigned *p, unsigned cmp, unsigned val)
{
	unsigned e = cmp;
	emu::jitter();
	__atomic_compare_exchange_n(p, &e, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
	emu::jitter();
	return e;
}
static inline unsigned long long atomicOr(unsigned long long *p, unsigned long long v) { emu::jitter(); return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicCAS(unsigned long long *p, unsigned long long cmp, unsigned long long val)
{
	unsigned long long e = cmp;
	emu::jitter();
	__atomic_compare_exchange_n(p, &e, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
	emu::jitter();
	return e;
}
static inline size_t __cvta_generic_to_shared(const void *p) { return (size_t) p; }
// (the runtime API the host code uses is emulated at the end of this header)
typedef int cudaError_t;
static inline cudaError_t cudaFree(void *p) { free(p); return 0; }

// ---- mbarrier + 1-D bulk TMA (host versions of the wrappers common.cuh guards out) --------------------
// 64-bit barrier word: [0] phase parity, [1..15] pending arrivals, [16..30] arrival count, [32..63] tx bytes (signed)
namespace emu {
struct BarView { uint32_t w0; int32_t tx; };
inline void bar_complete_if_done(BarView &v)
{
	if (((v.w0 >> 1) & 0x7fffu) == 0 && v.tx == 0)
	{
		const uint32_t init = (v.w0 >> 16) & 0x7fffu;
		v.w0 = ((v.w0 & 1u) ^ 1u) | (init << 1) | (init << 16);
	}
}
}  // namespace emu
// 32-bit shared-memory address of a pointer into the CTA's DYNAMIC shared memory (offset from its base; the only use)
static inline uint32_t smem_u32(const void *p)
{
	const ptrdiff_t off = (const unsigned char *) p - emu::dynamic_smem();
	if (off < 0 || off > (ptrdiff_t) (1 << 20))
	{
		fprintf(stderr, "emu: smem_u32 of a pointer outside dynamic shared memory\n");
		abort();
	}
	return (uint32_t) off;
}
static inline void	   mbar_init(uint64_t *bar, uint32_t count)
{
	emu::BarView v{(count << 1) | (count << 16), 0};
	memcpy(bar, &v, 8);
}
static inline void fence_mbar_init() {}
static inline void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
	pthread_mutex_lock(&emu::g_mbar_mu);
	emu::BarView v;
	memcpy(&v, bar, 8);
	v.tx += (int32_t) bytes;
	const uint32_t pend = ((v.w0 >> 1) & 0x7fffu) - 1u;
	v.w0 = (v.w0 & ~(0x7fffu << 1)) | ((pend & 0x7fffu) << 1);
	emu::bar_complete_if_done(v);
	memcpy(bar, &v, 8);
	pthread_mutex_unlock(&emu::g_mbar_mu);
}
static inline bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
	pthread_mutex_lock(&emu::g_mbar_mu);
	emu::BarView v;
	memcpy(&v, bar, 8);
	{
		// late schedule: the copies that signal this barrier land now
		std::vector<emu::PendingCopy> &pq = emu::W().cta->pending;
		for (size_t i = 0; i < pq.size();)
		{
			if (pq[i].bar != bar)
			{
				i++;
				continue;
			}
			memcpy(pq[i].dst, pq[i].src, pq[i].bytes);
			v.tx -= (int32_t) pq[i].bytes;
			pq[i] = pq.back();
			pq.pop_back();
		}
		emu::bar_complete_if_done(v);
		memcpy(bar, &v, 8);
	}
	pthread_mutex_unlock(&emu::g_mbar_mu);
	if ((v.w0 & 1u) != (parity & 1u)) return true;
	emu::yield();
	return false;
}
static inline void mbar_wait(uint64_t *bar, uint32_t parity)
{
	while (!mbar_try_wait(bar, parity)) {}
}
static inline uint64_t l2_policy_evict_first() { return 0; }
static inline uint64_t l2_policy_evict_last() { return 0; }
static inline void	   tma_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t)
{
	if ((bytes & 15u) || ((uintptr_t) dst & 15u) || ((uintptr_t) src & 15u))
	{
		fprintf(stderr, "emu: cp.async.bulk needs 16-byte aligned addresses and size (dst %p src %p bytes %u)\n", dst, src, bytes);
		abort();
	}
	pthread_mutex_lock(&emu::g_mbar_mu);
	if (emu::g_tma_late)
	{
		emu::W().cta->pending.push_back(emu::PendingCopy{dst, src, bytes, bar});
		pthread_mutex_unlock(&emu::g_mbar_mu);
		return;
	}
	memcpy(dst, src, bytes);
	emu::BarView v;
	memcpy(&v, bar, 8);
	v.tx -= (int32_t) bytes;
	emu::bar_complete_if_done(v);
	memcpy(bar, &v, 8);
	pthread_mutex_unlock(&emu::g_mbar_mu);
}
// 16-byte cp.async pieces: owned by the issuing THREAD.  Under PGEMB_EMU_TMA=late a piece lands only when its own thread
// waits for its groups -- another lane that reads it without the __syncwarp() after the wait sees the 0xAA fill.
static inline void cp_async_16(void *dst, const void *src)
{
	if (((uintptr_t) dst & 15u) || ((uintptr_t) src & 15u))
	{
		fprintf(stderr, "emu: cp.async 16 needs 16-byte aligned addresses (dst %p src %p)\n", dst, src);
		abort();
	}
	if (emu::g_tma_late)
		emu::L().cp_pending.push_back(emu::PendingCopy{dst, src, 16u, nullptr});
	else
		memcpy(dst, src, 16);
}
static inline void cp_async_16_x8(uint32_t dst_smem_u32, const void *src, uint32_t rem)
{
	for (uint32_t j = 0; j < 8u; j++)
		if (rem > 512u * j) cp_async_16(emu::dynamic_smem() + dst_smem_u32 + 512u * j, (const unsigned char *) src + 512u * j);
}
static inline void cp_async_16_s32(uint32_t dst_smem_u32, const void *src) { cp_async_16(emu::dynamic_smem() + dst_smem_u32, src); }
static inline void cp_async_commit() {}
static inline void cp_async_wait_all()
{
	std::vector<emu::PendingCopy> &pq = emu::L().cp_pending;
	for (const emu::PendingCopy &c : pq) memcpy(c.dst, c.src, c.bytes);
	pq.clear();
}
static inline void cp_async_wait_but2() { cp_async_wait_all(); }  // waiting for more than asked is a legal schedule
static inline uint32_t lanemask_lt() { return (1u << (emu::L().tid.x & 31u)) - 1u; }

// ---- the part of the CUDA runtime API capi.cu uses ---------------------------------------------------------
// Device memory is host memory, streams execute in call order (every "async" call completes before it returns),
// events are wall-clock time stamps.  Enough to run the library's host logic (workspaces, build orchestration,
// staging, error paths) over the emulated kernels.
#include <chrono>
enum cudaErrorEmu { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaLimit { cudaLimitPersistingL2CacheSize = 6 };
enum cudaStreamAttrID { cudaStreamAttributeAccessPolicyWindow = 1 };
enum cudaAccessProperty { cudaAccessPropertyNormal = 0, cudaAccessPropertyStreaming = 1, cudaAccessPropertyPersisting = 2 };
struct cudaAccessPolicyWindow { void *base_ptr; size_t num_bytes; float hitRatio; cudaAccessProperty hitProp, missProp; };
union cudaStreamAttrValue { cudaAccessPolicyWindow accessPolicyWindow; int pad[16]; };
struct cudaDeviceProp { int multiProcessorCount; int persistingL2CacheMaxSize; int accessPolicyMaxWindowSize; };
struct EmuStream { int id; };
struct EmuEvent { double t_ms; };
typedef EmuStream *cudaStream_t;
typedef EmuEvent  *cudaEvent_t;

static inline const char *cudaGetErrorString(cudaError_t e) { return e == 0 ? "no error" : (e == 2 ? "out of memory" : "invalid value"); }
static inline cudaError_t cudaGetLastError()
{
	const cudaError_t e = emu::g_launch_error;
	emu::g_launch_error = cudaSuccess;
	return e;
}
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaCtxResetPersistingL2Cache() { return cudaSuccess; }
static inline cudaError_t cudaDeviceSetLimit(cudaLimit, size_t) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int)
{
	const char *v = getenv("PGEMB_EMU_SMS");
	p->multiProcessorCount = (v && *v) ? atoi(v) : 2;
	p->persistingL2CacheMaxSize = 0;
	p->accessPolicyMaxWindowSize = 0;
	return cudaSuccess;
}
template <typename T> static inline cudaError_t cudaMalloc(T **p, size_t bytes)
{
	*p = (T *) aligned_alloc(256, (bytes + 255) / 256 * 256 + 256);
	if (*p) memset((void *) *p, 0xCD, bytes);  // device memory is not zeroed
	return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
template <typename T> static inline cudaError_t cudaMallocHost(T **p, size_t bytes) { return cudaMalloc(p, bytes); }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr)
{
	for (size_t r = 0; r < h; r++) memmove((char *) d + r * dp, (const char *) s + r * sp, w);
	return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new EmuStream{1}; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaStreamSetAttribute(cudaStream_t, cudaStreamAttrID, const cudaStreamAttrValue *) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new EmuEvent{0.0}; return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr)
{
	e->t_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
	return cudaSuccess;
}
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float) (b->t_ms - a->t_ms); return cudaSuccess; }
template <typename F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute a, int v)
{
	return (a == cudaFuncAttributeMaxDynamicSharedMemorySize && (v < 0 || (size_t) v > emu::kMaxDynamicSmem)) ? cudaErrorInvalidValue : cudaSuccess;
}
template <typename F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) { *n = 1; return cudaSuccess; }

namespace cub {
struct DeviceRadixSort
{
	template <typename K>
	static cudaError_t SortKeys(void *tmp, size_t &bytes, const K *in, K *out, int n, int = 0, int = sizeof(K) * 8, cudaStream_t = nullptr)
	{
		if (!tmp)
		{
			bytes = 16;
			return cudaSuccess;
		}
		std::copy(in, in + n, out);
		std::sort(out, out + n);
		return cudaSuccess;
	}
};
}  // namespace cub
