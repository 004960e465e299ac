// common.cuh -- shared device/host helpers for the H100 (sm_90a) HNSW candidate-scoring path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#include "../../include/pgemb_b200.h"

// dynamic shared memory of the running CTA (the host emulation in tests/emu hands out a per-CTA buffer instead)
#ifdef PGEMB_HOST_EMULATION
#define PGEMB_DYNAMIC_SMEM(name, alignment) unsigned char *name = emu::dynamic_smem()
#else
#define PGEMB_DYNAMIC_SMEM(name, alignment) extern __shared__ __align__(alignment) unsigned char name[]
#endif

// kernel launch (under the host emulation a launch runs the grid on the emulator, synchronously)
#ifdef PGEMB_HOST_EMULATION
#define PGEMB_LAUNCH(kernel, grid, block, smem, stream, ...) \
	emu::launch(dim3(grid), (unsigned) (block), (size_t) (smem), [=]() { kernel(__VA_ARGS__); })
#else
#define PGEMB_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

namespace pgemb {

constexpr int kWarp = 32;
constexpr uint32_t kFull = 0xffffffffu;

// ---------------------------------------------------------------------------------------------
// Order-preserving map fp32 -> u32 (ascending float order == ascending unsigned order).
// The reference compares (dist, id) pairs with std::pair's operator< (hnswalg.cpp:52-53); packing
// (f2o(dist) << 32 | id) into a u64 reproduces that order for all non-NaN distances. -0.0 never
// occurs (L2 = sqrtf(sum of squares), manhattan = sum of |.|, cosine = 1 - x in round-to-nearest),
// so the bit order and the float order agree on ties too.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f2o(float f)
{
#ifdef __CUDA_ARCH__
	uint32_t b = __float_as_uint(f);
#else
	union { float f; uint32_t u; } cv; cv.f = f; uint32_t b = cv.u;
#endif
	return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__host__ __device__ __forceinline__ float o2f(uint32_t o)
{
	uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
	return __uint_as_float(b);
#else
	union { float f; uint32_t u; } cv; cv.u = b; return cv.f;
#endif
}

// Queue key: [63:32] f2o(dist)  [31:1] node id  [0] "expanded" flag.  ids are unique inside a queue so
// the flag never decides an ordering; node ids must be < 2^31.
__device__ __forceinline__ uint64_t make_key(float d, uint32_t id) { return ((uint64_t) f2o(d) << 32) | ((uint64_t) id << 1); }
__device__ __forceinline__ uint32_t key_dist(uint64_t k) { return (uint32_t) (k >> 32); }
__device__ __forceinline__ uint32_t key_id(uint64_t k) { return ((uint32_t) k) >> 1; }
__device__ __forceinline__ bool     key_expanded(uint64_t k) { return (k & 1ull) != 0; }
__device__ __forceinline__ uint64_t key_order(uint64_t k) { return k >> 1; }	// comparable, flag stripped

#ifndef PGEMB_HOST_EMULATION  // tests/emu supplies host versions of the PTX wrappers below
// ---------------------------------------------------------------------------------------------
// Hopper async-copy plumbing: mbarrier + 1-D bulk TMA (cp.async.bulk -> SASS UBLKCP).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init()
{
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
	uint32_t ok;
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
		"selp.u32 %0, 1, 0, p;\n\t}"
		: "=r"(ok)
		: "r"(smem_u32(bar)), "r"(parity)
		: "memory");
	return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
	while (!mbar_try_wait(bar, parity)) { }
}
__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
	uint64_t p;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
	return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
	uint64_t p;
	asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
	return p;
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned; completes on `bar`.
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar, uint64_t policy)
{
	asm volatile(
		"cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
		::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
		: "memory");
}

#endif  // PGEMB_HOST_EMULATION

// NOTE (kept from the LDGSTS gather experiments, rounds 1-2: measured slower than the bulk copies at every row size and
// removed, profiles/README.md): `cp.async.cg.shared.global.L2::cache_hint` miscompiles with
// ptxas 12.9 for sm_100a (the architecture of those experiments) -- it emits `LDGSTS [R+UR0], desc[UR1]` whose uniform registers are never written and the
// instruction traps ("illegal instruction", pinpointed with compute-sanitizer).  Bulk TMA takes the same policy fine.

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
#ifndef PGEMB_HOST_EMULATION
__device__ __forceinline__ uint32_t lanemask_lt()
{
	uint32_t m;
	asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
	return m;
}
#endif

}  // namespace pgemb
