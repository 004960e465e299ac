// scan_umma_kernel.cuh -- K6: the brute-force operator path (`ORDER BY val <op> q LIMIT k` without the index,
// embedding.c:1022-1062 + embedding--0.3.6.sql:20-44; SURVEY.md 8(f3), section 2 "K6") as ONE dense contraction on the
// tensor cores of sm_90a.  This is the only place of the extension where a batched-query x row-block contraction is
// genuinely dense, so it is the only kernel here that uses wgmma / TMA tensor maps.
//
//     S[q][r] = sum_d Q[q][d] * V[r][d]          tf32 wgmma, fp32 accumulate in registers, operands K-major in shared memory
//
// A tensor-core product cannot give the reference's bits (TF32 keeps 10 mantissa bits; the reference's summation order is
// fixed, DESIGN.md section 4), so S is used only to DISCARD rows, never to rank them:
//
//   scan_filter_wgmma_kernel  persistent, warp-specialised: warpgroup 0 = TMA producer (one thread, cp.async.bulk.tensor.2d,
//                             128-byte swizzle, 4-stage mbarrier ring), warpgroups 1-2 = consumers (wgmma m64n256k8 tf32,
//                             64 queries x 256 rows each, then the filter on the accumulator registers).  S is never written:
//                             a (query,row) pair survives only if a RIGOROUS lower bound of its distance -- from S, the
//                             exact squared norms and the TF32 error bound |S - q.v| <= rel |q||v| -- does not exceed the
//                             query's current k-th best exact distance; survivors go to a per-query candidate list.
//   scan_rescore_kernel       one CTA per query: candidates are re-scored with the reference-exact arithmetic
//                             (dist_exact.cuh, one lane per candidate) and folded into the running top-k by (dist,label),
//                             exactly like scan_select_kernel; then the query's filter constants are refreshed for the next chunk.
//
// The host (capi.cu, scan_filter_pass) walks the table in geometrically growing chunks (256, 512, 1K, ... rows): the first
// chunk establishes the threshold, every later chunk is filtered with the exact threshold of everything before it, so
// ~k ln(N/k) + (rows inside the error band) candidates per query are re-scored in total.  Result = the exact path's: same
// labels, same order, bit-identical distances (tests/test_gpu_scan_umma.py).  Every re-scored candidate
// also CHECKS the error bound against its exact distance (tripwire -> the host repeats the scan on the exact kernels).
// A query whose candidate list overflows is re-scored against the whole chunk (exact, slow, still correct).
// Manhattan has no bilinear form and stays on the exact tiled kernel.
#pragma once
#include "aux_kernels.cuh"
#include "common.cuh"
#include "dist_exact.cuh"

#ifndef PGEMB_HOST_EMULATION
#include <cuda.h>  // CUtensorMap (type only; cuTensorMapEncodeTiled is fetched through cudaGetDriverEntryPoint)
#endif

namespace pgemb {

constexpr uint32_t kUmmaTQ = 128;	  // queries per tile = two wgmma M = 64 halves
constexpr uint32_t kUmmaTR = 256;	  // rows per tile    = wgmma N
constexpr uint32_t kUmmaBK = 32;	  // floats per k-block = one 128-byte swizzle atom
constexpr uint32_t kUmmaStages = 4;	  // shared-memory ring depth
constexpr uint32_t kUmmaThreads = 384;  // three warpgroups: producer + two consumers
constexpr uint32_t kUmmaABytes = kUmmaTQ * kUmmaBK * 4;	 // 16 KB
constexpr uint32_t kUmmaBBytes = kUmmaTR * kUmmaBK * 4;	 // 32 KB
constexpr uint32_t kUmmaStageBytes = kUmmaABytes + kUmmaBBytes;
// dynamic shared memory: ring (1024-byte aligned) + row constants (2 x 256 x float2) + barriers
constexpr uint32_t kUmmaSmem = 1024 + kUmmaStages * kUmmaStageBytes + 2 * kUmmaTR * 8 + 256;

constexpr float kFilterEps = 2e-4f;	 // slack for fp32 rounding of norms / of the reference's own summation (see below)

// ---- the filter predicate (shared by the tensor-core epilogue, the re-scoring kernel and the host emulation) -------------
// Let qn, vn be the squared norms (fp32 sums, relative error <= dim/4 * 2^-24 each), S the tensor-core product with
// |S - q.v| <= rel * sqrt(qn vn) (Cauchy-Schwarz bounds sum |q_i v_i|), T the k-th best EXACT distance so far (+inf if < k).
//   cosine: dist = 1 - q.v / sqrt(qn vn);  lower bound lb = 1 - S/sqrt(qn vn) - rel - eps.
//           discard  <=>  lb > T  <=>  S / sqrt(vn) < (1 - rel - eps - T) sqrt(qn)
//   L2:     dist^2 = qn + vn - 2 q.v;      lower bound lb2 = (qn + vn)(1 - eps) - 2 S - 2 rel sqrt(qn) sqrt(vn).
//           discard  <=>  lb2 > T^2 (1 + 4e-6)  <=>  S < (qn (1-eps) - T2)/2 + vn (1-eps)/2 - rel sqrt(qn) sqrt(vn)
// Comparisons are written so that NaN (zero vectors under cosine, inf - inf) NEVER discards.
template <int METRIC>
__host__ __device__ __forceinline__ float2 filter_qconst(float qn, float T, float rel)
{
	float2 c;
	if (METRIC == M_COS)
	{
		c.x = (1.0f - (rel + kFilterEps) - T) * sqrtf(qn);
		c.y = 0.0f;
	}
	else
	{
		const float T2 = T * T * (1.0f + 4e-6f);
		c.x = (qn * (1.0f - kFilterEps) - T2) * 0.5f;
		c.y = rel * sqrtf(qn);
	}
	return c;
}
template <int METRIC>
__host__ __device__ __forceinline__ float2 filter_rconst(float vn)
{
	float2 c;
	if (METRIC == M_COS)
	{
		c.x = 1.0f / sqrtf(vn);
		c.y = 0.0f;
	}
	else
	{
		c.x = vn * (1.0f - kFilterEps) * 0.5f;
		c.y = sqrtf(vn);
	}
	return c;
}
template <int METRIC>
__host__ __device__ __forceinline__ bool filter_pass(float s, float2 qc, float2 rc)
{
	if (METRIC == M_COS) return !(s * rc.x < qc.x);
	return !(s < (qc.x + rc.x) - qc.y * rc.y);
}
// the approximate distance (cosine) / squared distance (L2) the product stands for, and its error bound: the tripwire.
// |q||v| is taken as sqrt(qn) sqrt(vn): the product qn vn leaves the fp32 range (subnormal below |q||v| = 2^-63, zero below
// ~2^-75, inf above 2^64) long before the squared norms do, and would drop the rel term from the slack or make it infinite.
template <int METRIC>
__host__ __device__ __forceinline__ void filter_approx(float s, float qn, float vn, float rel, float *approx, float *slack)
{
	const float scale = sqrtf(qn) * sqrtf(vn);
	if (METRIC == M_COS)
	{
		*approx = 1.0f - s / scale;
		*slack = rel + kFilterEps;
	}
	else
	{
		*approx = qn + vn - 2.0f * s;
		*slack = 2.0f * rel * scale + kFilterEps * (qn + vn);
	}
}

struct ScanFilterParams
{
	uint32_t	   nq;		  // queries of this group (tensor map Q covers exactly these)
	uint32_t	   r0, nr;	  // chunk: rows [r0, r0 + nr) of the table
	uint32_t	   kblocks;	  // ceil(row_f / 32)
	uint32_t	   n_qtiles, n_rtiles;
	const float2  *qconst;	  // [nq]
	const float	  *vnorm2;	  // [N] squared norms, indexed by table row
	uint32_t	  *cand_rows; // [nq][cap]
	float		  *cand_s;	  // [nq][cap]
	uint32_t	  *cand_n;	  // [nq]   (may exceed cap: overflow)
	uint32_t	   cap;
	float		  *dbg_s;	  // tests only: when set, the epilogue writes the raw products S[q * nr + j] here and filters nothing
};

#ifndef PGEMB_HOST_EMULATION
// ---------------------------------------------------------------------------------------------------------------------
// PTX wrappers (wgmma / 2-D TMA).  SASS: HGMMA, UTMALDG, SYNCS (mbarrier).
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap *tmap, uint32_t bar_smem, int32_t c0, int32_t c1)
{
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst_smem),
				 "l"(tmap), "r"(bar_smem), "r"(c0), "r"(c1)
				 : "memory");
}
__device__ __forceinline__ void tmap_prefetch(const CUtensorMap *tmap) { asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulators are written asynchronously: tie every register to this point so that no read is scheduled above the wait
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[128])
{
#pragma unroll
	for (uint32_t i = 0; i < 128; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 256] (+)= A[64 x 8] * B[256 x 8]^T, tf32 operands from shared memory (both K-major), fp32 accumulators in registers
#define PGEMB_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define PGEMB_D16(i) PGEMB_D4(i), PGEMB_D4(i + 4), PGEMB_D4(i + 8), PGEMB_D4(i + 12)
__device__ __forceinline__ void wgmma_m64n256k8_tf32(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"setp.ne.b32 p, %130, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
		"%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
		"%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "
		"%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, "
		"%77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, "
		"%102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, "
		"%123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
		: PGEMB_D16(0), PGEMB_D16(16), PGEMB_D16(32), PGEMB_D16(48), PGEMB_D16(64), PGEMB_D16(80), PGEMB_D16(96), PGEMB_D16(112)
		: "l"(a_desc), "l"(b_desc), "r"(accumulate)
		: "memory");
}
#undef PGEMB_D16
#undef PGEMB_D4
// mbarrier wait that cannot hang the GPU: a pipeline bug (wrong byte count, wrong parity) would otherwise spin forever.  Every
// legitimate wait in this kernel is microseconds; after ~2^24 polls (seconds) the kernel traps and the launch fails loudly.
__device__ __forceinline__ void umma_wait(uint64_t *bar, uint32_t parity)
{
	for (uint32_t i = 0; i < (1u << 24); i++)
		if (mbar_try_wait(bar, parity)) return;
	__trap();
}

// Shared-memory matrix descriptor (sm_90 GMMA): K-major tile of 128-byte rows written by TMA with CU_TENSOR_MAP_SWIZZLE_128B.
// start address >> 4 in [0,14); LBO (ignored for swizzled K-major) = 1 in [16,30); SBO = 1024 B (8 rows x 128 B) >> 4 in
// [32,46); layout SWIZZLE_128B (1) in [62,64).
__device__ __forceinline__ uint64_t wgmma_smem_desc(uint32_t smem_addr)
{
	return (uint64_t) ((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t) 1 << 16) | ((uint64_t) (1024u >> 4) << 32) | ((uint64_t) 1 << 62);
}

// ---------------------------------------------------------------------------------------------------------------------
// The filter kernel.  grid = min(tiles, SMs) persistent CTAs; tile t -> (row tile t / n_qtiles, query tile t % n_qtiles):
// CTAs that run at the same time share row tiles, so the table streams from HBM once and is re-read from L2.
// Warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 each own 64 of the tile's 128 queries: they issue the
// wgmma chain of the tile (m64n256k8, 4 per k-block, one k-block in flight while the previous ring slot is released) and
// then filter their accumulators in registers.
// Accumulator layout (per warpgroup, thread = warp w, lane l): d[4 i + 2 h + b] = S[16 w + l / 4 + 8 h][8 i + 2 (l % 4) + b].
// ---------------------------------------------------------------------------------------------------------------------
template <int METRIC>
__global__ void __launch_bounds__(kUmmaThreads, 1)
	scan_filter_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_v, const ScanFilterParams p)
{
	static_assert(METRIC == M_L2 || METRIC == M_COS, "the filter needs a bilinear form");
	extern __shared__ unsigned char umma_smem_raw[];
	const uint32_t raw = smem_u32(umma_smem_raw);
	const uint32_t ring = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles must be 1024-byte aligned
	unsigned char *ring_p = umma_smem_raw + (ring - raw);
	float2		  *rc_s = reinterpret_cast<float2 *>(ring_p + kUmmaStages * kUmmaStageBytes);  // [2][kUmmaTR]
	uint64_t	  *bars = reinterpret_cast<uint64_t *>(ring_p + kUmmaStages * kUmmaStageBytes + 2 * kUmmaTR * 8);
	uint64_t	  *full = bars, *empty = bars + kUmmaStages;

	const uint32_t wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const uint32_t n_tiles = p.n_qtiles * p.n_rtiles;

	if (threadIdx.x == 0)
	{
		for (uint32_t s = 0; s < kUmmaStages; s++)
		{
			mbar_init(&full[s], 1);
			mbar_init(&empty[s], 8);  // one arrival per consumer warp
		}
		fence_mbar_init();
		tmap_prefetch(&tmap_q);
		tmap_prefetch(&tmap_v);
	}
	__syncthreads();

	if (wg == 0)
	{
		// ===== TMA producer (one thread) =====
		asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
		if (warp == 0 && lane == 0)
		{
			uint32_t it = 0;
			for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x)
			{
				const uint32_t rt = t / p.n_qtiles, qt = t % p.n_qtiles;
				const int32_t  q0 = (int32_t) (qt * kUmmaTQ), row0 = (int32_t) (p.r0 + rt * kUmmaTR);
				for (uint32_t kb = 0; kb < p.kblocks; kb++, it++)
				{
					const uint32_t s = it % kUmmaStages, ph = (it / kUmmaStages) & 1u;
					umma_wait(&empty[s], ph ^ 1u);
					mbar_arrive_expect_tx(&full[s], kUmmaStageBytes);
					const uint32_t a_dst = ring + s * kUmmaStageBytes, b_dst = a_dst + kUmmaABytes;
					tma_load_2d(a_dst, &tmap_q, smem_u32(&full[s]), (int32_t) (kb * kUmmaBK), q0);
					tma_load_2d(b_dst, &tmap_v, smem_u32(&full[s]), (int32_t) (kb * kUmmaBK), row0);
				}
			}
		}
		return;
	}

	// ===== consumers: warpgroups 1, 2 =====
	asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
	const uint32_t cw = warp & 3u;						// warp inside the warpgroup
	const uint32_t ct = threadIdx.x - 128u;				// 0..255
	const uint32_t a_off = (wg - 1u) * 64u * 128u;		// this warpgroup's 64 query rows of the A tile
	const uint32_t quad = lane & 3u;
	uint32_t	   it = 0, ti = 0;
	float		   d[128];
#pragma unroll
	for (uint32_t i = 0; i < 128; i++) d[i] = 0.0f;
	for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x, ti++)
	{
		const uint32_t rt = t / p.n_qtiles, qt = t % p.n_qtiles;
		const uint32_t row_rel0 = rt * kUmmaTR;					 // first row of the tile, relative to r0
		const uint32_t valid = min(kUmmaTR, p.nr - row_rel0);	 // rows of this tile inside the chunk
		// row constants of the tile -> shared memory (one row per thread; double-buffered: the barrier below also orders the
		// other warpgroup's reads of the previous tile before these writes are reused two tiles later)
		float2 *rc = rc_s + (ti & 1u) * kUmmaTR;
		rc[ct] = (ct < valid) ? filter_rconst<METRIC>(p.vnorm2[p.r0 + row_rel0 + ct]) : make_float2(0.f, 0.f);
		asm volatile("bar.sync 1, 256;" ::: "memory");

		// ---- the product: one k-block in flight, the ring slot of the previous one is released as soon as it retires ----
		for (uint32_t kb = 0; kb < p.kblocks; kb++, it++)
		{
			const uint32_t s = it % kUmmaStages, ph = (it / kUmmaStages) & 1u;
			umma_wait(&full[s], ph);
			const uint32_t a_src = ring + s * kUmmaStageBytes + a_off, b_src = ring + s * kUmmaStageBytes + kUmmaABytes;
			const uint64_t a_desc = wgmma_smem_desc(a_src), b_desc = wgmma_smem_desc(b_src);
			wgmma_fence();
#pragma unroll
			for (uint32_t j = 0; j < kUmmaBK / 8; j++)	// K = 8 tf32 (32 bytes) per instruction: +2 in the 16-byte address field
				wgmma_m64n256k8_tf32(d, a_desc + 2 * j, b_desc + 2 * j, (kb | j) != 0u ? 1u : 0u);
			wgmma_commit();
			wgmma_wait<1>();
			if (kb > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % kUmmaStages]);
		}
		wgmma_wait<0>();
		wgmma_fence_regs(d);
		if (lane == 0) mbar_arrive(&empty[(it - 1) % kUmmaStages]);

		// ---- epilogue: thread = two queries (h = 0, 1) x 64 columns ----
		const uint32_t qrow = qt * kUmmaTQ + (wg - 1u) * 64u + cw * 16u + (lane >> 2);
#pragma unroll
		for (uint32_t h = 0; h < 2; h++)
		{
			const uint32_t q = qrow + 8u * h;
			const bool	   q_ok = q < p.nq;
			if (p.dbg_s != nullptr)
			{
				if (q_ok)
				{
#pragma unroll
					for (uint32_t i = 0; i < kUmmaTR / 8; i++)
#pragma unroll
						for (uint32_t b = 0; b < 2; b++)
						{
							const uint32_t c = 8u * i + 2u * quad + b;
							if (c < valid) p.dbg_s[(size_t) q * p.nr + row_rel0 + c] = d[4 * i + 2 * h + b];
						}
				}
				continue;
			}
			const float2 qc = q_ok ? p.qconst[q] : make_float2(0.f, 0.f);
			// survivors: bit 2 i + b of `pass` = column 8 i + 2 (l % 4) + b
			uint64_t pass = 0;
#pragma unroll
			for (uint32_t i = 0; i < kUmmaTR / 8; i++)
#pragma unroll
				for (uint32_t b = 0; b < 2; b++)
				{
					const uint32_t c = 8u * i + 2u * quad + b;
					if (q_ok && c < valid && filter_pass<METRIC>(d[4 * i + 2 * h + b], qc, rc[c])) pass |= 1ull << (2 * i + b);
				}
			// ONE slot reservation per query and tile: the four lanes of a quad share the query, so their counts are summed
			const uint32_t cnt = (uint32_t) __popcll(pass);
			uint32_t	   incl = cnt;
#pragma unroll
			for (uint32_t off = 1; off < 4; off <<= 1)
			{
				const uint32_t v = __shfl_up_sync(kFull, incl, off, 4);
				if (quad >= off) incl += v;
			}
			const uint32_t total = __shfl_sync(kFull, incl, 3, 4);
			uint32_t	   first = 0;
			if (quad == 0 && total != 0u) first = atomicAdd(&p.cand_n[q], total);
			first = __shfl_sync(kFull, first, 0, 4) + incl - cnt;
			if (pass != 0ull)
			{
#pragma unroll
				for (uint32_t i = 0; i < kUmmaTR / 8; i++)
#pragma unroll
					for (uint32_t b = 0; b < 2; b++)
						if (pass & (1ull << (2 * i + b)))
						{
							const uint32_t slot = first + (uint32_t) __popcll(pass & ((1ull << (2 * i + b)) - 1ull));
							if (slot < p.cap)
							{
								p.cand_rows[(size_t) q * p.cap + slot] = p.r0 + row_rel0 + 8u * i + 2u * quad + b;
								p.cand_s[(size_t) q * p.cap + slot] = d[4 * i + 2 * h + b];
							}
						}
			}
		}
	}
}
#endif	// PGEMB_HOST_EMULATION

// ---------------------------------------------------------------------------------------------------------------------
// Re-scoring + selection.  One CTA (4 warps) per query.
//   phase A  all 4 warps: every listed candidate is re-scored with the reference-exact arithmetic, ONE lane per candidate
//            (the lane owns all accumulator chains of its pair and reads the row with 16-byte loads: 128 rows in flight per
//            query -- the loop is a chain of dependent L2/HBM round trips, so rows in flight is what counts).  Measured
//            alternative, dropped: staging the rows through shared memory in column blocks with coalesced cp.async pieces
//            (fewer LSU wavefronts) -- 7.7 instead of 6.7 ms per 1024 x 1M scan: more instructions, fewer resident CTAs.  Candidates that the
//            chunk-start threshold already excludes, and deleted rows, are skipped.  The exact distance replaces the product in
//            the candidate list (cand_s), a dead entry gets bit 31 of its row id.  Every re-scored pair CHECKS the assumed
//            error bound (tripwire).
//   phase B  warp 0 folds the (dist,label) pairs into the running k smallest exactly like scan_select_kernel and refreshes the
//            query's filter constants for the next chunk.
// A query whose list overflowed is handled by warp 0 alone: every row of the chunk is re-scored (exact, slow, still correct).
// counters: [0] candidates re-scored, [1] error-bound violations (tripwire), [2] queries whose list overflowed.
// ---------------------------------------------------------------------------------------------------------------------
template <int METRIC>
__global__ void __launch_bounds__(128) scan_rescore_kernel(const float *__restrict__ vectors, uint32_t row_f, uint32_t dim, const float *__restrict__ vnorm2,
														   const float *__restrict__ queries, uint32_t q_stride, const float *__restrict__ qnorm2,
														   const uint64_t *__restrict__ labels, uint32_t nq, uint32_t r0, uint32_t nr, uint32_t k, float rel,
														   uint32_t *__restrict__ cand_rows, float *__restrict__ cand_s, uint32_t *__restrict__ cand_n, uint32_t cap,
														   uint32_t *__restrict__ top_d, uint64_t *__restrict__ top_l, uint32_t *__restrict__ top_n,
														   uint32_t *__restrict__ tmp_d, uint64_t *__restrict__ tmp_l, float2 *__restrict__ qconst,
														   uint32_t *__restrict__ counters)
{
	static_assert(METRIC == M_L2 || METRIC == M_COS, "the filter needs a bilinear form");
	__shared__ uint32_t cd[kScanCand];
	__shared__ uint64_t cl[kScanCand];
	// the running top-k lives in shared memory while the kernel works on it (k <= kTopSmem; larger k stays in global memory): the
	// rank-by-counting merge reads every entry (n + nc) times -- from L2 that was as long as the re-scoring itself
	constexpr uint32_t kTopSmem = 256;
	__shared__ uint32_t top_d_s[2 * kTopSmem];
	__shared__ uint64_t top_l_s[2 * kTopSmem];
	const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const uint32_t q = blockIdx.x;
	if (q >= nq) return;
	const bool top_in_smem = k <= kTopSmem;
	uint32_t *gtd = top_d + (size_t) q * k;
	uint64_t *gtl = top_l + (size_t) q * k;
	uint32_t *td = top_in_smem ? top_d_s : gtd, *sd = top_in_smem ? top_d_s + kTopSmem : tmp_d + (size_t) q * k;
	uint64_t *tl = top_in_smem ? top_l_s : gtl, *sl = top_in_smem ? top_l_s + kTopSmem : tmp_l + (size_t) q * k;
	uint32_t  n = top_n[q];
	// Read by every warp BEFORE the barrier below: warp 0 resets cand_n[q] (and rewrites top_n[q]) when it is done, and on the
	// overflow path it gets there without another barrier -- a warp that read the list length after that would take the other
	// branch and wait at a barrier nobody else reaches (found by the emulator's fuzz campaign on a loaded host).
	const uint32_t listed = cand_n[q];
	if (top_in_smem)
		for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
		{
			top_d_s[i] = gtd[i];
			top_l_s[i] = gtl[i];
		}
	__syncthreads();
	const float	  *qp = queries + (size_t) q * q_stride;
	const float	   qn = qnorm2[q];
	const bool	   overflow = listed > cap;
	float2		   qc = filter_qconst<METRIC>(qn, n < k ? INFINITY : o2f(td[k - 1]), rel);
	uint32_t	  *crow = cand_rows + (size_t) q * cap;
	float		  *cs = cand_s + (size_t) q * cap;
	uint32_t	   n_resc = 0;

	// ---- phase B state (used by warp 0 only) ------------------------------------------------------------------------------
	__shared__ float2 qc_s;	 // the filter constants all warps test with: refreshed by warp 0 after every slice it folds
	uint32_t		  nc = 0;
	const uint32_t	  lt = (1u << lane) - 1u;
	auto less = [](uint32_t d1, uint64_t l1, uint32_t d2, uint64_t l2) { return d1 < d2 || (d1 == d2 && l1 < l2); };
	auto merge = [&]() {
		// rank every element of top (n) and cand (nc) in their union; keep ranks < k  (as scan_select_kernel)
		__syncwarp();
		const uint32_t total = n + nc;
		for (uint32_t i = lane; i < total; i += 32)
		{
			const bool	   from_top = i < n;
			const uint32_t d = from_top ? td[i] : cd[i - n];
			const uint64_t l = from_top ? tl[i] : cl[i - n];
			uint32_t	   rank = 0;
			for (uint32_t j = 0; j < n; j++) rank += (j != i && (less(td[j], tl[j], d, l) || (!less(d, l, td[j], tl[j]) && j < i))) ? 1u : 0u;
			for (uint32_t j = 0; j < nc; j++)
			{
				const uint32_t jj = n + j;
				rank += (jj != i && (less(cd[j], cl[j], d, l) || (!less(d, l, cd[j], cl[j]) && jj < i))) ? 1u : 0u;
			}
			if (rank < k) { sd[rank] = d; sl[rank] = l; }
		}
		__syncwarp();
		n = total < k ? total : k;
		for (uint32_t i = lane; i < n; i += 32) { td[i] = sd[i]; tl[i] = sl[i]; }
		nc = 0;
		__syncwarp();
	};
	auto offer = [&](bool have, uint32_t d, uint64_t l) {
		const bool	   take = have && ((n < k) || less(d, l, td[k - 1], tl[k - 1]));
		const uint32_t m = __ballot_sync(0xffffffffu, take);
		if (m)
		{
			if (nc + (uint32_t) __popc(m) > kScanCand) merge();
			if (take)
			{
				const uint32_t at = nc + __popc(m & lt);
				cd[at] = d;
				cl[at] = l;
			}
			nc += __popc(m);
			// the first k candidates establish the threshold: merge them at once
			if (n < k && nc >= k) merge();
		}
	};
	if (!overflow)
	{
		// The list is taken in slices of 512: all warps re-score a slice (phase A), warp 0 folds it (phase B) and publishes the
		// tightened threshold, so later slices skip what can no longer matter -- the order inside the list is arbitrary
		// (atomicAdd order of the filter kernel), any order gives the same top-k.
		constexpr uint32_t kSlice = 512;
		if (threadIdx.x == 0) qc_s = qc;
		__syncthreads();
		for (uint32_t s0 = 0; s0 < listed; s0 += kSlice)
		{
			const uint32_t s1 = min(listed, s0 + kSlice);
			const float2   qcur = qc_s;
			// ---- phase A: one lane per candidate --------------------------------------------------------------------------
			for (uint32_t base = s0; base < s1; base += 128)
			{
				const uint32_t e = base + threadIdx.x;
				const bool	   have = e < s1;
				const uint32_t row = crow[have ? e : s0] & 0x7fffffffu;	// (entry s0 may already carry its dead mark; idle lanes only shadow it)
				const float	   s = cs[have ? e : s0];
				const float	   vn = vnorm2[row];
				bool		   alive = have && ((labels[row] >> 48) & 1ull) == 0;
				if (alive) alive = filter_pass<METRIC>(s, qcur, filter_rconst<METRIC>(vn));
				if (__any_sync(0xffffffffu, alive))
				{
					// all lanes run the same code (full-mask shuffles inside); lanes without a live candidate compute and drop
					const float dex = distance_exact<METRIC, 1>(qp, vectors + (size_t) row * row_f, (int) dim, qn, vn, 0);
					if (alive)
					{
						float approx, slack;
						filter_approx<METRIC>(s, qn, vn, rel, &approx, &slack);
						const float ex = (METRIC == M_COS) ? dex : dex * dex;
						if (fabsf(ex - approx) > slack * 1.5f + 1e-6f * fabsf(ex)) atomicAdd(&counters[1], 1u);
						cs[e] = __uint_as_float(f2o(dex));
						n_resc++;
					}
				}
				if (have && !alive) crow[e] = row | 0x80000000u;
			}
			__syncthreads();
			// ---- phase B: warp 0 folds the slice ----------------------------------------------------------------------------
			if (w == 0)
			{
				for (uint32_t base = s0; base < s1; base += 32)
				{
					const uint32_t e = base + lane;
					bool		   have = e < s1;
					uint32_t	   row = 0, d = 0;
					uint64_t	   l = 0;
					if (have)
					{
						row = crow[e];
						have = (row & 0x80000000u) == 0u;
						if (have)
						{
							d = __float_as_uint(cs[e]);
							l = labels[row];
						}
					}
					offer(have, d, l);
				}
				if (nc) merge();
				if (lane == 0) qc_s = filter_qconst<METRIC>(qn, n < k ? INFINITY : o2f(td[k - 1]), rel);
			}
			__syncthreads();
		}
		if (w != 0)
		{
			if (n_resc) atomicAdd(&counters[0], n_resc);
			return;
		}
	}
	else
	{
		if (w != 0) return;
		// the list overflowed: every row of the chunk, 32 at a time, one lane per row (warp 0 alone)
		for (uint32_t base = 0; base < nr; base += 32)
		{
			const uint32_t e = base + lane;
			const uint32_t row = r0 + (e < nr ? e : nr - 1);
			const uint64_t l = labels[row];
			const bool	   have = e < nr && ((l >> 48) & 1ull) == 0;
			const float	   dex = distance_exact<METRIC, 1>(qp, vectors + (size_t) row * row_f, (int) dim, qn, vnorm2[row], 0);
			if (have) n_resc++;
			offer(have, f2o(dex), l);
		}
	}
	if (nc) merge();
	if (top_in_smem)
	{
		__syncwarp();
		for (uint32_t i = lane; i < n; i += 32)
		{
			gtd[i] = td[i];
			gtl[i] = tl[i];
		}
	}
	if (lane == 0)
	{
		top_n[q] = n;
		cand_n[q] = 0;
		qconst[q] = filter_qconst<METRIC>(qn, n < k ? INFINITY : o2f(td[k - 1]), rel);
		if (overflow) atomicAdd(&counters[2], 1u);
	}
	if (n_resc) atomicAdd(&counters[0], n_resc);
}

// initial filter constants (nothing selected yet: T = +inf, nothing is discarded) and empty candidate lists
template <int METRIC>
__global__ void scan_qconst_init_kernel(const float *__restrict__ qnorm2, uint32_t nq, float rel, float2 *__restrict__ qconst, uint32_t *__restrict__ cand_n)
{
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= nq) return;
	qconst[q] = filter_qconst<METRIC>(qnorm2[q], INFINITY, rel);
	cand_n[q] = 0;
}

#ifdef PGEMB_HOST_EMULATION
// Host stand-in for scan_filter_wgmma_kernel (tests/emu only): the same predicate on a product whose operands are cut to
// TF32 (10 mantissa bits, truncation) and, with PGEMB_EMU_GEMM_ERR_PPM = x, pushed by +-x ppm of |q||v|: truncation + push up to
// 90 % of the assumed bound must still give exact results, 4x the bound must trip the tripwire.  (The truncation alone can use
// 2 * 2^-10 of the bound -- one-dimensional rows do -- so a test's push has to leave that much room.)
template <int METRIC>
inline void scan_filter_emulated(const float *queries, uint32_t q_stride, const float *vectors, uint32_t row_f, uint32_t dim, float rel,
								 const float *qnorm2, const ScanFilterParams &p)
{
	// PGEMB_EMU_GEMM_ERR_PPM: every product is pushed by +-ppm * 1e-6 * |q||v| (sign pseudo-random per pair)
	const char *pe = getenv("PGEMB_EMU_GEMM_ERR_PPM");
	const float perturb = pe ? (float) atof(pe) * 1e-6f : 0.0f;
	auto		cut = [](float x) {
		   union { float f; uint32_t u; } c;
		   c.f = x;
		   c.u &= 0xffffe000u;
		   return c.f;
	};
	for (uint32_t q = 0; q < p.nq; q++)
		for (uint32_t j = 0; j < p.nr; j++)
		{
			const uint32_t row = p.r0 + j;
			const float	  *a = queries + (size_t) q * q_stride, *b = vectors + (size_t) row * row_f;
			float		   s = 0.f;
			for (uint32_t i = 0; i < dim; i++) s += cut(a[i]) * cut(b[i]);
			if (perturb != 0.0f) s += (((q * 2654435761u + row * 40503u) >> 7) & 1u ? 1.0f : -1.0f) * perturb * sqrtf(qnorm2[q]) * sqrtf(p.vnorm2[row]);
			if (p.dbg_s)
			{
				p.dbg_s[(size_t) q * p.nr + j] = s;
				continue;
			}
			if (filter_pass<METRIC>(s, p.qconst[q], filter_rconst<METRIC>(p.vnorm2[row])))
			{
				const uint32_t slot = p.cand_n[q]++;
				if (slot < p.cap)
				{
					p.cand_rows[(size_t) q * p.cap + slot] = row;
					p.cand_s[(size_t) q * p.cap + slot] = s;
				}
			}
		}
}
#endif

}  // namespace pgemb
