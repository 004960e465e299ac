// search_kernel.cuh -- K3: persistent best-first traversal, one WARP per query slot.
//
// Replaces, per query, the reference's  hnsw_search -> searchKnn -> searchBaseLayer  chain
// (hnswalg.cpp:256-277, :234-252, :42-114) including its innermost loop
// begin_read -> hnsw_dist_func -> end_read (hnswalg.cpp:95-97) with results identical to the
// reference (same ids, same order, same distances bit for bit).
//
// Structure per hop (one iteration of `while (!candidateSet.empty())`, hnswalg.cpp:67-112):
//   pop      nearest unexpanded candidate; ties: larger id first (pair(-dist,id) max-heap, :53,:69)
//   expand   its link list [count, ids...] (:76-77) -- normally already in shared memory, prefetched by
//            bulk TMA during the previous hop's queue update -- and test-and-set of the visited set (:92-93)
//   gather   K1: the unvisited neighbours' vectors are pulled HBM -> shared memory, one 1-D bulk TMA copy
//            per row (cp.async.bulk + mbarrier, L2 evict-first, a ring of 8 rows from the CTA's pool), scored with
//            the reference's exact fp32 summation order, 4 lanes per row
//   update   K2: warp-level top-ef queue update that is EQUIVALENT to the reference's sequential
//            push/pop loop (:99-108), exact distance ties included -- see "sequential equivalence".
//
// Sequential equivalence (proved in DESIGN.md section 5, model-checked in tests/test_batch_semantics.py).
// The reference scores the unvisited neighbours x_1..x_n in list order and accepts x_k iff
// `topResults.size() < ef || topResults.top().first > d_k`.  With R = current results:
//     accept(x_k)  <=>  #{ y in R u {x_1..x_{k-1}} : dist(y) <= d_k } < ef
// (rejected earlier items may be counted: they never change the ef-th smallest distance).  The new
// result set is the ef smallest (dist,id) pairs of R u accepted.  candidateSet = unexpanded members
// of the result set, plus ("overflow") accepted-but-evicted entries whose distance still EQUALS the
// current worst result distance -- only those can ever be popped before the `> lowerBound` break
// (:70).  Overflow entries exist only under exact distance ties; they are bounded by ef-1 and kept
// in a per-slot global buffer.
//
// Visited set: an open-addressing table (atomicCAS at L2, kept resident with an L2 persistence window)
// that migrates to the exact N-bit bitmap before it passes half full; both are reset in O(visited).
//
// One warp = one query slot; a CTA (one per SM) holds W slots that share a pool of R row rings (RingPool):
// a slot needs a ring only while it gathers+scores, so 12 slots time-share 6 rings in the 227 KB of an SM
// at dim 768 and overlap each other's dependent-latency phases (pop -> links -> visited -> rows).
// The only CTA-wide barrier is the one after the pool is initialised.
#pragma once
#include "common.cuh"
#include "dist_exact.cuh"
#include "search_config.h"  // RingPool, SearchConfig (host-side layout)

namespace pgemb {

struct SearchParams
{
	// index (HBM, SoA; DESIGN.md section 3)
	const float	   *vectors;	 // [n][row_f] f32, rows 16-B aligned, zero padded
	const uint32_t *links;		 // [n][link_stride] u32: [count, ids...]
	const uint64_t *labels;		 // [n]
	const float	   *norms;		 // [n] squared norms in cosine lane order (cosine only)
	uint32_t		n_items, dim, row_f, link_stride, maxM, entry;
	// queries
	const float	   *queries;	 // [nq][q_stride] or NULL
	const uint32_t *query_ids;	 // [nq] stored nodes used as queries (bind path) or NULL
	uint32_t		nq, q_stride, ef;
	uint32_t		raw_mode;	 // 1: emit searchBaseLayer's (dist,id) list (no label lookup / deleted filter)
	// outputs (any may be NULL except n_out)
	uint64_t *labels_out;		 // [nq][ef]
	float	 *dists_out;		 // [nq][ef]
	uint32_t *ids_out;			 // [nq][ef]
	int32_t	 *n_out;			 // [nq]
	uint32_t *stats_out;		 // [nq][4]: distance evals, expansions, link words, overflow high-water
	uint32_t *exp_out;			 // [nq][exp_cap] ids of the expanded nodes in order, or NULL (exact parallel build)
	uint32_t  exp_cap;
	uint32_t *exp_n_out;		 // [nq] number of expansions (may exceed exp_cap: the list is then incomplete)
	// per-slot workspace
	uint32_t	 *visited;		 // [slots][vis_words]   exact bitmap (fallback / small indexes)
	uint32_t	 *vlog;			 // [slots][vlog_cap]    table positions (hash mode) or ids (bitmap mode) to reset
	uint64_t	 *ovf;			 // [slots][ef]
	uint64_t	 *res_g;		 // [slots][2 * ef] result buffers in global memory (search_kernel<..., RESG = true> only: huge ef)
	uint32_t	 *vhash;		 // [slots][vh_size]     open-addressing visited set, 0xffffffff = empty
	uint32_t	  vis_words, vlog_cap;
	uint32_t	  vh_size, vh_shift;  // vh_size = 2^k entries (0: bitmap only), hash = (id * 2654435761) >> vh_shift
	uint32_t	  off_vhs, vhs_entries;	 // latency mode: the hash set lives in the CTA's shared memory (2^k entries, 0 = use vhash)
	unsigned int *counter;		 // work-stealing query counter
	const unsigned int *avail;	 // optional: number of queries whose data has landed (host API streams them in while the kernel runs)
	int			 *error_flag;	 // sticky: 1 = bad link id / count, 2 = overflow buffer exceeded
	// shared-memory layout (bytes from the dynamic smem base)
	// A CTA = W query slots (warps) sharing a POOL of `rings` row rings: a slot needs a ring only while it
	// gathers+scores (about half of a hop), so rings -- the shared-memory-hungry resource that bounds
	// bytes in flight -- are time-multiplexed between more slots than would fit with one ring each.
	uint32_t rings, ring_bytes, row_smem, row_bytes, qt_stride;
	uint32_t prefetch_links;
	uint32_t visited_pairs;	 // latency mode, 1: the ids of every link list are distinct -> both halves of a list are test-and-set concurrently
	uint32_t off_pool, off_ring, off_priv, priv_bytes;	 // CTA-level
	uint32_t off_qt, off_qtail, off_res, off_hopkey, off_acckey, off_evict, off_hopid, off_pf, off_pfbar;  // inside a slot's private block
};


// copy the shared-memory layout chosen by make_search_config into the kernel parameters
inline void apply_config(SearchParams &p, const SearchConfig &cfg, uint32_t row_f)
{
	p.off_vhs = cfg.off_vhs;
	p.vhs_entries = cfg.vhs_entries;
	p.rings = cfg.rings;
	p.ring_bytes = cfg.ring_bytes;
	p.off_pool = cfg.off_pool;
	p.off_priv = cfg.off_priv;
	p.priv_bytes = cfg.priv_bytes;
	p.off_pfbar = cfg.off_pfbar;
	p.row_smem = cfg.row_smem;
	p.row_bytes = row_f * 4u;
	p.qt_stride = cfg.qt_stride;
	p.off_qt = cfg.off_qt;
	p.off_qtail = cfg.off_qtail;
	p.off_pf = cfg.off_pf;
	p.off_ring = cfg.off_ring;
	p.off_res = cfg.off_res;
	p.off_hopkey = cfg.off_hopkey;
	p.off_acckey = cfg.off_acckey;
	p.off_evict = cfg.off_evict;
	p.off_hopid = cfg.off_hopid;
}

constexpr uint32_t kNone = 0xffffffffu;

// ---- 4 lanes per row, query pre-transposed -----------------------------------------------------------
// The query is stored lane-major in shared memory (qT): thread `sub` finds the values of ITS accumulator
// chain(s) for four consecutive steps in one 16-byte word, so a step costs one LDS.32 of the row instead
// of two loads (LDS issue, ~4 cycles per instruction per warp, is what bounds this loop).
//   cosine / manhattan:  qT[sub*QS + i]        = q[4i + sub]
//   L2 (2 chains/thread): qT[sub*QS + 4b + ..] = { q[16b+2s], q[16b+2s+1], q[16b+8+2s], q[16b+8+2s+1] }
template <int METRIC>
__device__ __forceinline__ float score_row4(const float *__restrict__ qts, const float *__restrict__ rowp, int sub, int main_n,
											const float *__restrict__ q_tail, int dim, float qn, float vn)
{
	if (METRIC == M_L2)
	{
		float		 S0 = 0.f, S1 = 0.f;
		const int	 nb = main_n >> 4;
		const float *vp = rowp + 2 * sub;
		// two 16-float blocks per iteration, the loads of the next pair interleaved with the arithmetic of the
		// current one (same reasoning as the cosine loop below)
#define PGEMB_L2_BLOCK(QQ, YA, YB)                                                                      \
	{                                                                                                   \
		const float d00 = __fsub_rn(QQ.x, YA.x), d10 = __fsub_rn(QQ.z, YB.x);                           \
		const float d01 = __fsub_rn(QQ.y, YA.y), d11 = __fsub_rn(QQ.w, YB.y);                           \
		S0 = __fadd_rn(S0, __fadd_rn(__fmul_rn(d00, d00), __fmul_rn(d10, d10)));                        \
		S1 = __fadd_rn(S1, __fadd_rn(__fmul_rn(d01, d01), __fmul_rn(d11, d11)));                        \
	}
		int		  b = 0;
		const int npair = nb >> 1;
		if (npair > 0)
		{
			float4 qa = *reinterpret_cast<const float4 *>(qts), qb = *reinterpret_cast<const float4 *>(qts + 4);
			float2 a0 = *reinterpret_cast<const float2 *>(vp), a1 = *reinterpret_cast<const float2 *>(vp + 8);
			float2 b0 = *reinterpret_cast<const float2 *>(vp + 16), b1 = *reinterpret_cast<const float2 *>(vp + 24);
#pragma unroll 1
			for (int it = 1; it < npair; it++)
			{
				const float *vn_ = vp + 32 * it;
				const float4 nqa = *reinterpret_cast<const float4 *>(qts + 8 * it);
				const float2 na0 = *reinterpret_cast<const float2 *>(vn_);
				const float2 na1 = *reinterpret_cast<const float2 *>(vn_ + 8);
				PGEMB_L2_BLOCK(qa, a0, a1)
				const float4 nqb = *reinterpret_cast<const float4 *>(qts + 8 * it + 4);
				const float2 nb0 = *reinterpret_cast<const float2 *>(vn_ + 16);
				const float2 nb1 = *reinterpret_cast<const float2 *>(vn_ + 24);
				PGEMB_L2_BLOCK(qb, b0, b1)
				qa = nqa; qb = nqb; a0 = na0; a1 = na1; b0 = nb0; b1 = nb1;
			}
			PGEMB_L2_BLOCK(qa, a0, a1)
			PGEMB_L2_BLOCK(qb, b0, b1)
			b = npair << 1;
		}
		for (; b < nb; b++)
		{
			const float4 qq = *reinterpret_cast<const float4 *>(qts + 4 * b);
			const float2 ya = *reinterpret_cast<const float2 *>(vp + 16 * b);
			const float2 yb = *reinterpret_cast<const float2 *>(vp + 16 * b + 8);
			PGEMB_L2_BLOCK(qq, ya, yb)
		}
#undef PGEMB_L2_BLOCK
		float full[8];
#pragma unroll
		for (int l = 0; l < 8; l++) full[l] = __shfl_sync(kFull, (l & 1) ? S1 : S0, l >> 1, 4);
		float res = hsum4(__fadd_rn(full[0], full[4]), __fadd_rn(full[1], full[5]), __fadd_rn(full[2], full[6]), __fadd_rn(full[3], full[7]));
		res = l2_tail_exact(res, q_tail, rowp + main_n, dim - main_n);
		return __fsqrt_rn(res);
	}
	else
	{
		constexpr int TERM = (METRIC == M_COS) ? 0 : 1;
		float		  s = 0.f;
		const int	  n4 = main_n >> 2;
		const float	 *vp = rowp + sub;
		int			  k = 0;
		// Software-pipelined by hand: the chain `s` is one dependent FADD per step (4-cycle latency) and a
		// warp can issue one LDS every ~4 cycles, so the loads of the NEXT 8 steps are interleaved with
		// the adds of the CURRENT 8 steps; left to itself ptxas issues 10 loads, stalls on the first
		// product, then runs the 8-add chain back to back (~115 cycles per 8 steps instead of ~45).
		const int nit = n4 >> 3;
		if (nit > 0)
		{
			const float4 *qp = reinterpret_cast<const float4 *>(qts);
			float4		  qa = qp[0], qb = qp[1];
			float		  v0 = vp[0], v1 = vp[4], v2 = vp[8], v3 = vp[12], v4 = vp[16], v5 = vp[20], v6 = vp[24], v7 = vp[28];
#pragma unroll 1
			for (int it = 1; it < nit; it++)
			{
				const float *vn_ = vp + 32 * it;
				const float4 na = qp[2 * it];
				s = __fadd_rn(s, term4<TERM>(qa.x, v0));
				const float w0 = vn_[0];
				s = __fadd_rn(s, term4<TERM>(qa.y, v1));
				const float w1 = vn_[4];
				s = __fadd_rn(s, term4<TERM>(qa.z, v2));
				const float w2 = vn_[8];
				s = __fadd_rn(s, term4<TERM>(qa.w, v3));
				const float w3 = vn_[12];
				const float4 nb = qp[2 * it + 1];
				s = __fadd_rn(s, term4<TERM>(qb.x, v4));
				const float w4 = vn_[16];
				s = __fadd_rn(s, term4<TERM>(qb.y, v5));
				const float w5 = vn_[20];
				s = __fadd_rn(s, term4<TERM>(qb.z, v6));
				const float w6 = vn_[24];
				s = __fadd_rn(s, term4<TERM>(qb.w, v7));
				const float w7 = vn_[28];
				qa = na; qb = nb;
				v0 = w0; v1 = w1; v2 = w2; v3 = w3; v4 = w4; v5 = w5; v6 = w6; v7 = w7;
			}
			s = __fadd_rn(s, term4<TERM>(qa.x, v0));
			s = __fadd_rn(s, term4<TERM>(qa.y, v1));
			s = __fadd_rn(s, term4<TERM>(qa.z, v2));
			s = __fadd_rn(s, term4<TERM>(qa.w, v3));
			s = __fadd_rn(s, term4<TERM>(qb.x, v4));
			s = __fadd_rn(s, term4<TERM>(qb.y, v5));
			s = __fadd_rn(s, term4<TERM>(qb.z, v6));
			s = __fadd_rn(s, term4<TERM>(qb.w, v7));
			k = nit << 3;
		}
		for (; k < n4; k++) s = __fadd_rn(s, term4<TERM>(qts[k], vp[4 * k]));
		const float f0 = __shfl_sync(kFull, s, 0, 4), f1 = __shfl_sync(kFull, s, 1, 4);
		const float f2 = __shfl_sync(kFull, s, 2, 4), f3 = __shfl_sync(kFull, s, 3, 4);
		float		res = hsum4(f0, f1, f2, f3);
		for (int e = main_n; e < dim; e++) res = __fadd_rn(res, term4<TERM>(q_tail[e - main_n], rowp[e]));
		if (METRIC == M_COS) return (sub == 0) ? cosine_finish(res, qn, vn) : res;
		return res;
	}
}

// ---- L2 with 8 lanes per row: every lane owns ONE of the reference's eight accumulator lanes -----------------
// Used for long rows (1536-d: 6 KB): a ring then holds 4 rows instead of 8, so twice as many rings fit and the
// slots/rings balance of the 768-d configuration is kept.  qT8[sub*QS + 2b + {0,1}] = { q[16b+sub], q[16b+8+sub] }.
__device__ __forceinline__ float score_row8_l2(const float *__restrict__ qts, const float *__restrict__ rowp, int sub, int main_n,
												const float *__restrict__ q_tail, int dim)
{
	float		 S = 0.f;
	const int	 nb = main_n >> 4;
	const float *vp = rowp + sub;
	// Four 16-float blocks per iteration, software-pipelined by hand like score_row4: the loads of the NEXT four blocks
	// (2 x LDS.128 of the query run -- qT8 runs are padded to 16 bytes -- and 8 x LDS.32 of the row) are interleaved with the
	// arithmetic of the current four; left to itself ptxas issues all loads of an unrolled batch, stalls on the first
	// difference and then runs the dependent adds back to back.
#define PGEMB_L2_STEP8(QX, QY, YA, YB)                                               \
	{                                                                                \
		const float d0_ = __fsub_rn(QX, YA), d1_ = __fsub_rn(QY, YB);                \
		S = __fadd_rn(S, __fadd_rn(__fmul_rn(d0_, d0_), __fmul_rn(d1_, d1_)));       \
	}
	int		  b = 0;
	const int nquad = nb >> 2;
	if (nquad > 0)
	{
		const float4 *qp = reinterpret_cast<const float4 *>(qts);
		float4		  qa = qp[0], qb = qp[1];
		float		  a0 = vp[0], a1 = vp[8], a2 = vp[16], a3 = vp[24], a4 = vp[32], a5 = vp[40], a6 = vp[48], a7 = vp[56];
#pragma unroll 1
		for (int it = 1; it < nquad; it++)
		{
			const float *vn_ = vp + 64 * it;
			const float4 nqa = qp[2 * it];
			const float	 w0 = vn_[0], w1 = vn_[8];
			PGEMB_L2_STEP8(qa.x, qa.y, a0, a1)
			const float w2 = vn_[16], w3 = vn_[24];
			PGEMB_L2_STEP8(qa.z, qa.w, a2, a3)
			const float4 nqb = qp[2 * it + 1];
			const float	 w4 = vn_[32], w5 = vn_[40];
			PGEMB_L2_STEP8(qb.x, qb.y, a4, a5)
			const float w6 = vn_[48], w7 = vn_[56];
			PGEMB_L2_STEP8(qb.z, qb.w, a6, a7)
			qa = nqa; qb = nqb;
			a0 = w0; a1 = w1; a2 = w2; a3 = w3; a4 = w4; a5 = w5; a6 = w6; a7 = w7;
		}
		PGEMB_L2_STEP8(qa.x, qa.y, a0, a1)
		PGEMB_L2_STEP8(qa.z, qa.w, a2, a3)
		PGEMB_L2_STEP8(qb.x, qb.y, a4, a5)
		PGEMB_L2_STEP8(qb.z, qb.w, a6, a7)
		b = nquad << 2;
	}
	for (; b < nb; b++)
	{
		const float2 qq = *reinterpret_cast<const float2 *>(qts + 2 * b);
		PGEMB_L2_STEP8(qq.x, qq.y, vp[16 * b], vp[16 * b + 8])
	}
#undef PGEMB_L2_STEP8
	float full[8];
#pragma unroll
	for (int l = 0; l < 8; l++) full[l] = __shfl_sync(kFull, S, l, 8);
	float res = hsum4(__fadd_rn(full[0], full[4]), __fadd_rn(full[1], full[5]), __fadd_rn(full[2], full[6]), __fadd_rn(full[3], full[7]));
	res = l2_tail_exact(res, q_tail, rowp + main_n, dim - main_n);
	return __fsqrt_rn(res);
}

template <int METRIC, int TPR>
__device__ __forceinline__ float score_row(const float *__restrict__ qts, const float *__restrict__ rowp, int sub, int main_n,
										   const float *__restrict__ q_tail, int dim, float qn, float vn)
{
	static_assert(TPR == 4 || (TPR == 8 && METRIC == M_L2), "8 lanes per row exist for L2 only (8 accumulator lanes)");
	if (TPR == 8) return score_row8_l2(qts, rowp, sub, main_n, q_tail, dim);
	return score_row4<METRIC>(qts, rowp, sub, main_n, q_tail, dim, qn, vn);
}

// ---- latency mode (COOP) -------------------------------------------------------------------------------
// With fewer queries than SMs a query has a whole SM to itself, and the per-hop latency -- not bytes in
// flight -- is what a caller of hnsw_search() waits for.  The CTA then runs ONE slot: warp 0 owns the
// traversal exactly as in the throughput kernel, and all warps (each with its own ring and mbarrier) gather
// and score one 8-row group of the hop at the same time, so a hop costs one DRAM round trip + one row
// scoring instead of ceil(n/8) of them back to back.  Two named barriers bracket the shared phase; every
// row is scored by the same score_row4 (same bits).
#ifndef PGEMB_HOST_EMULATION  // tests/emu supplies the host version
__device__ __forceinline__ void coop_bar(int id, uint32_t nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
#endif

template <int METRIC, int TPR>
__device__ __forceinline__ void coop_gather(const SearchParams &p, unsigned char *ring, uint64_t *rbar, uint32_t &rpar, uint32_t warp,
											uint32_t nwarps, uint32_t n, const uint32_t *hop_id, uint64_t *hop_key, const float *qT,
											const float *q_tail, float qn, int main_n, uint64_t pol_stream)
{
	const uint32_t lane = threadIdx.x & 31;
	constexpr int  kRows = 32 / TPR;
	const int	   row_in_stage = lane / TPR;
	const int	   sub = lane % TPR;
	const uint32_t G = (n + kRows - 1) / kRows;
	const float	  *qts = qT + sub * p.qt_stride;
	for (uint32_t g = warp; g < G; g += nwarps)
	{
		const uint32_t rows = min((uint32_t) kRows, n - g * kRows);
		if (lane == 0) mbar_arrive_expect_tx(rbar, rows * p.row_bytes);
		__syncwarp();
		if (lane < rows)
		{
			const uint32_t id = hop_id[g * kRows + lane];
			tma_load_1d(ring + (size_t) lane * p.row_smem, p.vectors + (size_t) id * p.row_f, p.row_bytes, rbar, pol_stream);
		}
		const uint32_t k = g * kRows + row_in_stage;
		const uint32_t kk = min(k, n - 1);
		const uint32_t my_id = hop_id[kk];
		float		   vn = 1.0f;
		if (METRIC == M_COS) vn = p.norms[my_id];
		mbar_wait(rbar, rpar);
		rpar ^= 1u;
		const float *rowp = reinterpret_cast<const float *>(ring + (size_t) row_in_stage * p.row_smem);
		const float	 d = score_row<METRIC, TPR>(qts, rowp, sub, main_n, q_tail, (int) p.dim, qn, vn);
		if (sub == 0 && k < n) hop_key[k] = make_key(d, my_id);
		__syncwarp();
	}
}

// RESG: the two result buffers of a slot live in global memory (p.res_g) instead of its shared-memory block -- the variant
// plan_search (capi.cu) falls back to when 2 x ef keys no longer fit a CTA, so that the caller's efSearch doubling (embedding.c:334)
// never fails before ef reaches the index size.  Same code path otherwise (the queue update then runs at L2 latency).
template <int METRIC, bool COOP, int TPR = 4, bool RESG = false>
__global__ void __launch_bounds__(1024) search_kernel(const SearchParams p)
{
	constexpr int kRows = 32 / TPR;	 // rows per ring
	PGEMB_DYNAMIC_SMEM(smem, 128);
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t warp = threadIdx.x >> 5;
	const uint32_t slot = COOP ? blockIdx.x : blockIdx.x * (blockDim.x >> 5) + warp;
	RingPool	  *pool = reinterpret_cast<RingPool *>(smem + p.off_pool);
	unsigned char *ring_base = smem + p.off_ring;
	unsigned char *priv = smem + p.off_priv + (COOP ? 0 : (size_t) warp * p.priv_bytes);  // this slot's private block
	float		  *qT = reinterpret_cast<float *>(priv + p.off_qt);
	float		  *q_tail = reinterpret_cast<float *>(priv + p.off_qtail);
	uint64_t	  *res = RESG ? p.res_g + (size_t) slot * 2u * p.ef : reinterpret_cast<uint64_t *>(priv + p.off_res);	// two buffers of ef keys
	uint64_t	  *hop_key = reinterpret_cast<uint64_t *>(priv + p.off_hopkey);
	uint64_t	  *acc_key = reinterpret_cast<uint64_t *>(priv + p.off_acckey);
	uint64_t	  *evict_key = reinterpret_cast<uint64_t *>(priv + p.off_evict);
	uint32_t	  *hop_id = reinterpret_cast<uint32_t *>(priv + p.off_hopid);
	uint32_t	  *pf_links = reinterpret_cast<uint32_t *>(priv + p.off_pf);
	uint64_t	  *pf_bar = reinterpret_cast<uint64_t *>(priv + p.off_pfbar);

	const uint32_t lt = lanemask_lt();
	const int	   row_in_stage = lane / TPR;
	const int	   sub = lane % TPR;
	const uint32_t ef = p.ef;
	const int	   dim = (int) p.dim;
	const int	   main_n = main_len<METRIC>(dim);
	// latency mode keeps the open-addressing visited set in shared memory when the CTA has room for it: a hop's
	// test-and-set round then costs shared-memory atomics instead of L2 round trips
	const bool	   vh_shared = COOP && p.vhs_entries != 0u;
	const uint32_t H = vh_shared ? p.vhs_entries : p.vh_size;
	const uint32_t vh_shift = vh_shared ? (32u - (uint32_t) __popc(p.vhs_entries - 1u)) : p.vh_shift;
	uint32_t	  *vis = p.visited + (size_t) slot * p.vis_words;
	uint32_t	  *vlog = p.vlog + (size_t) slot * p.vlog_cap;
	uint64_t	  *ovf = p.ovf + (size_t) slot * ef;
	uint32_t	  *vh = vh_shared ? reinterpret_cast<uint32_t *>(smem + p.off_vhs) : p.vhash + (size_t) slot * H;
	const uint64_t pol_stream = l2_policy_evict_first();
	const uint64_t pol_keep = l2_policy_evict_last();
	constexpr uint32_t kEmpty = 0xffffffffu;

	if (threadIdx.x == 0)
	{
		pool->state = (1u << p.rings) - 1u;	// all free, all parities 0
		for (uint32_t b = 0; b < p.rings; b++)
		{
			mbar_init(&pool->bar[b], 1);
		}
	}
	if (vh_shared)
		for (uint32_t i = threadIdx.x; i < H; i += blockDim.x) vh[i] = 0xffffffffu;
	if (lane == 0 && (!COOP || warp == 0)) mbar_init(pf_bar, 1);
	fence_mbar_init();
	__syncthreads();		   // the only CTA-wide barrier: from here on the slots run independently
	uint32_t coop_par = 0;	   // COOP: phase parity of this warp's own ring barrier
	if (COOP && warp != 0)
	{
		// helper warp: score one row group per hop on command of the owner (warp 0)
		unsigned char *my_ring = ring_base + (size_t) warp * p.ring_bytes;
		for (;;)
		{
			coop_bar(1, blockDim.x);
			const uint32_t hn = *reinterpret_cast<volatile uint32_t *>(&pool->coop_n);
			if (hn == kNone) break;
			const float hq = *reinterpret_cast<volatile float *>(&pool->coop_qn);
			coop_gather<METRIC, TPR>(p, my_ring, &pool->bar[warp], coop_par, warp, blockDim.x >> 5, hn, hop_id, hop_key, qT, q_tail, hq, main_n, pol_stream);
			coop_bar(2, blockDim.x);
		}
		return;
	}
	uint32_t pf_parity = 0;	   // phase parity for the link prefetch barrier
	bool	 pf_inflight = false;
	uint32_t pf_id = kNone;

	for (;;)
	{
		uint32_t qi = 0;
		if (lane == 0) qi = atomicAdd(p.counter, 1u);
		qi = __shfl_sync(kFull, qi, 0);
		if (qi >= p.nq) break;
		if (p.avail)
		{
			// the batch is still being copied in by the DMA engine: wait until query qi is there
			// (bounded: a few seconds of polling -- a chunk takes < 1 ms over PCIe -- then the query is processed
			// anyway and the launch is flagged)
			if (lane == 0)
			{
				uint32_t spins = 0;
				while (*reinterpret_cast<const volatile unsigned int *>(p.avail) <= qi)
				{
					__nanosleep(500);
					if (++spins > (8u << 20))
					{
						*p.error_flag = 4;
						break;
					}
				}
			}
			__syncwarp();
		}

		// ---- stage the query: lane-major transposed copy + natural-order tail -------------------
		{
			const float *qsrc = p.query_ids ? p.vectors + (size_t) p.query_ids[qi] * p.row_f : p.queries + (size_t) qi * p.q_stride;
			// eight loads in flight per lane before the first dependent store (one DRAM round trip per 256 floats)
			for (int e0 = 0; e0 < dim; e0 += 256)
			{
				float v8[8];
#pragma unroll
				for (int j = 0; j < 8; j++)
				{
					const int e = e0 + j * 32 + (int) lane;
					v8[j] = (e < dim) ? __ldcg(qsrc + e) : 0.0f;  // L2 only: the batch may still be streaming in (avail)
				}
#pragma unroll
				for (int j = 0; j < 8; j++)
				{
					const int	e = e0 + j * 32 + (int) lane;
					const float v = v8[j];
					if (e >= dim)
						continue;
					if (e >= main_n)
						q_tail[e - main_n] = v;
					else if (METRIC == M_L2 && TPR == 8)
					{
						const int b = e >> 4, o = e & 15;
						qT[(o & 7) * p.qt_stride + 2 * b + (o >> 3)] = v;
					}
					else if (METRIC == M_L2)
					{
						const int b = e >> 4, o = e & 15, l = o & 7;
						qT[(l >> 1) * p.qt_stride + 4 * b + ((o >> 3) << 1) + (l & 1)] = v;
					}
					else
						qT[(e & 3) * p.qt_stride + (e >> 2)] = v;
				}
			}
		}
		__syncwarp();
		float qn = 0.0f;
		if (METRIC == M_COS)
		{
			// |q|^2 in the reference's lane order (distfunc.c:141), once per query instead of once per call
			float		 s = 0.f;
			const float *qts = qT + sub * p.qt_stride;
			for (int k = 0; k < (main_n >> 2); k++) s = __fadd_rn(s, __fmul_rn(qts[k], qts[k]));
			const float f0 = __shfl_sync(kFull, s, 0, 4), f1 = __shfl_sync(kFull, s, 1, 4);
			const float f2 = __shfl_sync(kFull, s, 2, 4), f3 = __shfl_sync(kFull, s, 3, 4);
			qn = hsum4(f0, f1, f2, f3);
			for (int e = main_n; e < dim; e++) qn = __fadd_rn(qn, __fmul_rn(q_tail[e - main_n], q_tail[e - main_n]));
		}
		if (COOP && lane == 0) pool->coop_qn = qn;

		int		 cur = 0;		// which res buffer is live
		uint32_t r = 0;			// results held (<= ef), ascending (dist,id)
		uint32_t ovf_n = 0, ovf_hw = 0;
		uint32_t logn = 0;
		uint32_t vmode = (H == 0) ? 1u : 0u;  // 0: hash set (log holds table positions), 1: bitmap (log holds ids)
		uint32_t st_dist = 0, st_hops = 0, st_words = 0;

		// ---- entry point (hnswalg.cpp:55-65): scored like a one-element hop ---------------------
		uint32_t n = 0;
		if (p.n_items > 0 && p.entry < p.n_items)
		{
			if (lane == 0)
			{
				hop_id[0] = p.entry;
				if (vmode == 0)
				{
					const uint32_t h = (p.entry * 2654435761u) >> vh_shift;
					vh[h] = p.entry;
					vlog[0] = h;
				}
				else
				{
					atomicOr(&vis[p.entry >> 5], 1u << (p.entry & 31));
					if (p.vlog_cap > 0) vlog[0] = p.entry;
				}
			}
			n = 1;
			logn = 1;
		}
		__syncwarp();

		for (;;)
		{
			if (n > 0)
			{
				// ================= K1: gather + score the n rows in hop_id[] ======================
				st_dist += n;
				if constexpr (COOP)
				{
					if (lane == 0) pool->coop_n = n;
					__syncwarp();
					coop_bar(1, blockDim.x);
					coop_gather<METRIC, TPR>(p, ring_base, &pool->bar[0], coop_par, 0, blockDim.x >> 5, n, hop_id, hop_key, qT, q_tail, qn, main_n, pol_stream);
					coop_bar(2, blockDim.x);
				}
				else
				{
				const uint32_t G = (n + kRows - 1) / kRows;
				// ---- take a ring from the CTA's pool (held for this hop's gather only) ----------------
				uint32_t rb = 0;  // low byte: ring index, bit 8: its barrier's phase parity
				if (lane == 0)
				{
					for (;;)
					{
						const uint32_t m = *reinterpret_cast<volatile uint32_t *>(&pool->state);
						if ((m & 0xffffu) != 0u)
						{
							const uint32_t b = (uint32_t) __ffs(m & 0xffffu) - 1u;
							if (atomicCAS(&pool->state, m, m & ~(1u << b)) == m)
							{
								rb = b | (((m >> (16u + b)) & 1u) << 8);
								break;
							}
						}
						else
							__nanosleep(100);
					}
					__threadfence_block();
				}
				rb = __shfl_sync(kFull, rb, 0);
				uint32_t rpar = (rb >> 8) & 1u;
				rb &= 0xffu;
				const uint32_t rpar0 = rpar;
				unsigned char *ring = ring_base + (size_t) rb * p.ring_bytes;
				uint64_t	  *rbar = &pool->bar[rb];
				auto		   issue = [&](uint32_t g) {
					  const uint32_t rows = min((uint32_t) kRows, n - g * kRows);
					  if (lane == 0) mbar_arrive_expect_tx(rbar, rows * p.row_bytes);
					  __syncwarp();
					  if (lane < rows)
					  {
						  const uint32_t id = hop_id[g * kRows + lane];
						  tma_load_1d(ring + (size_t) lane * p.row_smem, p.vectors + (size_t) id * p.row_f, p.row_bytes, rbar, pol_stream);
					  }
				};
				issue(0);
				const float *qts = qT + sub * p.qt_stride;
				for (uint32_t g = 0; g < G; g++)
				{
					const uint32_t k = g * kRows + row_in_stage;
					const uint32_t kk = min(k, n - 1);
					const uint32_t my_id = hop_id[kk];
					float		   vn = 1.0f;
					if (METRIC == M_COS) vn = p.norms[my_id];  // in flight while the rows land
					mbar_wait(rbar, rpar);
					rpar ^= 1u;
					const float *rowp = reinterpret_cast<const float *>(ring + (size_t) row_in_stage * p.row_smem);
					const float	 d = score_row<METRIC, TPR>(qts, rowp, sub, main_n, q_tail, dim, qn, vn);
					if (sub == 0 && k < n) hop_key[k] = make_key(d, my_id);
					__syncwarp();
					if (g + 1 < G) issue(g + 1);
				}
				// ---- give the ring back ---------------------------------------------------------------
				if (lane == 0)
				{
					__threadfence_block();
					if (rpar != rpar0) atomicXor(&pool->state, 1u << (16u + rb));  // hand the new parity on ...
					atomicOr(&pool->state, 1u << rb);								 // ... then free the ring
				}
				}  // !COOP

				const uint64_t *Rb = res + (size_t) cur * ef;
				uint64_t	   *Ob = res + (size_t) (cur ^ 1) * ef;
				const uint32_t	W = (r == ef) ? key_dist(Rb[ef - 1]) : 0xffffffffu;

				// ---- prefetch the link row of the candidate that will be popped next -------------------
				// Known before the queue update: it is the nearer of (best unexpanded result so far, nearest
				// new neighbour) -- the nearest new neighbour is always accepted when it beats an existing
				// result.  Only a hint: a wrong guess (exact ties, overflow list) falls back to global loads.
				if (p.prefetch_links)
				{
					uint64_t bestp = ~0ull;	 // (dist << 32 | 0x7fffffff - id): smaller pops first
					for (uint32_t base = 0; base < r; base += 32)
					{
						const uint32_t i = base + lane;
						const bool	   un = (i < r) && !key_expanded(Rb[i]);
						const uint32_t m = __ballot_sync(kFull, un);
						if (m)
						{
							const uint64_t kx = Rb[base + __ffs(m) - 1];
							bestp = ((uint64_t) key_dist(kx) << 32) | (uint64_t) (0x7fffffffu - key_id(kx));
							break;
						}
					}
					uint64_t mine = ~0ull;
					for (uint32_t k = lane; k < n; k += 32)
					{
						const uint64_t kx = hop_key[k];
						if (r + n <= ef || key_dist(kx) < W)
						{
							const uint64_t pr = ((uint64_t) key_dist(kx) << 32) | (uint64_t) (0x7fffffffu - key_id(kx));
							mine = min(mine, pr);
						}
					}
					for (int off = 16; off > 0; off >>= 1) mine = min(mine, __shfl_xor_sync(kFull, mine, off));
					bestp = min(bestp, mine);
					if (bestp != ~0ull)
					{
						if (pf_inflight)
						{
							mbar_wait(pf_bar, pf_parity);  // an unused earlier prefetch: long complete, frees the buffer
							pf_parity ^= 1u;
						}
						pf_id = 0x7fffffffu - (uint32_t) (bestp & 0xffffffffu);
						__syncwarp();
						if (lane == 0)
						{
							mbar_arrive_expect_tx(pf_bar, p.link_stride * 4u);
							tma_load_1d(pf_links, p.links + (size_t) pf_id * p.link_stride, p.link_stride * 4u, pf_bar, pol_keep);
						}
						pf_inflight = true;
					}
				}

				// ================= K2: sequential-equivalent queue update ==========================
				const bool all_accept = (r + n <= ef);
				uint32_t   a = 0;
				for (uint32_t base = 0; base < n; base += 32)
				{
					const uint32_t k = base + lane;
					bool		   acc = false;
					uint64_t	   key = 0;
					if (k < n)
					{
						key = hop_key[k];
						const uint32_t od = key_dist(key);
						if (all_accept)
							acc = true;
						else if (r == ef && od >= W)
							acc = false;
						else
						{
							uint32_t lo = 0, hi = r;  // cR = #{R : dist <= od}
							while (lo < hi)
							{
								const uint32_t mid = (lo + hi) >> 1;
								if (key_dist(Rb[mid]) <= od) lo = mid + 1; else hi = mid;
							}
							if (lo < ef)
							{
								uint32_t c = lo;
								for (uint32_t j = 0; j < k; j++) c += (key_dist(hop_key[j]) <= od) ? 1u : 0u;
								acc = c < ef;
							}
						}
					}
					const uint32_t m = __ballot_sync(kFull, acc);
					if (acc) acc_key[a + __popc(m & lt)] = key;
					a += __popc(m);
				}
				__syncwarp();
				if (a > 0)
				{
					const uint32_t total = r + a;
					for (uint32_t t = lane; t < a; t += 32)
					{
						const uint64_t key = acc_key[t];
						const uint64_t ko = key_order(key);
						uint32_t	   lo = 0, hi = r;
						while (lo < hi)
						{
							const uint32_t mid = (lo + hi) >> 1;
							if (key_order(Rb[mid]) < ko) lo = mid + 1; else hi = mid;
						}
						uint32_t pos = lo;
						for (uint32_t j = 0; j < a; j++) pos += (key_order(acc_key[j]) < ko) ? 1u : 0u;
						if (pos < ef) Ob[pos] = key; else evict_key[pos - ef] = key;
					}
					for (uint32_t i = lane; i < r; i += 32)
					{
						const uint64_t key = Rb[i];
						const uint64_t ko = key_order(key);
						uint32_t	   pos = i;
						for (uint32_t j = 0; j < a; j++) pos += (key_order(acc_key[j]) < ko) ? 1u : 0u;
						if (pos < ef) Ob[pos] = key; else evict_key[pos - ef] = key;
					}
					__syncwarp();
					cur ^= 1;
					r = min(total, ef);
					if (total > ef)
					{
						const uint32_t Wn = key_dist(Ob[ef - 1]);
						if (ovf_n > 0 && Wn != W) ovf_n = 0;  // worst distance dropped: old ties are dead
						const uint32_t ne = total - ef;
						for (uint32_t base = 0; base < ne; base += 32)
						{
							const uint32_t e = base + lane;
							uint64_t	   ek = 0;
							bool		   keep = false;
							if (e < ne)
							{
								ek = evict_key[e];
								keep = !key_expanded(ek) && key_dist(ek) == Wn;
							}
							const uint32_t m = __ballot_sync(kFull, keep);
							const uint32_t at = ovf_n + __popc(m & lt);
							if (keep)
							{
								if (at < ef) ovf[at] = ek; else *p.error_flag = 2;
							}
							ovf_n = min(ovf_n + (uint32_t) __popc(m), ef);
						}
						ovf_hw = max(ovf_hw, ovf_n);
						__syncwarp();
					}
				}
			}

			// ================= pop the next candidate (hnswalg.cpp:69-74) =========================
			const uint64_t *Rb = res + (size_t) cur * ef;
			int				best = -1;
			for (uint32_t base = 0; base < r; base += 32)
			{
				const uint32_t i = base + lane;
				const bool	   un = (i < r) && !key_expanded(Rb[i]);
				const uint32_t m = __ballot_sync(kFull, un);
				if (m)
				{
					best = (int) base + __ffs(m) - 1;
					break;
				}
			}
			if (best >= 0)
			{
				// equal-distance group: the reference pops the LARGEST id first (pair(-d,id) order)
				const uint32_t D = key_dist(Rb[best]);
				for (uint32_t base = (uint32_t) best + 1; base < r; base += 32)
				{
					const uint32_t i = base + lane;
					const bool	   ing = (i < r) && key_dist(Rb[i]) == D;
					const bool	   un = ing && !key_expanded(Rb[i]);
					const uint32_t mg = __ballot_sync(kFull, ing);
					const uint32_t mu = __ballot_sync(kFull, un);
					if (mu) best = (int) base + 31 - __clz(mu);
					if (mg != kFull) break;
				}
			}
			uint32_t c = kNone;
			bool	 from_ovf = false;
			if (ovf_n > 0)
			{
				// candidates evicted from the result set that still tie with its worst distance
				uint64_t bp = ~0ull;  // (dist << 32 | (0x7fffffff - id)) : smaller is better
				uint32_t bi = 0;
				for (uint32_t i = lane; i < ovf_n; i += 32)
				{
					const uint64_t k = ovf[i];
					const uint64_t pr = ((uint64_t) key_dist(k) << 32) | (uint64_t) (0x7fffffffu - key_id(k));
					if (pr < bp) { bp = pr; bi = i; }
				}
				for (int off = 16; off > 0; off >>= 1)
				{
					const uint64_t op = __shfl_xor_sync(kFull, bp, off);
					const uint32_t oi = __shfl_xor_sync(kFull, bi, off);
					if (op < bp) { bp = op; bi = oi; }
				}
				uint64_t rp = ~0ull;
				if (best >= 0) rp = ((uint64_t) key_dist(Rb[best]) << 32) | (uint64_t) (0x7fffffffu - key_id(Rb[best]));
				if (bp < rp)
				{
					from_ovf = true;
					c = 0x7fffffffu - (uint32_t) (bp & 0xffffffffu);
					__syncwarp();
					if (lane == 0) ovf[bi] = ovf[ovf_n - 1];
					ovf_n -= 1;
					__syncwarp();
				}
			}
			if (!from_ovf)
			{
				if (best < 0) break;  // candidateSet exhausted (or only entries beyond lowerBound)
				c = key_id(Rb[best]);
				__syncwarp();
				if (lane == 0) res[(size_t) cur * ef + best] |= 1ull;
				__syncwarp();
			}

			// ================= expand c: link list + visited set (hnswalg.cpp:76-93) ==============
			// The whole link row is obtained in one go (count and ids together: a dependent second DRAM
			// round trip for the ids would sit on the critical path of every hop) -- from the prefetch
			// buffer when the guess was right, else from global memory.
			const bool hit = pf_inflight && pf_id == c;
			if (hit)
			{
				mbar_wait(pf_bar, pf_parity);
				pf_parity ^= 1u;
				pf_inflight = false;
			}
			else
			{
				if (pf_inflight)
				{
					mbar_wait(pf_bar, pf_parity);  // wrong guess still in flight into the buffer we are about to fill
					pf_parity ^= 1u;
					pf_inflight = false;
				}
				const uint32_t *L = p.links + (size_t) c * p.link_stride;
				for (uint32_t i = lane; i < p.link_stride; i += 32) pf_links[i] = L[i];
				__syncwarp();
			}
			uint32_t cnt = pf_links[0];
			if (cnt > p.maxM)
			{
				cnt = p.maxM;
				*p.error_flag = 1;
			}
			if (p.exp_out && lane == 0 && st_hops < p.exp_cap) p.exp_out[(size_t) qi * p.exp_cap + st_hops] = c;
			st_hops += 1;
			st_words += 1 + cnt;
			n = 0;
			if (vmode == 0 && logn + cnt > (H >> 1))
			{
				// the open-addressing set would pass half full: migrate to the exact N-bit bitmap
				for (uint32_t i = lane; i < logn; i += 32)
				{
					const uint32_t pos = vlog[i];
					const uint32_t vid = vh_shared ? *reinterpret_cast<volatile uint32_t *>(&vh[pos]) : __ldcg(&vh[pos]);  // global: written by L2 atomics, never read through L1
					vh[pos] = kEmpty;
					atomicOr(&vis[vid >> 5], 1u << (vid & 31));
					vlog[i] = vid;
				}
				__syncwarp();
				vmode = 1;
			}
			if (COOP && p.visited_pairs)
			{
				// Two 32-id chunks of the list per iteration with BOTH chunks' test-and-set atomics in flight before
				// the first result is consumed: a full 64-link list costs one L2 round trip instead of two dependent
				// ones.  Only legal when the ids of a list are distinct (the host guarantees it: links_distinct), so
				// that the outcome of a chunk's atomics cannot depend on the other chunk's.
				for (uint32_t base = 0; base < cnt; base += 64)
				{
					const uint32_t kA = base + lane, kB = base + 32 + lane;
					bool		   vA = kA < cnt, vB = kB < cnt;
					uint32_t	   idA = vA ? pf_links[1 + kA] : 0u, idB = vB ? pf_links[1 + kB] : 0u;
					if (vA && idA >= p.n_items) { vA = false; *p.error_flag = 1; }
					if (vB && idB >= p.n_items) { vB = false; *p.error_flag = 1; }
					bool	 uA = false, uB = false;
					uint32_t lA = idA, lB = idB;
					if (vmode == 0)
					{
						uint32_t hA = (idA * 2654435761u) >> vh_shift, hB = (idB * 2654435761u) >> vh_shift;
						bool	 pA = vA, pB = vB;	// still probing
						while (pA || pB)
						{
							uint32_t oA = 0u, oB = 0u;
							if (pA) oA = atomicCAS(&vh[hA], kEmpty, idA);
							if (pB) oB = atomicCAS(&vh[hB], kEmpty, idB);
							if (pA)
							{
								if (oA == kEmpty) { uA = true; lA = hA; pA = false; }
								else if (oA == idA) pA = false;
								else hA = (hA + 1) & (H - 1);
							}
							if (pB)
							{
								if (oB == kEmpty) { uB = true; lB = hB; pB = false; }
								else if (oB == idB) pB = false;
								else hB = (hB + 1) & (H - 1);
							}
						}
					}
					else
					{
						const uint32_t bA = 1u << (idA & 31), bB = 1u << (idB & 31);
						uint32_t	   oA = 0xffffffffu, oB = 0xffffffffu;
						if (vA) oA = atomicOr(&vis[idA >> 5], bA);
						if (vB) oB = atomicOr(&vis[idB >> 5], bB);
						uA = vA && !(oA & bA);
						uB = vB && !(oB & bB);
					}
					const uint32_t mA = __ballot_sync(kFull, uA), mB = __ballot_sync(kFull, uB);
					const uint32_t cA = (uint32_t) __popc(mA);
					if (uA)
					{
						const uint32_t off = __popc(mA & lt);
						hop_id[n + off] = idA;
						if (logn + off < p.vlog_cap) vlog[logn + off] = lA;
					}
					if (uB)
					{
						const uint32_t off = cA + __popc(mB & lt);
						hop_id[n + off] = idB;
						if (logn + off < p.vlog_cap) vlog[logn + off] = lB;
					}
					n += cA + (uint32_t) __popc(mB);
					logn += cA + (uint32_t) __popc(mB);
				}
			}
			else
			for (uint32_t base = 0; base < cnt; base += 32)
			{
				// list position k = base + lane lives in word k + 1
				const uint32_t k = base + lane;
				bool		   valid = k < cnt;
				uint32_t	   id = valid ? pf_links[1 + k] : 0u;
				if (!valid) id = 0u;
				if (valid && id >= p.n_items)
				{
					valid = false;
					*p.error_flag = 1;
				}
				const uint32_t mm = __match_any_sync(kFull, valid ? id : (0x80000000u | lane));
				const bool	   first = valid && ((uint32_t) (__ffs(mm) - 1) == lane);
				bool		   unv = false;
				uint32_t	   logv = id;
				if (vmode == 0)
				{
					if (first)
					{
						uint32_t h = (id * 2654435761u) >> vh_shift;
						for (;;)
						{
							const uint32_t old = atomicCAS(&vh[h], kEmpty, id);
							if (old == kEmpty) { unv = true; logv = h; break; }
							if (old == id) break;
							h = (h + 1) & (H - 1);
						}
					}
				}
				else
				{
					const uint32_t bit = 1u << (id & 31);
					uint32_t	   old = 0xffffffffu;
					if (first) old = atomicOr(&vis[id >> 5], bit);
					unv = first && !(old & bit);
				}
				const uint32_t m = __ballot_sync(kFull, unv);
				const uint32_t off = __popc(m & lt);
				if (unv)
				{
					hop_id[n + off] = id;
					if (logn + off < p.vlog_cap) vlog[logn + off] = logv;
				}
				n += __popc(m);
				logn += __popc(m);
			}
			__syncwarp();
		}

		// ---- emit (hnswalg.cpp:238-249, :262-270) ---------------------------------------------------
		const uint64_t *Rb = res + (size_t) cur * ef;
		uint64_t	   *lab = res + (size_t) (cur ^ 1) * ef;  // scratch: labels of the results
		const size_t	ob = (size_t) qi * ef;
		uint32_t		count = r;
		if (p.raw_mode)
		{
			for (uint32_t i = lane; i < ef; i += 32)
			{
				const bool ok = i < r;
				if (p.ids_out) p.ids_out[ob + i] = ok ? key_id(Rb[i]) : kNone;
				if (p.dists_out) p.dists_out[ob + i] = ok ? o2f(key_dist(Rb[i])) : __int_as_float(0x7f800000);
				if (p.labels_out) p.labels_out[ob + i] = ok ? (uint64_t) key_id(Rb[i]) : ~0ull;
			}
		}
		else
		{
			for (uint32_t i = lane; i < r; i += 32) lab[i] = p.labels[key_id(Rb[i])];
			__syncwarp();
			// order by (dist, label) among non-deleted entries (searchKnn builds pair<dist,label>)
			uint32_t cnt_live = 0;
			for (uint32_t base = 0; base < r; base += 32)
			{
				const uint32_t i = base + lane;
				bool		   live = false;
				uint32_t	   pos = 0;
				if (i < r)
				{
					const uint64_t li = lab[i];
					live = ((li >> 48) & 1ull) == 0;  // !hnsw_is_deleted, embedding.c:948-953
					if (live)
					{
						const uint32_t di = key_dist(Rb[i]);
						for (uint32_t j = 0; j < r; j++)
						{
							const uint64_t lj = lab[j];
							if ((lj >> 48) & 1ull) continue;
							const uint32_t dj = key_dist(Rb[j]);
							pos += (dj < di || (dj == di && (lj < li || (lj == li && j < i)))) ? 1u : 0u;
						}
						if (p.labels_out) p.labels_out[ob + pos] = li;
						if (p.dists_out) p.dists_out[ob + pos] = o2f(di);
						if (p.ids_out) p.ids_out[ob + pos] = key_id(Rb[i]);
					}
				}
				cnt_live += __popc(__ballot_sync(kFull, live));
			}
			count = cnt_live;
			for (uint32_t i = count + lane; i < ef; i += 32)
			{
				if (p.labels_out) p.labels_out[ob + i] = ~0ull;
				if (p.dists_out) p.dists_out[ob + i] = __int_as_float(0x7f800000);
				if (p.ids_out) p.ids_out[ob + i] = kNone;
			}
		}
		if (lane == 0)
		{
			p.n_out[qi] = (int32_t) count;
			if (p.exp_n_out) p.exp_n_out[qi] = st_hops;
			if (p.stats_out)
			{
				p.stats_out[(size_t) qi * 4 + 0] = st_dist;
				p.stats_out[(size_t) qi * 4 + 1] = st_hops;
				p.stats_out[(size_t) qi * 4 + 2] = st_words;
				p.stats_out[(size_t) qi * 4 + 3] = ovf_hw;
			}
		}

		// ---- reset the visited set: O(visited) via the log, full clear if the log overflowed ---------
		if (vmode == 0)
			for (uint32_t i = lane; i < logn; i += 32) vh[vlog[i]] = kEmpty;
		else if (logn <= p.vlog_cap)
			for (uint32_t i = lane; i < logn; i += 32) vis[vlog[i] >> 5] = 0u;
		else
			for (uint32_t i = lane; i < p.vis_words; i += 32) vis[i] = 0u;
		__syncwarp();
	}
	if (COOP)
	{
		// release the helper warps
		if (lane == 0) pool->coop_n = kNone;
		__syncwarp();
		coop_bar(1, blockDim.x);
	}
	// an unconsumed link prefetch must land before the CTA (and its shared memory) goes away
	if (pf_inflight) mbar_wait(pf_bar, pf_parity);
}

typedef void (*search_fn_t)(const SearchParams);

// The traversal instance for a metric, mode, lanes per row and result-queue placement (nullptr: there is none).  Host code,
// shared by capi.cu's plan_search and the emulation harness in tests/emu, so that both launch the same instance.
inline search_fn_t pick_search_kernel(int metric, bool coop, uint32_t tpr, bool res_global)
{
	if (res_global)
	{
		if (coop || tpr != 4) return nullptr;
		switch (metric)
		{
			case DIST_L2: return search_kernel<M_L2, false, 4, true>;
			case DIST_COSINE: return search_kernel<M_COS, false, 4, true>;
			case DIST_MANHATTAN: return search_kernel<M_MAN, false, 4, true>;
		}
		return nullptr;
	}
	if (metric == DIST_L2 && tpr == 8) return coop ? search_kernel<M_L2, true, 8> : search_kernel<M_L2, false, 8>;
	if (tpr != 4) return nullptr;
	switch (metric)
	{
		case DIST_L2: return coop ? search_kernel<M_L2, true> : search_kernel<M_L2, false>;
		case DIST_COSINE: return coop ? search_kernel<M_COS, true> : search_kernel<M_COS, false>;
		case DIST_MANHATTAN: return coop ? search_kernel<M_MAN, true> : search_kernel<M_MAN, false>;
	}
	return nullptr;
}

}  // namespace pgemb
