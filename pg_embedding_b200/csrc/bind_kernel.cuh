// bind_kernel.cuh -- K4: the insert side of the hot path.
//
// hnsw_bind_point (hnswalg.cpp:279-291) = bindPoint (:225-232) =
//     searchBaseLayer(point, efConstruction)            -> search_kernel in raw mode (query = stored node)
//     mutuallyConnectNewElement (:155-223):
//         getNeighborsByHeuristic(top, M) (:117-153)    -> select_kernel (one CTA per new node)
//         write own list, farthest first (:164-180)     -> select_kernel
//         per chosen neighbour: append the back-link or re-prune its full list with the heuristic
//         at NN = maxM and rewrite it farthest first (:182-222)
//                                                       -> backlink_kernel (one CTA per (target) list)
//
// Exactness notes (link lists checked byte for byte against the oracle: sequential binds in tests/test_gpu_parity.py, the
// batched bulk build against the oracle's batch model in tests/test_gpu_bulk_build.py):
//  * heuristic scan order = ascending distance to the base point, equal distances by DESCENDING id
//    (resultSet holds pair(-dist,id), :126,:133); a candidate is kept iff no already kept r has
//    dist(r,c) < dist(c,base) (:141-147, the early `break` only skips work); stop at NN kept (:131).
//    `top.size() < NN` returns the input unchanged (:119-120).
//  * both link lists are written in DESCENDING (dist,id) pair order (pop order of a max-heap, :164-167,
//    :213-218).
//  * node-to-node distances use the same exact-order arithmetic as the search (dist_exact.cuh) with the
//    cached squared norms for cosine.
//
// Batch use (bulk build): `n_new` nodes whose searches all ran against the graph as it was before the
// batch.  Own lists never conflict; back-links to the same target are serialised in source-id order by
// sorting (target,source) pairs and letting the CTA of each segment head apply its segment sequentially
// -- for n_new == 1 this is exactly one reference insert.
#pragma once
#ifndef PGEMB_HOST_EMULATION
#include <cub/cub.cuh>
#endif

#include "common.cuh"
#include "dist_exact.cuh"

struct pgemb_index;

namespace pgemb {

struct BindWorkspace
{
	size_t	  cap_points = 0, cap_ef = 0, cap_m = 0;
	uint32_t *d_qids = nullptr;		 // [points]
	uint32_t *d_cand_ids = nullptr;	 // [points][ef]
	float	 *d_cand_d = nullptr;	 // [points][ef]
	int32_t	 *d_cand_n = nullptr;	 // [points]
	uint64_t *d_pairs = nullptr;	 // [points*M] (target << 32 | source), ~0 = none
	uint64_t *d_pairs_sorted = nullptr;
	void	 *d_cub = nullptr;
	size_t	  cub_bytes = 0;
	// select_global_kernel only (efConstruction beyond a CTA's shared memory): candidate keys and scan order, [points][ef]
	uint64_t *d_sel_keys = nullptr;
	uint32_t *d_sel_ord = nullptr;
	// exact parallel build (speculative batches)
	static constexpr uint32_t kExpCap = 1024;
	uint32_t *d_exp = nullptr;		 // [points][kExpCap] expanded nodes of each speculative search
	uint32_t *d_exp_n = nullptr;	 // [points]
	uint32_t *d_stamp = nullptr;	 // [capacity] see validate_kernel
	uint32_t *d_first = nullptr;	 // first conflicting batch index
	size_t	  stamp_cap = 0;
};

inline void bind_ws_free(BindWorkspace &w)
{
	cudaFree(w.d_qids);
	cudaFree(w.d_cand_ids);
	cudaFree(w.d_cand_d);
	cudaFree(w.d_cand_n);
	cudaFree(w.d_pairs);
	cudaFree(w.d_pairs_sorted);
	cudaFree(w.d_cub);
	cudaFree(w.d_sel_keys);
	cudaFree(w.d_sel_ord);
	cudaFree(w.d_exp);
	cudaFree(w.d_exp_n);
	cudaFree(w.d_stamp);
	cudaFree(w.d_first);
	w = BindWorkspace();
}

struct GraphView
{
	const float	   *vectors;
	const float	   *norms;
	uint32_t	   *links;
	uint32_t		row_f, link_stride, dim, M, maxM;
	int			   *error_flag;
};

constexpr int kBindThreads = 256;

// Distance between two STORED nodes, LANES threads per pair, scalar loads straight from global/L2.
template <int METRIC>
__device__ __forceinline__ float node_dist(const GraphView &g, uint32_t a, uint32_t b, int sub)
{
	constexpr int L = MetricLanes<METRIC>::LANES;
	const float	 *va = g.vectors + (size_t) a * g.row_f;
	const float	 *vb = g.vectors + (size_t) b * g.row_f;
	float		  na = 0.f, nb = 0.f;
	if (METRIC == M_COS)
	{
		na = g.norms[a];
		nb = g.norms[b];
	}
	return distance_exact<METRIC, L>(va, vb, (int) g.dim, na, nb, sub);
}

// getNeighborsByHeuristic on a block.  cand[0..C) = keys ascending by (dist,id) (flag bit clear);
// ord[] scratch (C entries); kept[] receives up to NN keys in acceptance order.  Returns #kept.
// All kBindThreads threads must call it.
template <int METRIC>
__device__ uint32_t heuristic_block(const GraphView &g, const uint64_t *cand, uint32_t C, uint32_t NN, uint32_t *ord, uint64_t *kept)
{
	constexpr int  L = MetricLanes<METRIC>::LANES;
	constexpr int  NG = kBindThreads / L;
	const uint32_t tid = threadIdx.x;
	const int	   grp = tid / L, sub = tid % L;
	// scan order: ascending distance, equal distances by descending id
	for (uint32_t i = tid; i < C; i += kBindThreads)
	{
		const uint32_t d = key_dist(cand[i]);
		uint32_t	   gs = i, ge = i + 1;
		while (gs > 0 && key_dist(cand[gs - 1]) == d) gs--;
		while (ge < C && key_dist(cand[ge]) == d) ge++;
		ord[gs + (ge - 1 - i)] = i;
	}
	__syncthreads();
	uint32_t nkept = 0;
	for (uint32_t i = 0; i < C && nkept < NN; i++)
	{
		const uint64_t ck = cand[ord[i]];
		const uint32_t cid = key_id(ck);
		const float	   dq = o2f(key_dist(ck));
		int			   bad = 0;
		for (uint32_t base = 0; base < nkept; base += NG)
		{
			// every lane of a warp takes part in the shuffles: clamp instead of skipping
			const uint32_t k = base + grp;
			const uint32_t kk = k < nkept ? k : nkept - 1;
			const float	   dd = node_dist<METRIC>(g, key_id(kept[kk]), cid, sub);
			if (k < nkept && dd < dq) bad = 1;
		}
		const int any = __syncthreads_or(bad);
		if (!any)
		{
			if (tid == 0) kept[nkept] = ck;
			nkept++;
		}
		__syncthreads();
	}
	return nkept;
}

// Write `n` keys as a link list in DESCENDING (dist,id) order: links = [n, ids...]; rest untouched.
__device__ __forceinline__ void write_list_desc(uint32_t *L, const uint64_t *keys, uint32_t n)
{
	for (uint32_t i = threadIdx.x; i < n; i += kBindThreads)
	{
		const uint64_t k = key_order(keys[i]);
		uint32_t	   rank = 0;
		for (uint32_t j = 0; j < n; j++) rank += (key_order(keys[j]) > k) ? 1u : 0u;
		L[1 + rank] = key_id(keys[i]);
	}
	if (threadIdx.x == 0) L[0] = n;
}

// The same heuristic with its operands STAGED in shared memory (select_kernel<METRIC, true>: one insert at a time, where the
// heuristic -- not the search -- was the longest part of hnsw_bind_point: up to efConstruction sequential steps, each a chain of
// ~24 dependent L2 round trips per 768-d distance; ncu: 3.3 ms of a 200K-row insert).  The rows of the kept set (<= NN x row_f
// floats) stay in shared memory from the moment they are accepted, the next candidate's row is fetched by bulk TMA while the
// current one is tested, so a step costs a few shared-memory passes.  Same pairs, same argument order, same arithmetic as
// heuristic_block: same decisions, same bits.
//   rows_s: [NN + 2][row_f] floats (16-byte aligned): NN kept rows, then two candidate buffers;  bars: two mbarriers.
template <int METRIC>
__device__ uint32_t heuristic_block_staged(const GraphView &g, const uint64_t *cand, uint32_t C, uint32_t NN, uint32_t *ord, uint64_t *kept,
											float *rows_s, uint64_t *bars)
{
	constexpr int  L = MetricLanes<METRIC>::LANES;
	constexpr int  NG = kBindThreads / L;
	const uint32_t tid = threadIdx.x;
	const int	   grp = tid / L, sub = tid % L;
	const uint32_t row_b = g.row_f * 4u;
	float		  *cbuf = rows_s + (size_t) NN * g.row_f;
	__shared__ float kept_norm[256];  // squared norms of the kept rows (cosine), NN <= 256 checked by the caller
	for (uint32_t i = tid; i < C; i += kBindThreads)
	{
		const uint32_t d = key_dist(cand[i]);
		uint32_t	   gs = i, ge = i + 1;
		while (gs > 0 && key_dist(cand[gs - 1]) == d) gs--;
		while (ge < C && key_dist(cand[ge]) == d) ge++;
		ord[gs + (ge - 1 - i)] = i;
	}
	if (tid == 0)
	{
		mbar_init(&bars[0], 1);
		mbar_init(&bars[1], 1);
		fence_mbar_init();
	}
	__syncthreads();
	const uint64_t pol = l2_policy_evict_last();
	uint32_t	   par0 = 0, par1 = 0;
	if (tid == 0 && C > 0)
	{
		mbar_arrive_expect_tx(&bars[0], row_b);
		tma_load_1d(cbuf, g.vectors + (size_t) key_id(cand[ord[0]]) * g.row_f, row_b, &bars[0], pol);
	}
	uint32_t nkept = 0, i = 0;
	for (; i < C && nkept < NN; i++)
	{
		const uint32_t b = i & 1u;
		const uint64_t ck = cand[ord[i]];
		const uint32_t cid = key_id(ck);
		const float	   dq = o2f(key_dist(ck));
		float		  *crow = cbuf + (size_t) b * g.row_f;
		if (tid == 0 && i + 1 < C)
		{
			// the other buffer was last read in step i - 1 (all threads passed that step's final barrier)
			mbar_arrive_expect_tx(&bars[b ^ 1u], row_b);
			tma_load_1d(cbuf + (size_t) (b ^ 1u) * g.row_f, g.vectors + (size_t) key_id(cand[ord[i + 1]]) * g.row_f, row_b, &bars[b ^ 1u], pol);
		}
		float cn = 0.f;
		if (METRIC == M_COS) cn = g.norms[cid];
		if (b == 0) { mbar_wait(&bars[0], par0); par0 ^= 1u; } else { mbar_wait(&bars[1], par1); par1 ^= 1u; }
		int bad = 0;
		for (uint32_t base = 0; base < nkept; base += NG)
		{
			const uint32_t k = base + grp;
			const uint32_t kk = k < nkept ? k : nkept - 1;
			const float	   dd = distance_exact<METRIC, L>(rows_s + (size_t) kk * g.row_f, crow, (int) g.dim, kept_norm[kk], cn, sub);
			if (k < nkept && dd < dq) bad = 1;
		}
		const int any = __syncthreads_or(bad);
		if (!any)
		{
			float *dst = rows_s + (size_t) nkept * g.row_f;
			for (uint32_t e = tid; e < g.row_f; e += kBindThreads) dst[e] = crow[e];
			if (tid == 0)
			{
				kept[nkept] = ck;
				kept_norm[nkept] = cn;
			}
			nkept++;
		}
		__syncthreads();
	}
	// a candidate row may still be in flight into the buffer (prefetched for a step that never ran): let it land
	if (i < C)
	{
		if ((i & 1u) == 0) mbar_wait(&bars[0], par0); else mbar_wait(&bars[1], par1);
	}
	__syncthreads();
	return nkept;
}

// ---- select: heuristic at NN = M over the search result, write the new node's own list --------------
template <int METRIC, bool STAGED = false>
__global__ void __launch_bounds__(kBindThreads) select_kernel(GraphView g, const uint32_t *__restrict__ new_ids,
															   const uint32_t *__restrict__ cand_ids, const float *__restrict__ cand_d,
															   const int32_t *__restrict__ cand_n, uint32_t ef,
															   uint64_t *__restrict__ pairs /* [n_new][M] */)
{
	PGEMB_DYNAMIC_SMEM(sm, 16);
	uint64_t	  *cand = reinterpret_cast<uint64_t *>(sm);			// ef
	uint64_t	  *kept = cand + ef;								// max(M,1)
	uint32_t	  *ord = reinterpret_cast<uint32_t *>(kept + (g.M ? g.M : 1));	// ef
	// STAGED: [2 mbarriers][(M + 2) rows] behind the arrays above, 16-byte aligned (select_smem_bytes)
	uint64_t	  *stage_bars = reinterpret_cast<uint64_t *>(sm + ((size_t) ef * 8 + (size_t) (g.M ? g.M : 1) * 8 + (size_t) ef * 4 + 15) / 16 * 16);
	float		  *stage_rows = reinterpret_cast<float *>(stage_bars + 2);
	const uint32_t b = blockIdx.x;
	const uint32_t cur = new_ids[b];
	uint64_t	  *my_pairs = pairs + (size_t) b * (g.M ? g.M : 1);
	for (uint32_t i = threadIdx.x; i < g.M; i += kBindThreads) my_pairs[i] = ~0ull;
	if (cur == 0) return;  // "Do nothing for the first element", hnswalg.cpp:227-228
	const uint32_t C = (uint32_t) max(0, cand_n[b]);
	for (uint32_t i = threadIdx.x; i < C; i += kBindThreads)
		cand[i] = make_key(cand_d[(size_t) b * ef + i], cand_ids[(size_t) b * ef + i]);
	__syncthreads();
	uint32_t		nsel;
	const uint64_t *sel;
	if (C < g.M)
	{
		nsel = C;  // hnswalg.cpp:119-120: fewer than NN candidates -> all of them
		sel = cand;
	}
	else
	{
		nsel = STAGED ? heuristic_block_staged<METRIC>(g, cand, C, g.M, ord, kept, stage_rows, stage_bars) : heuristic_block<METRIC>(g, cand, C, g.M, ord, kept);
		sel = kept;
	}
	__syncthreads();
	uint32_t *L = g.links + (size_t) cur * g.link_stride;
	// "Should be blank" (hnswalg.cpp:170-171, :176-177)
	int bad = 0;
	for (uint32_t i = threadIdx.x; i <= nsel && i <= g.maxM; i += kBindThreads) bad |= (L[i] != 0u);
	if (__syncthreads_or(bad))
	{
		if (threadIdx.x == 0) *g.error_flag = 3;
		return;
	}
	write_list_desc(L, sel, nsel);
	// back-link work items, keyed (target, source) so that a sort serialises equal targets by source id
	for (uint32_t i = threadIdx.x; i < nsel; i += kBindThreads)
	{
		const uint32_t s = key_id(sel[i]);
		if (s == cur) *g.error_flag = 3;  // "Connection to the same element" (hnswalg.cpp:183-184)
		my_pairs[i] = ((uint64_t) s << 32) | (uint64_t) cur;
	}
}

// The same select with the candidate keys and the scan order in the bind workspace (keys, ord: [n_new][ef]) and only the
// kept keys in shared memory: for an efConstruction whose 12 x ef bytes exceed a CTA's shared memory.  Same heuristic, same
// order, same arithmetic -- the same lists.  A copy of select_kernel's unstaged body: moving that body into a shared device function
// changed the instructions nvcc emits for select_kernel, whose measured code stays as it is.
template <int METRIC>
__global__ void __launch_bounds__(kBindThreads) select_global_kernel(GraphView g, const uint32_t *__restrict__ new_ids,
																	  const uint32_t *__restrict__ cand_ids, const float *__restrict__ cand_d,
																	  const int32_t *__restrict__ cand_n, uint32_t ef,
																	  uint64_t *__restrict__ pairs, uint64_t *__restrict__ keys,
																	  uint32_t *__restrict__ ords)
{
	PGEMB_DYNAMIC_SMEM(sm, 16);
	uint64_t	  *cand = keys + (size_t) blockIdx.x * ef;			// ef, in the workspace
	uint64_t	  *kept = reinterpret_cast<uint64_t *>(sm);			// max(M,1)
	uint32_t	  *ord = ords + (size_t) blockIdx.x * ef;			// ef, in the workspace
	const uint32_t b = blockIdx.x;
	const uint32_t cur = new_ids[b];
	uint64_t	  *my_pairs = pairs + (size_t) b * (g.M ? g.M : 1);
	for (uint32_t i = threadIdx.x; i < g.M; i += kBindThreads) my_pairs[i] = ~0ull;
	if (cur == 0) return;  // "Do nothing for the first element", hnswalg.cpp:227-228
	const uint32_t C = (uint32_t) max(0, cand_n[b]);
	for (uint32_t i = threadIdx.x; i < C; i += kBindThreads)
		cand[i] = make_key(cand_d[(size_t) b * ef + i], cand_ids[(size_t) b * ef + i]);
	__syncthreads();
	uint32_t		nsel;
	const uint64_t *sel;
	if (C < g.M)
	{
		nsel = C;  // hnswalg.cpp:119-120: fewer than NN candidates -> all of them
		sel = cand;
	}
	else
	{
		nsel = heuristic_block<METRIC>(g, cand, C, g.M, ord, kept);
		sel = kept;
	}
	__syncthreads();
	uint32_t *L = g.links + (size_t) cur * g.link_stride;
	// "Should be blank" (hnswalg.cpp:170-171, :176-177)
	int bad = 0;
	for (uint32_t i = threadIdx.x; i <= nsel && i <= g.maxM; i += kBindThreads) bad |= (L[i] != 0u);
	if (__syncthreads_or(bad))
	{
		if (threadIdx.x == 0) *g.error_flag = 3;
		return;
	}
	write_list_desc(L, sel, nsel);
	// back-link work items, keyed (target, source) so that a sort serialises equal targets by source id
	for (uint32_t i = threadIdx.x; i < nsel; i += kBindThreads)
	{
		const uint32_t s = key_id(sel[i]);
		if (s == cur) *g.error_flag = 3;  // "Connection to the same element" (hnswalg.cpp:183-184)
		my_pairs[i] = ((uint64_t) s << 32) | (uint64_t) cur;
	}
}

// dynamic shared memory of select_kernel: candidate keys, kept keys, scan order (+ the staged rows)
inline size_t select_smem_bytes(size_t ef, size_t M, size_t row_f, bool staged)
{
	const size_t base = ef * 8 + (M ? M : 1) * 8 + ef * 4;
	if (!staged) return base;
	return (base + 15) / 16 * 16 + 16 + ((M ? M : 1) + 2) * row_f * 4;
}

// dynamic shared memory of select_global_kernel: the kept keys
inline size_t select_global_smem_bytes(size_t M) { return (M ? M : 1) * 8; }

// ---- back-links: one CTA per run of equal targets in the sorted (target,source) array ----------------
template <int METRIC>
__global__ void __launch_bounds__(kBindThreads) backlink_kernel(GraphView g, const uint64_t *__restrict__ pairs_sorted, uint32_t n_pairs)
{
	PGEMB_DYNAMIC_SMEM(sm, 16);
	const uint32_t C1 = g.maxM + 1;
	uint64_t	  *unsorted = reinterpret_cast<uint64_t *>(sm);	 // C1
	uint64_t	  *cand = unsorted + C1;						 // C1
	uint64_t	  *kept = cand + C1;							 // maxM (>=1)
	uint32_t	  *ord = reinterpret_cast<uint32_t *>(kept + (g.maxM ? g.maxM : 1));  // C1
	constexpr int  LN = MetricLanes<METRIC>::LANES;
	constexpr int  NG = kBindThreads / LN;
	const uint32_t tid = threadIdx.x;
	const int	   grp = tid / LN, sub = tid % LN;

	uint32_t	   e = blockIdx.x;
	const uint64_t head = pairs_sorted[e];
	if (head == ~0ull) return;
	const uint32_t target = (uint32_t) (head >> 32);
	if (e > 0 && (uint32_t) (pairs_sorted[e - 1] >> 32) == target) return;	// not a segment head
	uint32_t *L = g.links + (size_t) target * g.link_stride;

	for (; e < n_pairs; e++)
	{
		const uint64_t pr = pairs_sorted[e];
		if (pr == ~0ull || (uint32_t) (pr >> 32) != target) break;
		const uint32_t cur = (uint32_t) pr;
		const uint32_t cnt = L[0];
		if (cnt > g.maxM)
		{
			if (tid == 0) *g.error_flag = 3;  // "Bad sz_link_list_other" (hnswalg.cpp:190-191)
			return;
		}
		if (cnt < g.maxM)
		{
			__syncthreads();
			if (tid == 0)
			{
				L[1 + cnt] = cur;  // hnswalg.cpp:193-195
				L[0] = cnt + 1;
			}
			__syncthreads();
			continue;
		}
		// full list: candidates = {cur} u links(target), scored against target (hnswalg.cpp:198-210)
		for (uint32_t base = 0; base < C1; base += NG)
		{
			const uint32_t k = base + grp;
			const uint32_t kk = k < C1 ? k : C1 - 1;
			const uint32_t id = (kk == 0) ? cur : L[kk];
			const float	   d = node_dist<METRIC>(g, id, target, sub);
			if (k < C1 && sub == 0) unsorted[k] = make_key(d, id);
		}
		__syncthreads();
		for (uint32_t i = tid; i < C1; i += kBindThreads)
		{
			const uint64_t k = key_order(unsorted[i]);
			uint32_t	   rank = 0;
			for (uint32_t j = 0; j < C1; j++) rank += (key_order(unsorted[j]) < k) ? 1u : 0u;
			cand[rank] = unsorted[i];
		}
		__syncthreads();
		const uint32_t nk = heuristic_block<METRIC>(g, cand, C1, g.maxM, ord, kept);
		__syncthreads();
		write_list_desc(L, kept, nk);  // hnswalg.cpp:213-219 (slots beyond the new count keep stale ids, as in the reference)
		__syncthreads();
	}
}

// ---- exact parallel build: validation of speculative searches -------------------------------------------
// A batch of inserts i..i+B-1 is searched in parallel against the graph G0 as it was before the batch.
// Insert k's search is exactly the search the sequential algorithm would have run iff none of the nodes it
// EXPANDED (whose link lists it read) is modified by an earlier insert of the batch: the traversal is a
// function of the lists of the expanded nodes only.  Insert j modifies the lists of its selected neighbours
// (back-links, hnswalg.cpp:182-222); its own node is not in G0 and is reachable only through those lists.
// stamp[t] = smallest id of a batch insert that modifies node t (0xffffffff = none);
// insert k conflicts iff some expanded node e has stamp[e] < id_k.

__global__ void stamp_targets_kernel(const uint64_t *__restrict__ pairs, uint32_t n_pairs, uint32_t *__restrict__ stamp)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_pairs) return;
	const uint64_t pr = pairs[i];
	if (pr == ~0ull) return;
	atomicMin(&stamp[(uint32_t) (pr >> 32)], (uint32_t) pr);
}

__global__ void clear_stamps_kernel(const uint64_t *__restrict__ pairs, uint32_t n_pairs, uint32_t *__restrict__ stamp)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_pairs) return;
	const uint64_t pr = pairs[i];
	if (pr == ~0ull) return;
	stamp[(uint32_t) (pr >> 32)] = 0xffffffffu;
}

// one warp per batch insert; first_conflict = smallest batch index whose speculative search is invalid
__global__ void validate_kernel(const uint32_t *__restrict__ exp_ids, const uint32_t *__restrict__ exp_n, uint32_t exp_cap,
								const uint32_t *__restrict__ new_ids, uint32_t B, const uint32_t *__restrict__ stamp,
								uint32_t *__restrict__ first_conflict)
{
	const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	if (k >= B) return;
	const uint32_t id_k = new_ids[k];
	const uint32_t cnt = exp_n[k];
	bool		   bad = cnt > exp_cap;	 // incomplete list: cannot be validated
	const uint32_t m = cnt < exp_cap ? cnt : exp_cap;
	for (uint32_t i = lane; i < m; i += 32) bad |= stamp[exp_ids[(size_t) k * exp_cap + i]] < id_k;
	if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(first_conflict, k);
}

// undo the own-list writes of the rejected tail of a batch (their slots must be blank again, hnswalg.cpp:170-177)
__global__ void zero_links_kernel(uint32_t *__restrict__ links, uint32_t link_stride, const uint32_t *__restrict__ ids, uint32_t n)
{
	const uint32_t w = blockIdx.x;
	if (w >= n) return;
	uint32_t *L = links + (size_t) ids[w] * link_stride;
	for (uint32_t i = threadIdx.x; i < link_stride; i += blockDim.x) L[i] = 0u;
}

}  // namespace pgemb

pgemb_status bind_points(pgemb_index *idx, idx_t first, size_t n);
