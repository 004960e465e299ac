// aux_kernels.cuh -- small kernels around the traversal: cached norms, stand-alone distance batches
// (the reference's hnsw_dist_func / SQL distance operators, distfunc.c:171-174, embedding.c:1022-1062),
// reference-record (AoS) ingest/export, shard top-k merge.
#pragma once
#include "common.cuh"
#include "dist_exact.cuh"

namespace pgemb {

// ---- squared norms of stored rows, cosine lane order (4 threads per row) -----------------------
__global__ void norms_kernel(const float *__restrict__ vectors, uint32_t row_f, uint32_t dim, uint32_t first, uint32_t n,
							 float *__restrict__ norms)
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t row = t >> 2;
	const int	   sub = t & 3;
	// all 32 lanes of a warp must reach the shuffles: clamp the row instead of returning early
	const uint32_t rr = row < n ? row : (n ? n - 1 : 0);
	if (n == 0) return;
	const float *v = vectors + (size_t) (first + rr) * row_f;
	const float	 s = sqnorm_exact<4>(v, (int) dim, sub);
	if (row < n && sub == 0) norms[first + row] = s;
}

// ---- invariant check for caller-provided link lists: are the ids of every list distinct? ----------------
// (Lists written by the bind kernels always are; the traversal may then test-and-set both halves of a list
// concurrently, search_kernel.cuh `visited_pairs`.)  One warp per node; sets *dup_flag if any list repeats an id.
__global__ void links_distinct_kernel(const uint32_t *__restrict__ links, uint32_t link_stride, uint32_t maxM, uint32_t first, uint32_t n,
									  int *__restrict__ dup_flag)
{
	const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	if (w >= n) return;
	const uint32_t *L = links + (size_t) (first + w) * link_stride;
	uint32_t		cnt = L[0];
	if (cnt > maxM) cnt = maxM;
	bool dup = false;
	for (uint32_t k = lane; k < cnt; k += 32)
	{
		const uint32_t id = L[1 + k];
		for (uint32_t j = 0; j < k; j++) dup |= (L[1 + j] == id);
	}
	if (dup) *dup_flag = 1;
}

// ---- pair distances: out[i] = dist(a[i] | a[0], b[i]); LANES threads per pair, scalar loads --------
template <int METRIC>
__global__ void dist_pairs_kernel(const float *__restrict__ a, const float *__restrict__ b, uint32_t dim, uint32_t a_stride,
								  uint32_t b_stride, uint32_t n, int broadcast_a, float *__restrict__ out)
{
	constexpr int  TPR = MetricLanes<METRIC>::LANES;
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t pair = t / TPR;
	const int	   sub = t % TPR;
	if (n == 0) return;
	const uint32_t pp = pair < n ? pair : n - 1;
	const float	  *av = a + (broadcast_a ? 0 : (size_t) pp * a_stride);
	const float	  *bv = b + (size_t) pp * b_stride;
	float		   qn = 0.f, vn = 0.f;
	if (METRIC == M_COS)
	{
		qn = sqnorm_exact<4>(av, (int) dim, sub & 3);
		vn = sqnorm_exact<4>(bv, (int) dim, sub & 3);
	}
	const float d = distance_exact<METRIC, TPR>(av, bv, (int) dim, qn, vn, sub);
	if (pair < n && sub == 0) out[pair] = d;
}

// ---- gather distances: out[q][j] = dist(query q, stored node ids[q][j]) with cached norms ---------
template <int METRIC>
__global__ void dist_gather_kernel(const float *__restrict__ vectors, const float *__restrict__ norms, uint32_t row_f,
								   uint32_t dim, uint32_t n_items, const float *__restrict__ queries, uint32_t q_stride,
								   uint32_t nq, uint32_t k, const uint32_t *__restrict__ ids, float *__restrict__ out)
{
	constexpr int  TPR = MetricLanes<METRIC>::LANES;
	const uint64_t t = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	const uint64_t pair = t / TPR;
	const int	   sub = (int) (t % TPR);
	const uint64_t total = (uint64_t) nq * k;
	if (total == 0) return;
	const uint64_t pp = pair < total ? pair : total - 1;
	const uint32_t q = (uint32_t) (pp / k);
	uint32_t	   id = ids[pp];
	const bool	   ok = id < n_items;
	if (!ok) id = 0;
	const float *av = queries + (size_t) q * q_stride;
	const float *bv = vectors + (size_t) id * row_f;
	float		 qn = 0.f, vn = 0.f;
	if (METRIC == M_COS)
	{
		qn = sqnorm_exact<4>(av, (int) dim, sub & 3);
		vn = norms[id];
	}
	const float d = distance_exact<METRIC, TPR>(av, bv, (int) dim, qn, vn, sub);
	if (pair < total && sub == 0) out[pair] = ok ? d : __int_as_float(0x7fc00000);
}

// ---- exact scan (seq-scan `ORDER BY val <op> q LIMIT k`, embedding.c:1022-1062 + executor sort; knn.out:63-91) ----
// Step 1: out[q][j] = dist(query q, stored node r0 + j) for a chunk of nr rows, reference-exact arithmetic.
template <int METRIC>
__global__ void scan_dist_kernel(const float *__restrict__ vectors, const float *__restrict__ norms, uint32_t row_f, uint32_t dim,
								 const float *__restrict__ queries, uint32_t q_stride, uint32_t nq, uint32_t r0, uint32_t nr,
								 float *__restrict__ out)
{
	constexpr int  TPR = MetricLanes<METRIC>::LANES;
	const uint64_t t = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x;
	const uint64_t pair = t / TPR;
	const int	   sub = (int) (t % TPR);
	const uint64_t total = (uint64_t) nq * nr;
	if (total == 0) return;
	const uint64_t pp = pair < total ? pair : total - 1;  // clamp: all lanes of a warp take part in the shuffles
	const uint32_t q = (uint32_t) (pp / nr), j = (uint32_t) (pp % nr);
	const float	  *av = queries + (size_t) q * q_stride;
	const float	  *bv = vectors + (size_t) (r0 + j) * row_f;
	float		   qn = 0.f, vn = 0.f;
	if (METRIC == M_COS)
	{
		qn = sqnorm_exact<4>(av, (int) dim, sub & 3);
		vn = norms[r0 + j];
	}
	const float d = distance_exact<METRIC, TPR>(av, bv, (int) dim, qn, vn, sub);
	if (pair < total && sub == 0) out[pair] = d;
}

// Epilogue of the brute-force scan (both entry points; the host-pointer one copies its output back): the running top-k (order
// keys, labels, counts) in the caller's layout -- distances as floats, unused tail = (~0, +inf).
__global__ void scan_finish_kernel(const uint32_t *__restrict__ top_d, const uint64_t *__restrict__ top_l, const uint32_t *__restrict__ top_n, uint32_t nq,
								   uint32_t k, uint64_t *__restrict__ labels_out, float *__restrict__ dists_out, int32_t *__restrict__ n_out)
{
	const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (size_t) nq * k) return;
	const uint32_t q = (uint32_t) (i / k), j = (uint32_t) (i % k);
	const uint32_t n = top_n[q];
	const bool	   ok = j < n;
	labels_out[i] = ok ? top_l[i] : ~(uint64_t) 0;
	if (dists_out) dists_out[i] = ok ? o2f(top_d[i]) : INFINITY;
	if (j == 0) n_out[q] = (int32_t) n;
}

// Step 2: fold a chunk of distances into the running k smallest (dist,label) pairs of every query.
// One warp per query.  top_d holds f2o(dist); candidates better than the current worst pair are gathered in shared
// memory and merged by rank whenever the buffer fills (the threshold only tightens, so gathering with a stale
// threshold is conservative and the final set is exact).
constexpr uint32_t kScanCand = 256;
__global__ void scan_select_kernel(const float *__restrict__ dist, const uint64_t *__restrict__ labels, uint32_t nq, uint32_t r0,
								   uint32_t nr, uint32_t k, uint32_t *__restrict__ top_d, uint64_t *__restrict__ top_l,
								   uint32_t *__restrict__ top_n, uint32_t *__restrict__ tmp_d, uint64_t *__restrict__ tmp_l)
{
	__shared__ uint32_t cd[4][kScanCand];
	__shared__ uint64_t cl[4][kScanCand];
	const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const uint32_t q = blockIdx.x * 4 + w;
	if (q >= nq) return;
	uint32_t *td = top_d + (size_t) q * k, *sd = tmp_d + (size_t) q * k;
	uint64_t *tl = top_l + (size_t) q * k, *sl = tmp_l + (size_t) q * k;
	uint32_t  n = top_n[q];
	uint32_t  nc = 0;
	const uint32_t lt = (1u << lane) - 1u;
	auto less = [](uint32_t d1, uint64_t l1, uint32_t d2, uint64_t l2) { return d1 < d2 || (d1 == d2 && l1 < l2); };
	auto merge = [&]() {
		// rank every element of top (n) and cand (nc) in their union; keep ranks < k
		__syncwarp();
		const uint32_t total = n + nc;
		for (uint32_t i = lane; i < total; i += 32)
		{
			const bool	   from_top = i < n;
			const uint32_t d = from_top ? td[i] : cd[w][i - n];
			const uint64_t l = from_top ? tl[i] : cl[w][i - n];
			uint32_t	   rank = 0;
			for (uint32_t j = 0; j < n; j++) rank += (j != i && (less(td[j], tl[j], d, l) || (!less(d, l, td[j], tl[j]) && j < i))) ? 1u : 0u;
			for (uint32_t j = 0; j < nc; j++)
			{
				const uint32_t jj = n + j;
				rank += (jj != i && (less(cd[w][j], cl[w][j], d, l) || (!less(d, l, cd[w][j], cl[w][j]) && jj < i))) ? 1u : 0u;
			}
			if (rank < k) { sd[rank] = d; sl[rank] = l; }
		}
		__syncwarp();
		n = total < k ? total : k;
		for (uint32_t i = lane; i < n; i += 32) { td[i] = sd[i]; tl[i] = sl[i]; }
		nc = 0;
		__syncwarp();
	};
	for (uint32_t base = 0; base < nr; base += 32)
	{
		const uint32_t j = base + lane;
		bool		   take = false;
		uint32_t	   d = 0;
		uint64_t	   l = 0;
		if (j < nr)
		{
			l = labels[r0 + j];
			if (((l >> 48) & 1ull) == 0)
			{
				d = f2o(dist[(size_t) q * nr + j]);
				take = (n < k) || less(d, l, td[k - 1], tl[k - 1]);
			}
		}
		const uint32_t m = __ballot_sync(0xffffffffu, take);
		if (m)
		{
			if (nc + (uint32_t) __popc(m) > kScanCand) merge();
			// (after a merge the threshold is tighter; keeping the already tested candidates is still exact)
			if (take)
			{
				const uint32_t at = nc + __popc(m & lt);
				cd[w][at] = d;
				cl[w][at] = l;
			}
			nc += __popc(m);
		}
	}
	if (nc) merge();
	if (lane == 0) top_n[q] = n;
}

// ---- reference record layout (embedding.c:224-228, :619-621) <-> SoA --------------------------------
// record = [u32 count | u32 links[maxM] | f32 coords[dim] | u64 label], records `stride` bytes apart.
// One warp per record; byte-granular because the 8-byte label is only 4-byte aligned in general.
__global__ void records_unpack_kernel(const unsigned char *__restrict__ recs, size_t stride, uint32_t n, uint32_t first,
									  uint32_t dim, uint32_t maxM, uint32_t row_f, uint32_t link_stride,
									  float *__restrict__ vectors, uint32_t *__restrict__ links, uint64_t *__restrict__ labels)
{
	const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	if (w >= n) return;
	const unsigned char *rec = recs + (size_t) w * stride;
	const uint32_t		*rl = reinterpret_cast<const uint32_t *>(rec);
	const float			*rc = reinterpret_cast<const float *>(rec + (size_t) (maxM + 1) * 4);
	const uint32_t		*rlab = reinterpret_cast<const uint32_t *>(rec + (size_t) (maxM + 1) * 4 + (size_t) dim * 4);
	const size_t		 id = (size_t) first + w;
	for (uint32_t i = lane; i < link_stride; i += 32) links[id * link_stride + i] = (i <= maxM) ? rl[i] : 0u;
	for (uint32_t i = lane; i < row_f; i += 32) vectors[id * row_f + i] = (i < dim) ? rc[i] : 0.0f;
	if (lane == 0) labels[id] = (uint64_t) rlab[0] | ((uint64_t) rlab[1] << 32);
}

__global__ void records_pack_kernel(unsigned char *__restrict__ recs, size_t stride, uint32_t n, uint32_t first, uint32_t dim,
									uint32_t maxM, uint32_t row_f, uint32_t link_stride, const float *__restrict__ vectors,
									const uint32_t *__restrict__ links, const uint64_t *__restrict__ labels)
{
	const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	if (w >= n) return;
	unsigned char *rec = recs + (size_t) w * stride;
	uint32_t	  *rl = reinterpret_cast<uint32_t *>(rec);
	float		  *rc = reinterpret_cast<float *>(rec + (size_t) (maxM + 1) * 4);
	uint32_t	  *rlab = reinterpret_cast<uint32_t *>(rec + (size_t) (maxM + 1) * 4 + (size_t) dim * 4);
	const size_t   id = (size_t) first + w;
	for (uint32_t i = lane; i <= maxM; i += 32) rl[i] = links[id * link_stride + i];
	for (uint32_t i = lane; i < dim; i += 32) rc[i] = vectors[id * row_f + i];
	if (lane == 0)
	{
		const uint64_t l = labels[id];
		rlab[0] = (uint32_t) l;
		rlab[1] = (uint32_t) (l >> 32);
	}
}

// ---- K5: per-query merge of n_shards ascending (dist,label) lists of length k -------------------------
// Order = (dist,label) lexicographic, the pair order of searchKnn's result queue (hnswalg.cpp:236-247).
// One warp per query; rank of an element = its index in its own list + sum over the other lists of the
// number of smaller elements (binary search), so no sort is needed.
//
// The lists are addressed through one base pointer per shard, so the same kernel merges
//   * a buffer gathered by ONE NCCL all-gather (base + s * stride), and
//   * the peers' result buffers read DIRECTLY over NVLink (CUDA-IPC / peer-mapped pointers): then `flags` is this rank's
//     flag array -- flags[s] >= seq means shard s has published its lists of step `seq` (the peer's copy engine stores the
//     flag after its search kernel, in stream order) -- and every warp first waits for all its peers (ld.acquire.sys), so the
//     exchange needs no collective launch at all: merge = wait + peer loads + rank-by-counting in one kernel.
constexpr uint32_t kMaxShards = 16;
struct ShardLists
{
	const float	   *dist[kMaxShards];  // [nq][k]
	const uint64_t *lab[kMaxShards];   // [nq][k]
	const int32_t  *cnt[kMaxShards];   // [nq]
};

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t *p)
{
#ifdef PGEMB_HOST_EMULATION
	return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
	uint32_t v;
	asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
#endif
}

__global__ void merge_topk_lists_kernel(uint32_t nq, uint32_t n_shards, uint32_t k, const ShardLists in, const uint32_t *__restrict__ flags,
										uint32_t seq, uint32_t self, float *__restrict__ dout, uint64_t *__restrict__ lout,
										int32_t *__restrict__ nout, int *__restrict__ error_flag)
{
	const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	if (q >= nq) return;
	if (flags != nullptr)
	{
		// lane s waits for shard s (sequence numbers only grow; compared as a wrapping distance)
		if (lane < n_shards && lane != self)
		{
			uint32_t spins = 0;
			while ((int32_t) (ld_acquire_sys_u32(flags + lane) - seq) < 0)
			{
				__nanosleep(200);
				if (++spins > (16u << 20))	// seconds: a peer died or never searched -- flag it, do not hang the GPU
				{
					if (error_flag) *error_flag = 5;
					break;
				}
			}
		}
		__syncwarp();
	}
	uint32_t total = 0;
	for (uint32_t s = 0; s < n_shards; s++) total += (uint32_t) max(0, min((int32_t) k, in.cnt[s][q]));
	const uint32_t keep = min(total, k);
	for (uint32_t e = lane; e < n_shards * k; e += 32)
	{
		const uint32_t s = e / k, i = e % k;
		const uint32_t ns = (uint32_t) max(0, min((int32_t) k, in.cnt[s][q]));
		if (i >= ns) continue;
		const size_t   base = (size_t) q * k;
		const float	   fd = in.dist[s][base + i];
		const uint32_t od = f2o(fd);
		const uint64_t ol = in.lab[s][base + i];
		uint32_t	   rank = i;
		for (uint32_t s2 = 0; s2 < n_shards; s2++)
		{
			if (s2 == s) continue;
			const uint32_t	n2 = (uint32_t) max(0, min((int32_t) k, in.cnt[s2][q]));
			const float	   *d2p = in.dist[s2] + base;
			const uint64_t *l2p = in.lab[s2] + base;
			uint32_t		lo = 0, hi = n2;
			while (lo < hi)
			{
				const uint32_t mid = (lo + hi) >> 1;
				const uint32_t d2 = f2o(d2p[mid]);
				const uint64_t l2 = l2p[mid];
				// element of another shard sorts first if smaller, or equal with the lower shard index
				const bool less = d2 < od || (d2 == od && (l2 < ol || (l2 == ol && s2 < s)));
				if (less) lo = mid + 1; else hi = mid;
			}
			rank += lo;
		}
		if (rank < keep)
		{
			dout[(size_t) q * k + rank] = fd;
			lout[(size_t) q * k + rank] = ol;
		}
	}
	for (uint32_t i = keep + lane; i < k; i += 32)
	{
		dout[(size_t) q * k + i] = __int_as_float(0x7f800000);
		lout[(size_t) q * k + i] = ~0ull;
	}
	if (lane == 0) nout[q] = (int32_t) keep;
}

}  // namespace pgemb
