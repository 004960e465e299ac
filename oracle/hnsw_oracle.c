/*
 * hnsw_oracle.c -- CPU restatement ("port") of pg_embedding's HNSW hot path in plain C.
 *
 * TEST INFRASTRUCTURE ONLY: the checker for the CUDA path.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  It is never the thing shipped.
 *
 * Parity status: PINNED.  tests/test_oracle_*.py check this file (a) against the reference's own
 * golden results (test/expected/knn.out, gh-2.out, gh-3.out) and (b) bit-for-bit -- distances, link
 * lists and result labels -- against the UNMODIFIED reference sources compiled in place into
 * oracle/_ref/libpgemb_ref.so (see oracle/Makefile).
 *
 * What is restated (reference file:line):
 *   hnsw_dist_func + the three metrics ........ distfunc.c:28-65, :133-155, :157-174
 *   searchBaseLayer ........................... hnswalg.cpp:42-114
 *   getNeighborsByHeuristic ................... hnswalg.cpp:117-153
 *   mutuallyConnectNewElement ................. hnswalg.cpp:155-223
 *   bindPoint / hnsw_bind_point ............... hnswalg.cpp:225-232, :279-291
 *   searchKnn / hnsw_search ................... hnswalg.cpp:234-277
 *
 * FLOATING-POINT ORDER.  The reference builds distfunc.c with -Ofast (reference Makefile:14), so the
 * order of the fp32 additions is whatever the compiler's vectoriser chose, not the source order.
 * The orders below are those of the reference object as built by oracle/Makefile in this image
 * (gcc 13.3, x86-64, `gcc -Ofast`; read off `objdump -d`, summarised in DESIGN.md section 4).  They are
 * written out explicitly and this file is compiled WITHOUT fast-math / fp-contraction, so it
 * reproduces that object bit-for-bit; the CUDA kernels implement the same orders.
 *
 *   L2 (AVX2 path, selected by __builtin_cpu_supports("avx2"), distfunc.c:162):
 *       8 lane accumulators S[j]; per 16-float block  S[j] += (d[j]^2 + d[8+j]^2)
 *       (the two products are added to each other FIRST, then to the accumulator; no FMA);
 *       horizontal: t[j]=S[j]+S[j+4] (j<4);  res=(t0+t2)+(t1+t3);
 *       tail r=dim%16: if r>=8 one 8-wide block E[k]=d^2 folded to u[j]=E[j]+E[j+4];
 *                      rem=r%8: if rem>=4: res += hsum4(F[j]+u[j]) with F the next 4 squares
 *                               else if r>=8: res = hsum4(u) + res;
 *                      then the last rem%4 squares are added one by one;  sqrtf.
 *   cosine:  4 lane accumulators each for dot, |a|^2, |b|^2 (mul then add, no FMA);
 *            hsum4(s)=(s0+s2)+(s1+s3); tail dim%4 added one by one;
 *            result = (float)(1.0 - (double)dot / sqrt((double)(nb*na)))   [nb*na in fp32]
 *   manhattan: 4 lane accumulators of |a-b| (fp32), hsum4, tail one by one.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdbool.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>

#include "embedding.h"

/* ======================================================================================
 * Distances
 * ==================================================================================== */

static inline float
hsum4(const float s[4])
{
	return (s[0] + s[2]) + (s[1] + s[3]);
}

/* distfunc.c:28-65 as compiled (see header comment). */
static float
l2_dist_avx2_order(const float *x, const float *y, size_t n)
{
	float  S[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	float  t[4], u[4] = {0, 0, 0, 0};
	float  res;
	size_t main_n = (n / 16) * 16;
	size_t r = n - main_n;
	size_t pos;
	size_t rem;
	bool   have8;

	for (size_t i = 0; i < main_n; i += 16)
		for (int j = 0; j < 8; j++)
		{
			float d0 = x[i + j] - y[i + j];
			float d1 = x[i + 8 + j] - y[i + 8 + j];
			float p0 = d0 * d0;
			float p1 = d1 * d1;
			float pp = p0 + p1;

			S[j] = S[j] + pp;
		}
	for (int j = 0; j < 4; j++)
		t[j] = S[j] + S[j + 4];
	res = (t[0] + t[2]) + (t[1] + t[3]);

	if (r == 0)
		return sqrtf(res);

	pos = main_n;
	have8 = r >= 8;
	if (have8)
	{
		float E[8];

		for (int k = 0; k < 8; k++)
		{
			float d = x[pos + k] - y[pos + k];

			E[k] = d * d;
		}
		for (int j = 0; j < 4; j++)
			u[j] = E[j] + E[j + 4];
		pos += 8;
	}
	rem = r - (have8 ? 8 : 0);
	if (rem >= 4)
	{
		float w[4];

		for (int j = 0; j < 4; j++)
		{
			float d = x[pos + j] - y[pos + j];
			float F = d * d;

			w[j] = F + u[j];
		}
		res = res + hsum4(w);
		pos += 4;
		rem -= 4;
	}
	else if (have8)
		res = hsum4(u) + res;

	for (size_t k = 0; k < rem; k++)
	{
		float d = x[pos + k] - y[pos + k];

		res = res + d * d;
	}
	return sqrtf(res);
}

/* The three lane-strided partial sums of distfunc.c:133-145; exposed so that the norms can be
 * checked separately (the CUDA path caches |b|^2 per stored node -- same bits, DESIGN.md section 4). */
static void
cosine_sums(const float *a, const float *b, size_t n, float *dot_out, float *na_out, float *nb_out)
{
	float  sd[4] = {0, 0, 0, 0}, sa[4] = {0, 0, 0, 0}, sb[4] = {0, 0, 0, 0};
	float  dot, na, nb;
	size_t main_n = (n / 4) * 4;

	if (n <= 3)
		main_n = 0; /* the vector loop is skipped for dim<=3 (same result: it would run 0 times) */
	for (size_t i = 0; i < main_n; i += 4)
		for (int j = 0; j < 4; j++)
		{
			float av = a[i + j], bv = b[i + j];

			sd[j] = sd[j] + bv * av;
			sb[j] = sb[j] + bv * bv;
			sa[j] = sa[j] + av * av;
		}
	dot = hsum4(sd);
	na = hsum4(sa);
	nb = hsum4(sb);
	for (size_t k = main_n; k < n; k++)
	{
		float av = a[k], bv = b[k];

		dot = dot + av * bv;
		na = na + av * av;
		nb = nb + bv * bv;
	}
	*dot_out = dot;
	*na_out = na;
	*nb_out = nb;
}

static inline float
cosine_finish(float dot, float na, float nb)
{
	float prod = nb * na;

	return (float) (1.0 - (double) dot / sqrt((double) prod));
}

static float
cosine_dist_order(const float *a, const float *b, size_t n)
{
	float dot, na, nb;

	cosine_sums(a, b, n, &dot, &na, &nb);
	return cosine_finish(dot, na, nb);
}

/* distfunc.c:147-155 as compiled. */
static float
manhattan_dist_order(const float *a, const float *b, size_t n)
{
	float  s[4] = {0, 0, 0, 0};
	float  res;
	size_t main_n = (n / 4) * 4;

	for (size_t i = 0; i < main_n; i += 4)
		for (int j = 0; j < 4; j++)
			s[j] = s[j] + fabsf(a[i + j] - b[i + j]);
	res = hsum4(s);
	for (size_t k = main_n; k < n; k++)
		res = res + fabsf(a[k] - b[k]);
	return res;
}

/* distfunc.c:159-174 */
void
hnsw_init_dist_func(void)
{
}

dist_t
hnsw_dist_func(dist_func_t dist, coord_t const *ax, coord_t const *bx, size_t dim)
{
	switch (dist)
	{
		case DIST_L2:
			return l2_dist_avx2_order(ax, bx, dim);
		case DIST_COSINE:
			return cosine_dist_order(ax, bx, dim);
		case DIST_MANHATTAN:
			return manhattan_dist_order(ax, bx, dim);
	}
	return NAN;
}

/* Squared-norm in the cosine lane order (what the CUDA path stores per node). */
float
oracle_cosine_norm(const float *b, size_t n)
{
	float dot, na, nb;

	cosine_sums(b, b, n, &dot, &na, &nb);
	return nb;
}

float
oracle_cosine_from_parts(const float *a, const float *b, size_t n)
{
	/* dist recomposed from separately computed parts -- must equal cosine_dist_order bit for bit */
	float dot, na, nb, na2, nb2, tmp;

	cosine_sums(a, b, n, &dot, &tmp, &tmp);
	na = oracle_cosine_norm(a, n);
	nb = oracle_cosine_norm(b, n);
	(void) na2;
	(void) nb2;
	return cosine_finish(dot, na, nb);
}

/* ======================================================================================
 * A max-heap of (dist, id) pairs with std::pair's lexicographic order (hnswalg.cpp:52-53).
 * Any correct heap gives the reference's results: all operations are push / top / pop-max and
 * the pairs in a queue are distinct (ids are unique per queue).
 * ==================================================================================== */

typedef struct
{
	float	 d;
	uint64_t id; /* idx_t or label_t */
} Pair;

typedef struct
{
	Pair  *v;
	size_t n, cap;
} Heap;

static inline bool
pair_less(Pair a, Pair b)
{
	return a.d < b.d || (!(b.d < a.d) && a.id < b.id);
}

static void
heap_push(Heap *h, float d, uint64_t id)
{
	size_t i;

	if (h->n == h->cap)
	{
		h->cap = h->cap ? h->cap * 2 : 64;
		h->v = (Pair *) realloc(h->v, h->cap * sizeof(Pair));
	}
	i = h->n++;
	h->v[i].d = d;
	h->v[i].id = id;
	while (i > 0)
	{
		size_t p = (i - 1) / 2;
		Pair   tmp;

		if (!pair_less(h->v[p], h->v[i]))
			break;
		tmp = h->v[p];
		h->v[p] = h->v[i];
		h->v[i] = tmp;
		i = p;
	}
}

static Pair
heap_pop(Heap *h)
{
	Pair   top = h->v[0];
	size_t i = 0;

	h->v[0] = h->v[--h->n];
	for (;;)
	{
		size_t l = 2 * i + 1, r = l + 1, m = i;
		Pair   tmp;

		if (l < h->n && pair_less(h->v[m], h->v[l]))
			m = l;
		if (r < h->n && pair_less(h->v[m], h->v[r]))
			m = r;
		if (m == i)
			break;
		tmp = h->v[m];
		h->v[m] = h->v[i];
		h->v[i] = tmp;
		i = m;
	}
	return top;
}

static void
heap_free(Heap *h)
{
	free(h->v);
	h->v = NULL;
	h->n = h->cap = 0;
}

/* ======================================================================================
 * searchBaseLayer (hnswalg.cpp:42-114)
 * ==================================================================================== */

static Heap
search_base_layer(HnswMetadata *meta, const coord_t *point, size_t ef)
{
	Heap	  top = {0}, cand = {0};
	size_t	  vwords = 64 * 1024; /* hnswalg.cpp:46 */
	uint32_t *visited = (uint32_t *) calloc(vwords, sizeof(uint32_t));
	coord_t	 *coords;
	idx_t	 *links;
	idx_t	  ep = meta->enterpoint_node;
	float	  d, lower;

	if (!hnsw_begin_read(meta, ep, NULL, &coords, NULL)) /* empty index, hnswalg.cpp:56-57 */
	{
		free(visited);
		return top;
	}
	d = hnsw_dist_func(meta->dist_func, point, coords, meta->dim);
	hnsw_end_read(meta);

	heap_push(&top, d, ep);
	heap_push(&cand, -d, ep);
	visited[ep >> 5] = 1u << (ep & 31);
	lower = d;

	while (cand.n > 0)
	{
		Pair   c = cand.v[0];
		size_t cnt;

		if (-c.d > lower) /* hnswalg.cpp:70 */
			break;
		heap_pop(&cand);

		hnsw_begin_read(meta, (idx_t) c.id, &links, NULL, NULL);
		cnt = links[0];
		for (size_t j = 0; j < cnt; j++) /* pass 1: grow the bitset + prefetch, hnswalg.cpp:79-88 */
		{
			size_t t = links[1 + j];

			if (vwords <= (t >> 5))
			{
				size_t nw = (t >> 5) + 1;

				visited = (uint32_t *) realloc(visited, nw * sizeof(uint32_t));
				memset(visited + vwords, 0, (nw - vwords) * sizeof(uint32_t));
				vwords = nw;
			}
			if (!(visited[t >> 5] & (1u << (t & 31))))
				hnsw_prefetch(meta, (idx_t) t);
		}
		for (size_t j = 0; j < cnt; j++) /* pass 2: score, hnswalg.cpp:89-110 */
		{
			size_t t = links[1 + j];

			if (visited[t >> 5] & (1u << (t & 31)))
				continue;
			visited[t >> 5] |= 1u << (t & 31);

			hnsw_begin_read(meta, (idx_t) t, NULL, &coords, NULL);
			d = hnsw_dist_func(meta->dist_func, point, coords, meta->dim);
			hnsw_end_read(meta);

			if (top.v[0].d > d || top.n < ef) /* hnswalg.cpp:99 */
			{
				heap_push(&cand, -d, t);
				heap_push(&top, d, t);
				if (top.n > ef)
					heap_pop(&top);
				lower = top.v[0].d;
			}
		}
		hnsw_end_read(meta);
	}
	heap_free(&cand);
	free(visited);
	return top;
}

/* ======================================================================================
 * getNeighborsByHeuristic (hnswalg.cpp:117-153)
 * ==================================================================================== */

static void
select_neighbors_heuristic(HnswMetadata *meta, Heap *top, size_t NN)
{
	Heap   byNear = {0};
	Pair  *kept;
	size_t nkept = 0;

	if (top->n < NN) /* hnswalg.cpp:119-120 (note: == NN still prunes) */
		return;

	while (top->n > 0)
	{
		Pair p = heap_pop(top);

		heap_push(&byNear, -p.d, p.id);
	}
	kept = (Pair *) malloc(sizeof(Pair) * (NN ? NN : 1));
	while (byNear.n > 0 && nkept < NN)
	{
		Pair  c = heap_pop(&byNear); /* nearest first; equal distance -> larger id first */
		float dq = -c.d;
		bool  good = true;

		for (size_t k = 0; k < nkept; k++)
		{
			coord_t *pc, *pr;
			float	 dd;

			hnsw_begin_read(meta, (idx_t) kept[k].id, NULL, &pr, NULL);
			hnsw_begin_read(meta, (idx_t) c.id, NULL, &pc, NULL);
			dd = hnsw_dist_func(meta->dist_func, pr, pc, meta->dim);
			hnsw_end_read(meta);
			hnsw_end_read(meta);
			if (dd < dq)
			{
				good = false;
				break;
			}
		}
		if (good)
			kept[nkept++] = c;
	}
	for (size_t k = 0; k < nkept; k++)
		heap_push(top, -kept[k].d, kept[k].id);
	free(kept);
	heap_free(&byNear);
}

/* ======================================================================================
 * mutuallyConnectNewElement (hnswalg.cpp:155-223).  Returns false where the reference throws.
 * ==================================================================================== */

static bool
connect_new_element(HnswMetadata *meta, const coord_t *point, idx_t cur, Heap *top)
{
	idx_t  *sel;
	size_t	nsel = 0;
	idx_t  *links;
	coord_t *pc, *pn;

	(void) point;
	select_neighbors_heuristic(meta, top, meta->M);

	sel = (idx_t *) malloc(sizeof(idx_t) * (top->n ? top->n : 1));
	while (top->n > 0) /* farthest first, hnswalg.cpp:164-167 */
		sel[nsel++] = (idx_t) heap_pop(top).id;

	hnsw_begin_write(meta, cur, &links, NULL, NULL);
	if (links[0] != 0) /* "Should be blank", hnswalg.cpp:170-171 */
		goto fail_write;
	links[0] = (idx_t) nsel;
	for (size_t k = 0; k < nsel; k++)
	{
		if (links[1 + k] != 0) /* hnswalg.cpp:176-177 */
			goto fail_write;
		links[1 + k] = sel[k];
	}
	hnsw_end_write(meta);

	for (size_t k = 0; k < nsel; k++)
	{
		size_t maxM = meta->maxM;
		idx_t  cnt;

		if (sel[k] == cur) /* hnswalg.cpp:183-184 */
		{
			free(sel);
			return false;
		}
		hnsw_begin_write(meta, sel[k], &links, &pn, NULL);
		cnt = links[0];
		if (cnt > maxM) /* hnswalg.cpp:190-191 */
			goto fail_write;
		if (cnt < maxM)
		{
			links[1 + cnt] = cur; /* hnswalg.cpp:193-195 */
			links[0] = cnt + 1;
		}
		else
		{
			Heap   candidates = {0};
			float  dmax;
			size_t w = 0;

			hnsw_begin_read(meta, cur, NULL, &pc, NULL);
			dmax = hnsw_dist_func(meta->dist_func, pc, pn, meta->dim);
			hnsw_end_read(meta);
			heap_push(&candidates, dmax, cur);
			for (size_t j = 0; j < cnt; j++)
			{
				hnsw_begin_read(meta, links[1 + j], NULL, &pc, NULL);
				heap_push(&candidates, hnsw_dist_func(meta->dist_func, pc, pn, meta->dim), links[1 + j]);
				hnsw_end_read(meta);
			}
			select_neighbors_heuristic(meta, &candidates, maxM);
			while (candidates.n > 0) /* farthest first, hnswalg.cpp:213-219 */
				links[1 + w++] = (idx_t) heap_pop(&candidates).id;
			links[0] = (idx_t) w;
			heap_free(&candidates);
		}
		hnsw_end_write(meta);
	}
	free(sel);
	return true;

fail_write:
	hnsw_end_write(meta);
	free(sel);
	return false;
}

/* hnswalg.cpp:225-232, :279-291 */
bool
hnsw_bind_point(HnswMetadata *meta, const coord_t *point, idx_t cur)
{
	Heap top;
	bool ok;

	if (cur == 0)
		return true;
	top = search_base_layer(meta, point, meta->efConstruction);
	ok = connect_new_element(meta, point, cur, &top);
	heap_free(&top);
	if (!ok)
		fprintf(stderr, "oracle: bind_point(%u) failed\n", cur);
	return ok;
}

/* hnswalg.cpp:234-277 */
bool
hnsw_search(HnswMetadata *meta, const coord_t *point, size_t *n_results, label_t **results)
{
	size_t k = meta->efSearch;
	Heap   cands = search_base_layer(meta, point, k);
	Heap   byLabel = {0};
	size_t n;

	while (cands.n > k)
		heap_pop(&cands);
	while (cands.n > 0)
	{
		Pair	p = heap_pop(&cands);
		label_t label;

		hnsw_begin_read(meta, (idx_t) p.id, NULL, NULL, &label);
		if (!hnsw_is_deleted(label)) /* post-filter, hnswalg.cpp:245 */
			heap_push(&byLabel, p.d, label);
		hnsw_end_read(meta);
	}
	n = byLabel.n;
	*results = (label_t *) malloc((n ? n : 1) * sizeof(label_t));
	if (*results == NULL)
	{
		heap_free(&cands);
		heap_free(&byLabel);
		return false;
	}
	for (size_t i = n; i-- != 0;) /* ascending by (distance, label), hnswalg.cpp:265-269 */
		(*results)[i] = heap_pop(&byLabel).id;
	*n_results = n;
	heap_free(&cands);
	heap_free(&byLabel);
	return true;
}

/* Extension for tests: the same search but also returning distances and internal ids
 * (before the label lookup), ascending by (dist, id). Returns count. */
long
oracle_search_ids(HnswMetadata *meta, const coord_t *point, size_t ef, idx_t *ids_out, dist_t *dists_out)
{
	Heap   top = search_base_layer(meta, point, ef);
	size_t n;

	while (top.n > ef)
		heap_pop(&top);
	n = top.n;
	for (size_t i = n; i-- != 0;)
	{
		Pair p = heap_pop(&top);

		ids_out[i] = (idx_t) p.id;
		dists_out[i] = p.d;
	}
	heap_free(&top);
	return (long) n;
}

/* Extension for tests: one batch of pgemb_build_bulk (include/pgemb_b200.h) on the stored, unbound nodes
 * [first, first+n), stated with the primitives above.  Every member runs bindPoint's search against the graph
 * as it was when the batch started; then each member, in id order, runs mutuallyConnectNewElement on its own
 * search result.  This is the CUDA batch exactly: the members' link lists are blank and no stored list names
 * them, so no search of the batch can reach one, and no member is ever a back-link target.  Hence a member's
 * own list depends only on its search and on vectors, and every target takes its back-links in source-id
 * order -- the order here.  Node 0 is skipped (hnswalg.cpp:227-228).  Returns 0, or -2 where the reference
 * would throw. */
int
oracle_bind_batch(HnswMetadata *meta, idx_t first, size_t n)
{
	Heap *tops = (Heap *) calloc(n ? n : 1, sizeof(Heap));
	bool  ok = true;

	for (size_t i = 0; i < n; i++)
	{
		coord_t *pc;

		if (first + i == 0)
			continue;
		hnsw_begin_read(meta, (idx_t) (first + i), NULL, &pc, NULL);
		tops[i] = search_base_layer(meta, pc, meta->efConstruction);
		hnsw_end_read(meta);
	}
	for (size_t i = 0; i < n; i++)
	{
		if (first + i != 0)
			ok = connect_new_element(meta, NULL, (idx_t) (first + i), &tops[i]) && ok;
		heap_free(&tops[i]);
	}
	free(tops);
	return ok ? 0 : -2;
}
