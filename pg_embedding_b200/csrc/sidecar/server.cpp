// pgemb_sidecar -- the GPU-owning process behind libpgemb_client.so (protocol: ipc.h).
//
// It holds one device index (pgemb_index, the HBM mirror of a relation's graph) per relation key and serves the
// requests backends publish in shared memory.  Searches that are pending at the same time -- the reference issues
// hnsw_search one query per call, one call per backend at a time (embedding.c:317,335) -- are gathered per
// (relation, efSearch) into ONE pgemb_search_batch launch: a single query cannot fill an H100, the concurrent queries
// of many backends can (DESIGN.md section 6).  Index-less scans (`ORDER BY val <op> q LIMIT k` without the index) are
// gathered the same way per (relation, metric, k) into ONE pgemb_scan_topk_op call: every scan reads the whole table, so sharing
// that read pays even more there (DESIGN.md section 12).  The SQL distance operators' hnsw_dist_func calls (one pair each,
// embedding.c:1022-1062) are gathered per (metric, dim) into ONE pgemb_dist_batch call.  Everything else (mirror maintenance,
// hnsw_bind_point, link write-back) is run one request at a time, which is also the reference's rule for writers
// (embedding.c:627-629: X-lock on page 0).
//
// The library that does the work is dlopen()ed (--lib, default: libpgemb_b200.so next to this executable), so the
// same binary serves the product library on the GPU and, in the CPU test-suite, the host-emulated build of it.
// There is no computation in this file: no CPU fallback exists here either.
#include <dlfcn.h>
#include <errno.h>
#include <fcntl.h>
#include <linux/futex.h>
#include <signal.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../../include/pgemb_b200.h"
#include "ipc.h"

namespace {

// ---- the C ABI, resolved from the dlopen()ed library (include/pgemb_b200.h) ----------------------------------------
struct Api
{
	const char *(*last_error)(void);
	const char *(*version)(void);
	int (*device_count)(void);
	pgemb_status (*index_create)(const HnswMetadata *, size_t, int, pgemb_index **);
	void (*index_destroy)(pgemb_index *);
	size_t (*index_size)(const pgemb_index *);
	size_t (*index_capacity)(const pgemb_index *);
	pgemb_status (*append_records)(pgemb_index *, size_t, const void *, size_t);
	pgemb_status (*export_records)(const pgemb_index *, size_t, size_t, void *, size_t);
	pgemb_status (*get_links)(const pgemb_index *, size_t, size_t, idx_t *);
	pgemb_status (*set_labels)(pgemb_index *, size_t, size_t, const label_t *);
	pgemb_status (*truncate)(pgemb_index *);
	pgemb_status (*reserve)(pgemb_index *, size_t);
	pgemb_status (*search_batch)(pgemb_index *, size_t, const coord_t *, size_t, label_t *, dist_t *, idx_t *, int32_t *, uint32_t *);
	pgemb_status (*scan_topk_op)(pgemb_index *, dist_func_t, size_t, const coord_t *, size_t, label_t *, dist_t *, int32_t *);
	pgemb_status (*dist_batch)(dist_func_t, size_t, size_t, const coord_t *, int, const coord_t *, dist_t *);
	bool (*bind_point)(HnswMetadata *, const coord_t *, idx_t);	 // the reference-shaped hnsw_bind_point
	pgemb_status (*build_bulk)(pgemb_index *, size_t, size_t, size_t, double *);
	pgemb_status (*build_exact)(pgemb_index *, size_t, size_t, size_t, double *, uint64_t *);
	void (*init_dist_func)(void);
};

template <typename F> bool sym(void *h, const char *name, F &out)
{
	out = reinterpret_cast<F>(dlsym(h, name));
	if (!out) fprintf(stderr, "pgemb_sidecar: %s is not exported by the library\n", name);
	return out != nullptr;
}

bool load_api(const char *path, Api &a)
{
	void *h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
	if (!h)
	{
		fprintf(stderr, "pgemb_sidecar: cannot load %s: %s\n", path, dlerror());
		return false;
	}
	return sym(h, "pgemb_last_error", a.last_error) && sym(h, "pgemb_version", a.version) && sym(h, "pgemb_device_count", a.device_count) &&
		   sym(h, "pgemb_index_create", a.index_create) && sym(h, "pgemb_index_destroy", a.index_destroy) && sym(h, "pgemb_index_size", a.index_size) &&
		   sym(h, "pgemb_index_capacity", a.index_capacity) && sym(h, "pgemb_index_append_records", a.append_records) &&
		   sym(h, "pgemb_index_export_records", a.export_records) && sym(h, "pgemb_index_get_links", a.get_links) &&
		   sym(h, "pgemb_index_set_labels", a.set_labels) && sym(h, "pgemb_index_truncate", a.truncate) && sym(h, "pgemb_index_reserve", a.reserve) && sym(h, "pgemb_search_batch", a.search_batch) &&
		   sym(h, "pgemb_scan_topk_op", a.scan_topk_op) && sym(h, "pgemb_dist_batch", a.dist_batch) && sym(h, "hnsw_bind_point", a.bind_point) && sym(h, "pgemb_build_bulk", a.build_bulk) && sym(h, "pgemb_build_exact", a.build_exact) &&
		   sym(h, "hnsw_init_dist_func", a.init_dist_func);
}

// ---- shared-memory helpers -----------------------------------------------------------------------------------------
inline uint32_t ld(const uint32_t *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void		st(uint32_t *p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }

long futex(uint32_t *addr, int op, uint32_t val, const struct timespec *ts) { return syscall(SYS_futex, addr, op, val, ts, nullptr, 0); }

double now_s()
{
	struct timespec t;
	clock_gettime(CLOCK_MONOTONIC, &t);
	return (double) t.tv_sec + 1e-9 * (double) t.tv_nsec;
}

volatile sig_atomic_t g_stop = 0;
void				  on_signal(int) { g_stop = 1; }

// A batched group: (PGEMB_OP_SEARCH, relation, ef, 0), (PGEMB_OP_SCAN, relation, k, metric code) or (PGEMB_OP_DIST, metric, dim, 0).
// A scan's metric code is ipc.h's a1: 1 + dist_func_t, or 0 = the mirror's metric (resolved by collect() when the mirror exists).
using GroupKey = std::tuple<uint32_t, uint64_t, uint64_t, uint64_t>;

struct Server
{
	Api				api;
	PgembIpcHeader *hdr = nullptr;
	unsigned char  *base = nullptr;
	size_t			bytes = 0;
	int				device = 0;
	size_t			max_batch = 4096;
	long			linger_us = 50;	 // upper bound of the adaptive wait for the callers that are about to resubmit (0 = never wait)
	size_t			target = 1;		 // how many concurrent searchers the recent rounds showed (see serve_once)
	double			last_service_s = 0.0;	// duration of the previous round's launches
	size_t			carry = 0;				// searches that queued up while the current round's launches ran
	bool			carry_counted = false;
	std::unordered_map<uint64_t, PgembHostIndex> mirrors;  // {meta, dev}: what the reference-shaped entry points down-cast their HnswMetadata* to
	// per-batch scratch
	std::vector<float>	  qbuf;
	std::vector<float>	  bbuf;	 // second vectors of the distance pairs
	std::vector<label_t>  lbuf;
	std::vector<float>	  dbuf;
	std::vector<int32_t>  nbuf;

	PgembIpcSlot *slot(uint32_t i) const { return reinterpret_cast<PgembIpcSlot *>(base + hdr->slots_off + (size_t) i * hdr->slot_stride); }
	float		 *slot_vec(PgembIpcSlot *s) const { return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s) + pgemb_ipc_payload_vec_off()); }
	label_t		 *slot_labels(PgembIpcSlot *s) const
	{
		return reinterpret_cast<label_t *>(reinterpret_cast<unsigned char *>(s) + pgemb_ipc_payload_labels_off(hdr->max_dim));
	}
	float *slot_dists(PgembIpcSlot *s) const
	{
		return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s) + pgemb_ipc_payload_dists_off(hdr->max_dim, hdr->max_ef));
	}
	unsigned char *bulk() const { return base + hdr->bulk_off; }

	void finish(PgembIpcSlot *s, pgemb_status status, const char *msg)
	{
		s->status = status;
		if (status != PGEMB_OK)
		{
			snprintf(s->err, sizeof(s->err), "%s", msg ? msg : "");
		}
		else
			s->err[0] = 0;
		__atomic_fetch_add(&hdr->n_requests, 1, __ATOMIC_RELAXED);
		st(&s->state, PGEMB_SLOT_DONE);
		__atomic_thread_fence(__ATOMIC_SEQ_CST);
		if (ld(&s->abandoned))
		{
			// the client stopped waiting (cancelled query): nobody will read the result
			const uint32_t op = s->op, owner = (uint32_t) s->owner_pid;
			uint32_t	   expect = PGEMB_SLOT_DONE;
			// FREE slots carry no pid: the next claimer stores its own AFTER its CAS, and reclaim() must not judge it by ours.
			// (If the client's own CAS wins the race instead, the pid it leaves behind is that of a live backend.)
			__atomic_store_n(&s->owner_pid, 0, __ATOMIC_RELEASE);
			if (__atomic_compare_exchange_n(&s->state, &expect, (uint32_t) PGEMB_SLOT_FREE, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED))
			{
				// we freed the slot (not the client): a bulk request's hold on the bulk area ends with it
				const bool bulk_op = op == PGEMB_OP_APPEND_RECORDS || op == PGEMB_OP_GET_LINKS || op == PGEMB_OP_EXPORT_RECORDS || op == PGEMB_OP_SET_LABELS;
				uint32_t   o = owner;
				if (bulk_op) __atomic_compare_exchange_n(&hdr->bulk_lock, &o, 0u, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED);
			}
			return;
		}
		futex(&s->state, FUTEX_WAKE, 1, nullptr);
	}
	void finish_api(PgembIpcSlot *s, pgemb_status status) { finish(s, status, status == PGEMB_OK ? nullptr : api.last_error()); }

	PgembHostIndex *find(PgembIpcSlot *s)
	{
		auto it = mirrors.find(s->index_key);
		if (it == mirrors.end())
		{
			finish(s, PGEMB_ERR_ARG, "no device index attached for this relation key");
			return nullptr;
		}
		return &it->second;
	}

	bool bulk_owned_by(PgembIpcSlot *s, size_t need)
	{
		if (ld(&hdr->bulk_lock) != (uint32_t) s->owner_pid || need > hdr->bulk_bytes)
		{
			finish(s, PGEMB_ERR_ARG, "bulk area not held by the requester or request larger than the bulk area");
			return false;
		}
		return true;
	}

	// ---- everything except searches, scans and distances: one at a time, in slot order ----------------------------
	void run_control(PgembIpcSlot *s)
	{
		PgembHostIndex *m = nullptr;
		switch (s->op)
		{
			// the requests on an attached mirror
			case PGEMB_OP_APPEND_RECORDS:
			case PGEMB_OP_BIND:
			case PGEMB_OP_GET_LINKS:
			case PGEMB_OP_EXPORT_RECORDS:
			case PGEMB_OP_SET_LABELS:
			case PGEMB_OP_TRUNCATE:
			case PGEMB_OP_SIZE:
			case PGEMB_OP_BUILD:
				if (!(m = find(s))) return;
		}
		switch (s->op)
		{
			case PGEMB_OP_PING: finish(s, PGEMB_OK, nullptr); return;
			case PGEMB_OP_ATTACH:
			{
				HnswMetadata meta;
				memcpy(&meta, slot_vec(s), sizeof(meta));
				auto it = mirrors.find(s->index_key);
				if (it != mirrors.end())
				{
					// the reference checks {dims, maxM} of an existing index against the options (embedding.c:594-602)
					const HnswMetadata &have = it->second.meta;
					if (have.dim != meta.dim || have.maxM != meta.maxM || have.dist_func != meta.dist_func)
					{
						finish(s, PGEMB_ERR_ARG, "attach: dims / maxM / distance function differ from the attached index");
						return;
					}
				}
				else
				{
					if (meta.dim < 1 || meta.dim > hdr->max_dim)
					{
						finish(s, PGEMB_ERR_ARG, "attach: dims outside the sidecar's --max-dim");
						return;
					}
					PgembHostIndex created = {meta, nullptr};
					const pgemb_status r = api.index_create(&meta, (size_t) s->a0, device, &created.dev);
					if (r != PGEMB_OK)
					{
						finish_api(s, r);
						return;
					}
					it = mirrors.emplace(s->index_key, created).first;
				}
				if ((size_t) s->a0 > api.index_capacity(it->second.dev))
				{
					// the relation has grown beyond the mirror: make room (ids and contents are kept)
					const pgemb_status r = api.reserve(it->second.dev, (size_t) s->a0);
					if (r != PGEMB_OK)
					{
						finish_api(s, r);
						return;
					}
				}
				s->a1 = api.index_size(it->second.dev);
				s->a2 = api.index_capacity(it->second.dev);
				finish(s, PGEMB_OK, nullptr);
				return;
			}
			case PGEMB_OP_APPEND_RECORDS:
			{
				if (!bulk_owned_by(s, (size_t) s->a0 * (size_t) s->a1)) return;
				// a relation grows page by page (embedding.c:636-691): the mirror grows with it, doubling
				const size_t have = api.index_size(m->dev), cap = api.index_capacity(m->dev), need = have + (size_t) s->a0;
				if (need > cap)
				{
					const pgemb_status r = api.reserve(m->dev, need > 2 * cap ? need : 2 * cap);
					if (r != PGEMB_OK)
					{
						finish_api(s, r);
						return;
					}
				}
				finish_api(s, api.append_records(m->dev, (size_t) s->a0, bulk(), (size_t) s->a1));
				return;
			}
			case PGEMB_OP_BIND:
			{
				m->meta.efConstruction = (size_t) s->a1;  // re-read on every call, like the library does for a local caller
				const bool ok = api.bind_point(&m->meta, nullptr, (idx_t) s->a0);
				finish(s, ok ? PGEMB_OK : PGEMB_ERR_STATE, ok ? nullptr : api.last_error());
				return;
			}
			case PGEMB_OP_GET_LINKS:
				if (!bulk_owned_by(s, (size_t) s->a1 * (m->meta.maxM + 1) * sizeof(idx_t))) return;
				finish_api(s, api.get_links(m->dev, (size_t) s->a0, (size_t) s->a1, reinterpret_cast<idx_t *>(bulk())));
				return;
			case PGEMB_OP_EXPORT_RECORDS:
				if (!bulk_owned_by(s, (size_t) s->a1 * (size_t) s->a2)) return;
				finish_api(s, api.export_records(m->dev, (size_t) s->a0, (size_t) s->a1, bulk(), (size_t) s->a2));
				return;
			case PGEMB_OP_SET_LABELS:
				if (!bulk_owned_by(s, (size_t) s->a1 * sizeof(label_t))) return;
				finish_api(s, api.set_labels(m->dev, (size_t) s->a0, (size_t) s->a1, reinterpret_cast<const label_t *>(bulk())));
				return;
			case PGEMB_OP_TRUNCATE: finish_api(s, api.truncate(m->dev)); return;
			case PGEMB_OP_DROP:
			{
				auto it = mirrors.find(s->index_key);
				if (it != mirrors.end())
				{
					api.index_destroy(it->second.dev);
					mirrors.erase(it);
				}
				finish(s, PGEMB_OK, nullptr);
				return;
			}
			case PGEMB_OP_SIZE:
				s->a0 = api.index_size(m->dev);
				s->a1 = api.index_capacity(m->dev);
				finish(s, PGEMB_OK, nullptr);
				return;
			case PGEMB_OP_BUILD:
			{
				double		 sec = 0.0;
				pgemb_status r;
				if (s->a3)
					r = api.build_exact(m->dev, (size_t) s->a0, (size_t) s->a1, (size_t) s->a2, &sec, nullptr);
				else
					r = api.build_bulk(m->dev, (size_t) s->a0, (size_t) s->a1, (size_t) s->a2, &sec);
				memcpy(&s->a2, &sec, sizeof(sec));
				finish_api(s, r);
				return;
			}
			case PGEMB_OP_SHUTDOWN:
				g_stop = 1;
				finish(s, PGEMB_OK, nullptr);
				return;
			default: finish(s, PGEMB_ERR_ARG, "unknown request"); return;
		}
	}

	// ---- batched requests: all pending requests of one group -> one library call per max_batch --------------------
	// Searches launch pgemb_search_batch, scans pgemb_scan_topk_op and distances pgemb_dist_batch.  Scans are grouped by metric
	// (one pass over the table serves one operator) and by k, not folded into the largest k of the relation: a query's
	// re-scoring work grows with k (DESIGN.md section 6).  Every distance pair is independent and gets the bits of a one-pair
	// call: the same dist_pairs_kernel evaluates each pair alone.
	void run_group(const GroupKey &key, const std::vector<PgembIpcSlot *> &group)
	{
		const auto [op, g, k, mc] = key;  // g: relation key (search, scan) or metric (distance); k: ef, k or dim; mc: scan metric code
		PgembHostIndex *m = nullptr;
		const char	   *bad = nullptr;
		if (op == PGEMB_OP_DIST)
		{
			// the whole group shares the bad (metric, dim): each request fails by itself, the other groups are not affected
			if (k < 1 || k > hdr->max_dim || g > 2) bad = "dist: bad dimension or metric";
		}
		else if (auto it = mirrors.find(g); it == mirrors.end())
			bad = "no device index attached for this relation key";
		else if (op == PGEMB_OP_SEARCH && (k < 1 || k > hdr->max_ef))
			bad = "efSearch outside the sidecar's --max-ef";
		else if (op == PGEMB_OP_SCAN && (k < 1 || k > std::min<size_t>(4096, hdr->max_ef)))
			bad = "scan: k outside 1 .. min(4096, the sidecar's --max-ef)";
		else if (op == PGEMB_OP_SCAN && mc > 3)
			bad = "scan: unknown distance function";
		else
			m = &it->second;
		if (bad)
		{
			for (PgembIpcSlot *s : group) finish(s, PGEMB_ERR_ARG, bad);
			return;
		}
		const size_t dim = m ? m->meta.dim : k;
		for (size_t lo = 0; lo < group.size(); lo += max_batch)
		{
			const size_t nq = std::min(max_batch, group.size() - lo);
			auto		 count = [nq](uint64_t &calls, uint64_t &served, uint64_t &largest) {
				calls += 1;
				served += nq;
				if (nq > largest) largest = nq;
			};
			qbuf.resize(nq * dim);
			for (size_t i = 0; i < nq; i++) memcpy(&qbuf[i * dim], slot_vec(group[lo + i]), dim * sizeof(float));
			pgemb_status r;
			if (op == PGEMB_OP_SEARCH)
			{
				lbuf.resize(nq * k);
				nbuf.assign(nq, 0);
				r = api.search_batch(m->dev, nq, qbuf.data(), k, lbuf.data(), nullptr, nullptr, nbuf.data(), nullptr);
				if (!carry_counted)
				{
					// who queued up while the launch ran (BEFORE any result of this round is published: a caller that gets its
					// result resubmits at once and would be counted twice)
					carry_counted = true;
					for (uint32_t i = 0; i < hdr->n_slots; i++)
					{
						const PgembIpcSlot *c = slot(i);
						if (ld(&c->state) == PGEMB_SLOT_READY && c->op == PGEMB_OP_SEARCH) carry++;
					}
				}
				count(hdr->n_batches, hdr->n_searches, hdr->max_batch);
			}
			else if (op == PGEMB_OP_SCAN)
			{
				lbuf.resize(nq * k);
				dbuf.resize(nq * k);
				nbuf.assign(nq, 0);
				const dist_func_t metric = mc ? (dist_func_t) (mc - 1) : m->meta.dist_func;
				r = api.scan_topk_op(m->dev, metric, nq, qbuf.data(), k, lbuf.data(), dbuf.data(), nbuf.data());
				count(hdr->n_scan_calls, hdr->n_scans, hdr->max_scan_batch);
			}
			else
			{
				bbuf.resize(nq * dim);
				dbuf.resize(nq);
				for (size_t i = 0; i < nq; i++) memcpy(&bbuf[i * dim], slot_vec(group[lo + i]) + hdr->max_dim, dim * sizeof(float));
				r = api.dist_batch((dist_func_t) g, dim, nq, qbuf.data(), 0, bbuf.data(), dbuf.data());
				count(hdr->n_dist_calls, hdr->n_dists, hdr->max_dist_batch);
			}
			for (size_t i = 0; i < nq; i++)
			{
				PgembIpcSlot *s = group[lo + i];
				if (r == PGEMB_OK && op == PGEMB_OP_DIST)
				{
					uint32_t bits;
					memcpy(&bits, &dbuf[i], 4);
					s->a2 = bits;
				}
				else if (r == PGEMB_OK)
				{
					const size_t n = (size_t) (nbuf[i] > 0 ? nbuf[i] : 0);
					s->n_out = nbuf[i];
					memcpy(slot_labels(s), &lbuf[i * k], n * sizeof(label_t));
					if (op == PGEMB_OP_SCAN) memcpy(slot_dists(s), &dbuf[i * k], n * sizeof(float));
				}
				finish_api(s, r);
			}
		}
	}

	// one pass over the slots; returns the number of requests served
	size_t serve_once()
	{
		std::vector<PgembIpcSlot *> control;
		std::map<GroupKey, std::vector<PgembIpcSlot *>> batched;
		size_t found = 0, nsearch = 0;
		auto   collect = [&]() {
			for (uint32_t i = 0; i < hdr->n_slots; i++)
			{
				PgembIpcSlot *s = slot(i);
				if (ld(&s->state) != PGEMB_SLOT_READY) continue;
				st(&s->state, PGEMB_SLOT_BUSY);
				found++;
				if (s->op == PGEMB_OP_SEARCH)
				{
					batched[{s->op, s->index_key, s->ef, 0}].push_back(s);
					nsearch++;
				}
				else if (s->op == PGEMB_OP_SCAN)
				{
					// not part of the searches' linger bookkeeping (nsearch / target / carry).  A scan that asks for the mirror's
					// metric joins the group of the scans that name that metric.
					uint64_t mc = s->a1;
					if (auto it = mirrors.find(s->index_key); mc == 0 && it != mirrors.end()) mc = 1 + (uint64_t) it->second.meta.dist_func;
					batched[{s->op, s->index_key, s->a0, mc}].push_back(s);
				}
				else if (s->op == PGEMB_OP_DIST)
					batched[{s->op, s->a1, s->a0, 0}].push_back(s);	 // touches no mirror, so no place in the write/search order; never lingers
				else
					control.push_back(s);
			}
		};
		// serve every collected group of one kind, in key order
		auto run_groups = [&](uint32_t op) {
			const auto first = batched.lower_bound(GroupKey{op, 0, 0, 0}), last = batched.lower_bound(GroupKey{op + 1, 0, 0, 0});
			for (auto it = first; it != last; ++it) run_group(it->first, it->second);
			batched.erase(first, last);
		};
		collect();
		if (found == 0) return 0;
		// Distances first, as soon as they are collected: a one-pair request must not wait behind the searches' launches or
		// their linger below.  Whatever queued up while the previous pass ran is served by one call per (metric, dim).
		run_groups(PGEMB_OP_DIST);
		// Keeping the callers together.  A caller resubmits a few microseconds after it got its result, so a server that
		// launches whatever is queued the moment it becomes free splits P steady callers into two groups that are served
		// alternately -- each waits two launches per result.  `target` is the number of concurrent searchers the last
		// round showed (its batch + those that were already queued when it finished, see below); when fewer are here
		// now, the rest are about to arrive: wait for them, at most linger_us.  One caller never waits (target = 1).
		if (linger_us > 0 && nsearch > 0 && nsearch < target)
		{
			// a caller needs its wake-up latency (it sleeps on a futex while a launch runs) plus a few microseconds to be
			// back: wait linger_us, or a quarter of the previous round if that is longer (never more than 2 ms)
			double wait = 1e-6 * (double) linger_us;
			if (0.25 * last_service_s > wait) wait = 0.25 * last_service_s;
			if (wait > 2e-3) wait = 2e-3;
			const double until = now_s() + wait;
			while (nsearch < target && now_s() < until)
			{
				collect();
				run_groups(PGEMB_OP_DIST);
			}
		}
		for (PgembIpcSlot *s : control) run_control(s);
		const double t_run = now_s();
		carry = 0;
		carry_counted = false;
		run_groups(PGEMB_OP_SEARCH);
		if (nsearch > 0)
		{
			last_service_s = now_s() - t_run;
			if (const char *dbg = getenv("PGEMB_SIDECAR_DEBUG"))
			{
				FILE *f = fopen(dbg, "a");
				if (f) { fprintf(f, "round: nsearch %zu target %zu service %.0f us\n", nsearch, target, last_service_s * 1e6); fclose(f); }
			}
			// carry: callers of the "other group" (counted in run_group, before this round's results went out)
			const size_t seen = nsearch + carry, decayed = target - (target + 9) / 10;	// forget departed callers by 10 % a round
			target = seen > decayed ? seen : decayed;
			if (target < 1) target = 1;
			if (target > hdr->n_slots) target = hdr->n_slots;
		}
		// Scans last: a scan sees every write whose request completed before it was submitted, as a search does.  They
		// never linger: a scan call takes milliseconds, and the next batch queues up by itself while it runs.  A scan and a
		// search of the same mirror never run at the same time (the index's staging buffers and workspace are shared).
		run_groups(PGEMB_OP_SCAN);
		return found;
	}

	// slots / bulk lock left behind by clients that died.  A slot is taken back only if the SAME dead owner was seen on two
	// consecutive passes (a second apart) in the SAME state, and then by a CAS on that state: a claimer that is between its CAS
	// and the store of its pid (owner_pid 0, or -- after a cancelled request -- the previous user's) is never mistaken for a
	// dead one.
	std::vector<int32_t>  suspect_pid;
	std::vector<uint32_t> suspect_state;
	void reclaim()
	{
		if (suspect_pid.size() != hdr->n_slots)
		{
			suspect_pid.assign(hdr->n_slots, 0);
			suspect_state.assign(hdr->n_slots, 0);
		}
		for (uint32_t i = 0; i < hdr->n_slots; i++)
		{
			PgembIpcSlot  *s = slot(i);
			const uint32_t stt = ld(&s->state);
			const int32_t  owner = __atomic_load_n(&s->owner_pid, __ATOMIC_ACQUIRE);
			const bool	   dead = (stt == PGEMB_SLOT_CLAIMED || stt == PGEMB_SLOT_DONE) && owner > 0 && kill(owner, 0) != 0 && errno == ESRCH;
			if (!dead)
			{
				suspect_pid[i] = 0;
				continue;
			}
			if (suspect_pid[i] == owner && suspect_state[i] == stt)
			{
				uint32_t expect = stt;
				if (__atomic_load_n(&s->owner_pid, __ATOMIC_ACQUIRE) == owner)
				{
					__atomic_store_n(&s->owner_pid, 0, __ATOMIC_RELEASE);
					if (!__atomic_compare_exchange_n(&s->state, &expect, (uint32_t) PGEMB_SLOT_FREE, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED))
					{
						int32_t zero = 0;  // the state moved on under us (cannot happen with a dead owner): put the pid back unless somebody else's is there
						__atomic_compare_exchange_n(&s->owner_pid, &zero, owner, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED);
					}
				}
				suspect_pid[i] = 0;
			}
			else
			{
				suspect_pid[i] = owner;
				suspect_state[i] = stt;
			}
		}
		uint32_t owner = ld(&hdr->bulk_lock);
		if (owner != 0 && kill((pid_t) owner, 0) != 0 && errno == ESRCH)
			__atomic_compare_exchange_n(&hdr->bulk_lock, &owner, 0u, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED);
	}

	void loop()
	{
		double last_reclaim = now_s();
		double idle_since = now_s();
		while (!g_stop)
		{
			const size_t served = serve_once();
			const double t = now_s();
			if (t - last_reclaim > 1.0)
			{
				reclaim();	// also under constant load: a dead client must not keep the bulk area or a slot for ever
				last_reclaim = t;
			}
			if (served > 0)
			{
				idle_since = t;
				continue;
			}
			if (t - idle_since < 200e-6) continue;	// stay hot for a moment: the next query of a scan follows at once
			// sleep until a client bumps submit_seq (it wakes us only when it sees server_sleeping)
			const uint32_t seq = ld(&hdr->submit_seq);
			st(&hdr->server_sleeping, 1);
			__atomic_thread_fence(__ATOMIC_SEQ_CST);
			if (serve_once() == 0 && !g_stop)
			{
				struct timespec ts = {0, 100 * 1000 * 1000};
				futex(&hdr->submit_seq, FUTEX_WAIT, seq, &ts);
			}
			st(&hdr->server_sleeping, 0);
			idle_since = now_s();
		}
	}
};

void usage()
{
	fprintf(stderr,
			"usage: pgemb_sidecar --shm /NAME [--lib PATH] [--device K] [--slots N] [--max-dim D] [--max-ef E] [--bulk-mb M]\n"
			"                     [--max-batch B] [--linger-us U (max adaptive wait for resubmitting callers, default 50, 0 = off)]\n");
}

}  // namespace

int main(int argc, char **argv)
{
	std::string shm_name, lib_path;
	uint32_t	n_slots = 256, max_dim = 2000, max_ef = 16384;	// max_ef sizes the label area of a slot (8 B each): hnsw_gettuple doubles efSearch
																// (embedding.c:334) -- LIMITs beyond max_ef / 2 rows fail with "HNSW index search failed"
	size_t		bulk_mb = 64;
	Server		srv;
	for (int i = 1; i < argc; i++)
	{
		const std::string a = argv[i];
		auto			  val = [&]() -> const char			   *{
			 if (i + 1 >= argc)
			 {
				 usage();
				 exit(2);
			 }
			 return argv[++i];
		};
		if (a == "--shm") shm_name = val();
		else if (a == "--lib") lib_path = val();
		else if (a == "--device") srv.device = atoi(val());
		else if (a == "--slots") n_slots = (uint32_t) atoi(val());
		else if (a == "--max-dim") max_dim = (uint32_t) atoi(val());
		else if (a == "--max-ef") max_ef = (uint32_t) atoi(val());
		else if (a == "--bulk-mb") bulk_mb = (size_t) atol(val());
		else if (a == "--max-batch") srv.max_batch = (size_t) atol(val());
		else if (a == "--linger-us") srv.linger_us = atol(val());
		else
		{
			usage();
			return 2;
		}
	}
	if (shm_name.empty() || shm_name[0] != '/' || n_slots < 1 || max_dim < 1 || max_ef < 1 || srv.max_batch < 1)
	{
		usage();
		return 2;
	}
	if (lib_path.empty())
	{
		char	self[4096];
		ssize_t n = readlink("/proc/self/exe", self, sizeof(self) - 1);
		if (n <= 0) return 2;
		self[n] = 0;
		std::string dir(self);
		dir = dir.substr(0, dir.find_last_of('/'));
		lib_path = dir + "/libpgemb_b200.so";
	}
	if (!load_api(lib_path.c_str(), srv.api)) return 3;
	if (srv.api.device_count() < 1)
	{
		fprintf(stderr, "pgemb_sidecar: no CUDA device (%s): the hot path has no CPU fallback\n", srv.api.last_error());
		return 4;
	}
	srv.api.init_dist_func();

	const size_t stride = pgemb_ipc_slot_stride(max_dim, max_ef);
	const size_t slots_off = (sizeof(PgembIpcHeader) + 63u) & ~(size_t) 63u;
	const size_t bulk_off = (slots_off + stride * n_slots + 4095u) & ~(size_t) 4095u;
	const size_t bytes = bulk_off + (bulk_mb << 20);
	shm_unlink(shm_name.c_str());  // a stale segment of a dead sidecar
	const int fd = shm_open(shm_name.c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
	// posix_fallocate: a /dev/shm that is too small fails here, not with SIGBUS when a client touches the bulk area
	int fe = 0;
	if (fd < 0 || ftruncate(fd, (off_t) bytes) != 0 || (fe = posix_fallocate(fd, 0, (off_t) bytes)) != 0)
	{
		if (fe) errno = fe;
		perror("pgemb_sidecar: shm_open/ftruncate/posix_fallocate");
		if (fd >= 0) shm_unlink(shm_name.c_str());
		return 5;
	}
	void *mem = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
	close(fd);
	if (mem == MAP_FAILED)
	{
		perror("pgemb_sidecar: mmap");
		shm_unlink(shm_name.c_str());
		return 5;
	}
	memset(mem, 0, bulk_off);
	srv.base = static_cast<unsigned char *>(mem);
	srv.bytes = bytes;
	srv.hdr = static_cast<PgembIpcHeader *>(mem);
	PgembIpcHeader *h = srv.hdr;
	h->version = PGEMB_IPC_VERSION;
	h->n_slots = n_slots;
	h->max_dim = max_dim;
	h->max_ef = max_ef;
	h->slot_stride = (uint32_t) stride;
	h->slots_off = slots_off;
	h->bulk_off = bulk_off;
	h->bulk_bytes = bulk_mb << 20;
	h->server_pid = (int32_t) getpid();
	h->magic = PGEMB_IPC_MAGIC;

	struct sigaction sa;
	memset(&sa, 0, sizeof(sa));
	sa.sa_handler = on_signal;
	sigaction(SIGTERM, &sa, nullptr);
	sigaction(SIGINT, &sa, nullptr);

	st(&h->ready, 1);
	fprintf(stderr, "pgemb_sidecar: serving %s (%s, device %d, %u slots, bulk %zu MB)\n", shm_name.c_str(), srv.api.version(), srv.device, n_slots, bulk_mb);
	srv.loop();
	st(&h->ready, 0);
	// fail whatever is still queued, then let go of the device memory
	for (uint32_t i = 0; i < n_slots; i++)
	{
		PgembIpcSlot  *s = srv.slot(i);
		const uint32_t stt = ld(&s->state);
		if (stt == PGEMB_SLOT_READY || stt == PGEMB_SLOT_BUSY) srv.finish(s, PGEMB_ERR_STATE, "sidecar is shutting down");
	}
	for (auto &kv : srv.mirrors) srv.api.index_destroy(kv.second.dev);
	shm_unlink(shm_name.c_str());
	munmap(mem, bytes);
	fprintf(stderr, "pgemb_sidecar: stopped\n");
	return 0;
}
