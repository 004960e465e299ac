// pgemb::search_kernel (throughput and latency mode) on the host SIMT emulator (tests/emu).
// The harness plays the part of capi.cu's plan_search and launch_search: same make_search_config, same pick_search_kernel,
// same parameter block.
#include <cuda_runtime.h>  // the stand-in in tests/emu/fake_cuda

#include "../../pg_embedding_b200/csrc/bind_kernel.cuh"
#include "../../pg_embedding_b200/csrc/search_kernel.cuh"

using namespace pgemb;

extern "C" int emu_search_ex(int metric, int coop, const float *vectors, const uint32_t *links, const uint64_t *labels, const float *norms,
							 uint32_t n_items, uint32_t dim, uint32_t row_f, uint32_t link_stride, uint32_t maxM, const float *queries,
							 uint32_t nq, uint32_t ef, int raw_mode, uint64_t *labels_out, float *dists_out, uint32_t *ids_out,
							 int32_t *n_out, uint32_t *stats_out, uint32_t want_warps, uint32_t want_rings, uint32_t grid, uint32_t vh_size,
							 uint32_t visited_pairs, uint32_t smem_visited, int *error_out);

// returns 0 on success, >0 = make_search_config's code, -1 = bad metric; *error_out = the kernel's sticky error flag
extern "C" int emu_search(int metric, int coop, const float *vectors, const uint32_t *links, const uint64_t *labels, const float *norms,
						  uint32_t n_items, uint32_t dim, uint32_t row_f, uint32_t link_stride, uint32_t maxM, const float *queries,
						  uint32_t nq, uint32_t ef, int raw_mode, uint64_t *labels_out, float *dists_out, uint32_t *ids_out,
						  int32_t *n_out, uint32_t *stats_out, uint32_t want_warps, uint32_t want_rings, uint32_t grid, uint32_t vh_size,
						  uint32_t visited_pairs, int *error_out)
{
	return emu_search_ex(metric, coop, vectors, links, labels, norms, n_items, dim, row_f, link_stride, maxM, queries, nq, ef, raw_mode, labels_out,
						 dists_out, ids_out, n_out, stats_out, want_warps, want_rings, grid, vh_size, visited_pairs, 0, error_out);
}

extern "C" int emu_search_ex(int metric, int coop, const float *vectors, const uint32_t *links, const uint64_t *labels, const float *norms,
							 uint32_t n_items, uint32_t dim, uint32_t row_f, uint32_t link_stride, uint32_t maxM, const float *queries,
							 uint32_t nq, uint32_t ef, int raw_mode, uint64_t *labels_out, float *dists_out, uint32_t *ids_out,
							 int32_t *n_out, uint32_t *stats_out, uint32_t want_warps, uint32_t want_rings, uint32_t grid, uint32_t vh_size,
							 uint32_t visited_pairs, uint32_t smem_visited, int *error_out)
{
	SearchShape sh;
	sh.metric = metric;
	sh.dim = dim;
	sh.row_f = row_f;
	sh.link_stride = link_stride;
	sh.maxM = maxM;
	sh.ef = ef;
	sh.sm_count = grid;
	SearchTuning tu;
	tu.want_warps = (int) want_warps;
	tu.want_rings = (int) want_rings;
	tu.want_coop_warps = (int) want_warps;
	sh.tpr = (smem_visited & 0x80000000u) ? 8u : 4u;		  // bit 31: 8 lanes per L2 row
	const bool res_global = (smem_visited & 0x20000000u) != 0u;  // bit 29: result buffers in global memory (the huge-ef variant)
	sh.res_global = res_global;
	smem_visited &= 0x1fffffffu;
	tu.smem_visited = (int) smem_visited;
	SearchConfig cfg;
	const int rc = make_search_config(sh, tu, coop != 0, &cfg);
	if (rc) return rc;
	if (coop && smem_visited && cfg.vhs_entries == 0) return 77;  // the test asked for the shared-memory set
	const uint32_t slots = coop ? grid : grid * cfg.warps;
	const uint32_t vis_words = (n_items + 31) / 32 + 1;
	const uint32_t vlog_cap = n_items < 32768 ? n_items + 1 : 32768;
	std::vector<uint32_t> visited((size_t) slots * vis_words, 0u), vlog((size_t) slots * vlog_cap, 0u);
	std::vector<uint32_t> vhash((size_t) slots * (vh_size ? vh_size : 1), 0xffffffffu);
	std::vector<uint64_t> ovf((size_t) slots * ef, 0ull);
	std::vector<uint64_t> resg(res_global ? (size_t) slots * 2 * ef : 1, 0ull);
	unsigned int counter = 0;
	int			 err = 0;

	SearchParams p;
	memset(&p, 0, sizeof(p));
	p.vectors = vectors;
	p.links = links;
	p.labels = labels;
	p.norms = norms;
	p.n_items = n_items;
	p.dim = dim;
	p.row_f = row_f;
	p.link_stride = link_stride;
	p.maxM = maxM;
	p.entry = 0;
	p.queries = queries;
	p.nq = nq;
	p.q_stride = dim;
	p.ef = ef;
	p.raw_mode = raw_mode ? 1u : 0u;
	p.labels_out = labels_out;
	p.dists_out = dists_out;
	p.ids_out = ids_out;
	p.n_out = n_out;
	p.stats_out = stats_out;
	p.visited = visited.data();
	p.vlog = vlog.data();
	p.ovf = ovf.data();
	p.res_g = res_global ? resg.data() : nullptr;
	p.vhash = vhash.data();
	p.vis_words = vis_words;
	p.vlog_cap = vlog_cap;
	p.vh_size = vh_size;
	{
		uint32_t lg = 0;
		while ((1u << lg) < vh_size) lg++;
		p.vh_shift = 32u - lg;
	}
	p.counter = &counter;
	p.error_flag = &err;
	p.prefetch_links = 1;
	p.visited_pairs = visited_pairs;  // used by the latency-mode kernel only
	apply_config(p, cfg, row_f);
	unsigned g = nq < grid ? nq : grid;
	if (g == 0) g = 1;
	if (res_global && (coop || cfg.tpr != 4)) return 79;
	const search_fn_t fn = pick_search_kernel(metric, coop != 0, cfg.tpr, res_global);
	if (!fn) return -1;
	PGEMB_LAUNCH(fn, g, cfg.warps * 32, cfg.smem, 0, p);
	// the visited sets must be left clean for the next launch
	for (uint32_t v : visited)
		if (v != 0u) err |= 0x100;
	for (uint32_t v : vhash)
		if (v != 0xffffffffu) err |= 0x200;
	if (error_out) *error_out = err;
	return 0;
}

// ---- sequential inserts: n x hnsw_bind_point as capi.cu's bind_points() issues them -------------------------------
// per insert: traversal in raw mode (query = the stored node, ef = efConstruction), select_kernel, backlink_kernel.
template <int METRIC> static void connect_one(GraphView g, const uint32_t *new_id, const uint32_t *cand_ids, const float *cand_d,
											  const int32_t *cand_n, uint32_t efc, uint64_t *pairs)
{
	const size_t M = g.M ? g.M : 1, maxM1 = g.maxM + 1;
	const size_t sel_smem = efc * 8 + M * 8 + efc * 4;
	const size_t bl_smem = maxM1 * 8 * 2 + (g.maxM ? g.maxM : 1) * 8 + maxM1 * 4;
	emu::launch(dim3(1), kBindThreads, sel_smem, [=]() { select_kernel<METRIC>(g, new_id, cand_ids, cand_d, cand_n, efc, pairs); });
	const uint32_t n_pairs = (uint32_t) M;
	emu::launch(dim3(n_pairs), kBindThreads, bl_smem, [=]() { backlink_kernel<METRIC>(g, pairs, n_pairs); });
}

extern "C" int emu_bind_sequence(int metric, int coop, const float *vectors, uint32_t *links, const float *norms, uint32_t n_items,
								 uint32_t dim, uint32_t row_f, uint32_t link_stride, uint32_t M, uint32_t maxM, uint32_t efc, uint32_t first,
								 uint32_t count, int *error_out)
{
	SearchShape sh;
	sh.metric = metric;
	sh.dim = dim;
	sh.row_f = row_f;
	sh.link_stride = link_stride;
	sh.maxM = maxM;
	sh.ef = efc;
	sh.sm_count = 1;
	SearchTuning tu;
	tu.want_warps = 2;
	tu.want_rings = 2;
	tu.want_coop_warps = 3;
	SearchConfig cfg;
	const int rc = make_search_config(sh, tu, coop != 0, &cfg);
	if (rc) return rc;
	const uint32_t slots = cfg.warps, vh_size = 64, vis_words = (n_items + 31) / 32 + 1, vlog_cap = n_items + 1;
	std::vector<uint32_t> visited((size_t) slots * vis_words, 0u), vlog((size_t) slots * vlog_cap, 0u), vhash((size_t) slots * vh_size, 0xffffffffu);
	std::vector<uint64_t> ovf((size_t) slots * efc, 0ull), pairs(M ? M : 1, ~0ull), labels(n_items, 0ull);
	std::vector<uint32_t> cand_ids(efc, 0u);
	std::vector<float>	  cand_d(efc, 0.f);
	int32_t				  cand_n = 0;
	unsigned int		  counter = 0;
	int					  err = 0;
	GraphView g;
	g.vectors = vectors;
	g.norms = norms;
	g.links = links;
	g.row_f = row_f;
	g.link_stride = link_stride;
	g.dim = dim;
	g.M = M;
	g.maxM = maxM;
	g.error_flag = &err;
	for (uint32_t i = 0; i < count; i++)
	{
		const uint32_t id = first + i;
		if (id == 0) continue;	// hnswalg.cpp:227-228
		SearchParams p;
		memset(&p, 0, sizeof(p));
		p.vectors = vectors;
		p.links = links;
		p.labels = labels.data();
		p.norms = norms;
		p.n_items = n_items;
		p.dim = dim;
		p.row_f = row_f;
		p.link_stride = link_stride;
		p.maxM = maxM;
		p.entry = 0;
		p.query_ids = &id;
		p.nq = 1;
		p.ef = efc;
		p.raw_mode = 1;
		p.dists_out = cand_d.data();
		p.ids_out = cand_ids.data();
		p.n_out = &cand_n;
		p.visited = visited.data();
		p.vlog = vlog.data();
		p.ovf = ovf.data();
	p.res_g = nullptr;
		p.vhash = vhash.data();
		p.vis_words = vis_words;
		p.vlog_cap = vlog_cap;
		p.vh_size = vh_size;
		p.vh_shift = 32u - 6u;
		counter = 0;
		p.counter = &counter;
		p.error_flag = &err;
		p.prefetch_links = 1;
		apply_config(p, cfg, row_f);
		const search_fn_t fn = pick_search_kernel(metric, coop != 0, cfg.tpr, false);
		if (!fn) return -1;
		PGEMB_LAUNCH(fn, 1, cfg.warps * 32, cfg.smem, 0, p);
		if (metric == 0) connect_one<M_L2>(g, &id, cand_ids.data(), cand_d.data(), &cand_n, efc, pairs.data());
		else if (metric == 1) connect_one<M_COS>(g, &id, cand_ids.data(), cand_d.data(), &cand_n, efc, pairs.data());
		else connect_one<M_MAN>(g, &id, cand_ids.data(), cand_d.data(), &cand_n, efc, pairs.data());
		if (err) break;
	}
	if (error_out) *error_out = err;
	return 0;
}
