// Dumps make_search_config's result for a grid of shapes as CSV (tests/test_search_config.py checks the invariants the
// kernel relies on: total size, alignment of every region a bulk copy or a vector load touches, ring / slot counts).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include "../../pg_embedding_b200/csrc/search_config.h"
using namespace pgemb;
int main()
{
	printf("metric,dim,maxM,ef,coop,tpr,rc,warps,rings,ring_bytes,priv_bytes,row_smem,qt_stride,smem,slots,off_pool,off_ring,off_priv,off_qt,off_qtail,off_res,off_hopkey,off_acckey,off_evict,off_hopid,off_pf,off_pfbar,pool_size\n");
	for (int metric = 0; metric < 3; metric++)
		for (uint32_t dim : {1u, 2u, 3u, 4u, 5u, 15u, 16u, 17u, 31u, 33u, 63u, 64u, 100u, 127u, 128u, 129u, 300u, 767u, 768u, 769u, 1024u, 1536u, 1999u, 2000u})
			for (uint32_t maxM : {0u, 2u, 6u, 32u, 64u, 200u, 254u, 256u, 258u, 1024u, 1800u, 2036u, 4096u})
				for (uint32_t ef : {1u, 5u, 64u, 200u, 1000u, 4000u})
					for (int coop = 0; coop < 2; coop++)
						for (uint32_t tpr : {4u, 8u})
						{
							if (tpr == 8 && metric != 0) continue;
							SearchShape sh;
							sh.metric = metric;
							sh.dim = dim;
							sh.row_f = (dim + 3) & ~3u;
							sh.link_stride = (maxM + 1 + 3) & ~3u;
							sh.maxM = maxM;
							sh.ef = ef;
							sh.sm_count = 132;  // H100 SXM
							sh.tpr = tpr;
							SearchTuning tu;
							SearchConfig c;
							const int rc = make_search_config(sh, tu, coop != 0, &c);
							printf("%d,%u,%u,%u,%d,%u,%d,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%u,%zu\n", metric, dim, maxM, ef, coop, tpr, rc, c.warps,
								   c.rings, c.ring_bytes, c.priv_bytes, c.row_smem, c.qt_stride, c.smem, c.slots, c.off_pool, c.off_ring, c.off_priv, c.off_qt,
								   c.off_qtail, c.off_res, c.off_hopkey, c.off_acckey, c.off_evict, c.off_hopid, c.off_pf, c.off_pfbar, sizeof(RingPool));
						}
	return 0;
}
