// search_config.h -- shared-memory layout and slot/ring counts of the traversal kernel (DESIGN.md section 6).
// Plain host C++ (no CUDA): used by capi.cu to launch search_kernel and by the host emulation harness in
// tests/emu, so both see the very same layout.
#pragma once
#include <stdint.h>

namespace pgemb {

struct RingPool
{
	// One atomic word is the whole lock state: bit b (b < 16) set = ring b is free; bit 16+b = the phase parity the
	// next wait on ring b's mbarrier must observe.  A slot learns the parity from the very value its acquiring
	// atomicCAS observed and hands the updated parity back with atomics before it sets the free bit again, so no
	// plain shared-memory word is ever shared between slots.
	uint32_t state;
	uint32_t pad;
	uint64_t bar[15];		// one mbarrier per ring
	// latency mode (COOP): the owner warp publishes the hop's row count (kNone = quit) and |q|^2 here
	uint32_t coop_n;
	float	 coop_qn;
};
constexpr uint32_t kMaxRings = 15;
constexpr uint32_t kMaxCtaSmem = 232448u;  // dynamic shared memory a CTA may opt in to on the H100 (227 KB)

struct SearchConfig
{
	uint32_t warps = 0, rings = 0, ring_bytes = 0, priv_bytes = 0, row_smem = 0, qt_stride = 0, smem = 0, slots = 0;
	uint32_t off_pool = 0, off_ring = 0, off_priv = 0;
	uint32_t off_qt = 0, off_qtail = 0, off_res = 0, off_hopkey = 0, off_acckey = 0, off_evict = 0, off_hopid = 0, off_pf = 0, off_pfbar = 0;
	uint32_t ef = 0;
	uint32_t tpr = 4;
	uint32_t off_vhs = 0, vhs_entries = 0;	// latency mode: visited hash set in shared memory
	bool	 res_global = false;
};

struct SearchShape
{
	int		 metric = 0;  // DIST_L2 = 0, DIST_COSINE = 1, DIST_MANHATTAN = 2
	uint32_t dim = 0, row_f = 0, link_stride = 0, maxM = 0, ef = 0, sm_count = 0;
	uint32_t tpr = 4;  // lanes per row: 4, or 8 (L2 only: a ring then holds 4 rows)
	// the two result buffers (2 x ef keys) live in global memory instead of the slot's private shared-memory block: for ef so
	// large that they no longer fit (the reference doubles efSearch without bound, embedding.c:334)
	bool res_global = false;
};

struct SearchTuning
{
	double duty = 0.5;		   // fraction of a hop a slot holds a ring for
	int	   want_warps = 0;	   // overrides (0 = choose)
	int	   want_rings = 0;
	int	   want_coop_warps = 0;
	int	   smem_visited = 0;	  // latency mode: entries (power of two) of the shared-memory visited set to try for, 0 = off
};

inline uint32_t cfg_align_up(uint32_t x, uint32_t a) { return (x + a - 1) / a * a; }

// returns 0 = ok, 1 = the working set does not fit shared memory, 2 = the overrides do not fit
inline int make_search_config(const SearchShape &sh, const SearchTuning &tu, bool coop, SearchConfig *c)
{
	const int	   metric = sh.metric;
	const uint32_t row_bytes = sh.row_f * 4u;
	// bank-conflict-free pitch of a row in shared memory for the 4-lanes-per-row mapping:
	// == 16 (mod 128) for the LDS.32 of cosine/manhattan, == 32 (mod 128) for the LDS.64 of L2
	const uint32_t resid = (metric == 0) ? 32u : 16u;
	uint32_t	   row_smem = row_bytes / 128u * 128u + resid;
	if (row_smem < row_bytes) row_smem += 128u;
	const uint32_t maxM = sh.maxM;
	const uint32_t hopcap = maxM > 1 ? maxM : 1;
	const uint32_t max_cta = kMaxCtaSmem;
	const uint32_t ef = sh.ef;
	if (!sh.res_global && ef > (max_cta / 16u)) return 1;  // 2 x ef x 8 bytes alone exceed a CTA's shared memory
	// lane-major transposed query: per lane-thread a run of floats padded so that the four runs start
	// 16 bytes apart modulo 128 (conflict-free LDS.128)
	const uint32_t dim = sh.dim;
	const uint32_t tpr = (metric == 0 && sh.tpr == 8) ? 8u : 4u;
	const uint32_t rows_per_ring = 32u / tpr;
	// floats per lane run: 4 lanes x dim/4 (two L2 chains interleaved per lane), or 8 lanes x dim/8
	const uint32_t run = (metric == 0) ? ((dim & ~15u) >> (tpr == 8 ? 3 : 2)) : ((dim & ~3u) >> 2);
	// runs start 16 bytes apart modulo 128: the LDS.128 of the 4 (or 8) distinct runs a warp reads hit distinct banks, and
	// every run is 16-byte aligned
	const uint32_t qt_stride = cfg_align_up(run ? run : 1, 32) + 4u;

	SearchConfig t;
	t.tpr = tpr;
	t.res_global = sh.res_global;
	// ---- a slot's private block ----
	uint32_t off = 0;
	t.off_qt = off;			off = cfg_align_up(off + tpr * qt_stride * 4u, 16);
	t.off_qtail = off;		off = cfg_align_up(off + 16u * 4u, 16);
	t.off_res = off;		off += sh.res_global ? 0u : 2u * ef * 8u;
	t.off_hopkey = off;		off += hopcap * 8u;
	t.off_acckey = off;		off += hopcap * 8u;
	t.off_evict = off;		off += hopcap * 8u;
	t.off_hopid = off;		off = cfg_align_up(off + hopcap * 4u, 16);
	t.off_pf = off;			off = cfg_align_up(off + sh.link_stride * 4u, 8);
	t.off_pfbar = off;		off += 8u;
	t.priv_bytes = cfg_align_up(off, 128);
	t.ring_bytes = cfg_align_up(rows_per_ring * row_smem, 128);
	const uint32_t pool_bytes = cfg_align_up((uint32_t) sizeof(RingPool), 128);
	// ---- how many slots (warps) and rings per CTA (= per SM) ----
	// A slot holds a ring for about `duty` of a hop; throughput ~ min(W / T_hop, R / (duty * T_hop)).
	const double duty = tu.duty;
	uint32_t	 bestW = 0, bestR = 0;
	double		 bestv = -1.0;
	for (uint32_t W = 1; W <= 32; W++)
	{
		if (pool_bytes + W * t.priv_bytes + t.ring_bytes > max_cta) break;
		uint32_t R = (max_cta - pool_bytes - W * t.priv_bytes) / t.ring_bytes;
		if (R > W) R = W;
		if (R > kMaxRings) R = kMaxRings;
		const double v = (W < R / duty) ? (double) W : R / duty;
		if (v > bestv + 1e-9)
		{
			bestv = v;
			bestW = W;
			bestR = R;
		}
	}
	if (bestW == 0) return 1;
	if (coop)
	{
		// latency mode: one slot per CTA, every warp owns a ring; no more warps than a full hop has row groups
		uint32_t	   R = (max_cta - pool_bytes - t.priv_bytes) / t.ring_bytes;
		const uint32_t groups = (hopcap + rows_per_ring - 1u) / rows_per_ring;
		if (R > groups) R = groups;
		if (R > kMaxRings) R = kMaxRings;
		const int wantC = tu.want_coop_warps;
		if (wantC > 0 && (uint32_t) wantC < R) R = (uint32_t) wantC;
		if (R < 1) R = 1;
		t.warps = R;
		t.rings = R;
		t.off_pool = 0;
		t.off_ring = pool_bytes;
		t.off_priv = pool_bytes + R * t.ring_bytes;
		t.smem = t.off_priv + t.priv_bytes;
		if (tu.smem_visited > 0)
		{
			// whatever is left of the CTA's 227 KB, as a power-of-two table of u32 (never below 1024 entries)
			uint32_t e = 1024;
			while (e * 2u <= (uint32_t) tu.smem_visited && t.smem + e * 2u * 4u <= max_cta) e *= 2u;
			if (t.smem + e * 4u <= max_cta)
			{
				t.off_vhs = t.smem;
				t.vhs_entries = e;
				t.smem += e * 4u;
			}
		}
		t.row_smem = row_smem;
		t.qt_stride = qt_stride;
		t.ef = ef;
		t.slots = sh.sm_count;
		*c = t;
		return 0;
	}
	const int wantW = tu.want_warps, wantR = tu.want_rings;
	if (wantW > 0 && wantW <= 32) bestW = (uint32_t) wantW;
	if (wantR > 0 && wantR <= (int) kMaxRings) bestR = (uint32_t) wantR;
	if (bestR > bestW) bestR = bestW;
	while (bestR > 1 && pool_bytes + bestW * t.priv_bytes + bestR * t.ring_bytes > max_cta) bestR--;
	if (pool_bytes + bestW * t.priv_bytes + bestR * t.ring_bytes > max_cta) return 2;
	t.warps = bestW;
	t.rings = bestR;
	t.off_pool = 0;
	t.off_ring = pool_bytes;
	t.off_priv = pool_bytes + bestR * t.ring_bytes;
	t.smem = t.off_priv + bestW * t.priv_bytes;
	t.row_smem = row_smem;
	t.qt_stride = qt_stride;
	t.ef = ef;
	t.slots = bestW * sh.sm_count;
	*c = t;
	return 0;
}

}  // namespace pgemb
