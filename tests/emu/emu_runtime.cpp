// Scheduler and launcher of the host SIMT emulator (see fake_cuda/cuda_runtime.h).  Test infrastructure.
#include <cuda_runtime.h>
#include <signal.h>
#include <utility>
#include <vector>

namespace emu {

thread_local Warp *tl_warp = nullptr;
dim3			   g_block_dim, g_grid_dim;
pthread_mutex_t	   g_mbar_mu = PTHREAD_MUTEX_INITIALIZER;
int				   g_tma_late = 0;
int				   g_jitter = 0;
int				   g_tma_unwaited = 0;
int				   g_launch_error = 0;

// SIGUSR1 (e.g. `timeout -s USR1`): where every warp of the CTA in flight stands -- for hangs under the emulator
static Warp *volatile g_live[64];
static volatile unsigned g_live_n = 0;
static void dump_state(int)
{
	fprintf(stderr, "emu: state of the CTA in flight (%u warps)\n", g_live_n);
	for (unsigned wi = 0; wi < g_live_n && wi < 64; wi++)
	{
		Warp *w = g_live[wi];
		if (!w) continue;
		fprintf(stderr, "  warp %u kind %d bar %d cur %d:", wi, w->kind, w->bar_id, w->cur);
		for (int i = 0; i < 32; i++) fprintf(stderr, " %c%d", w->lane[i].st == DONE ? 'D' : w->lane[i].st == AT_COLL ? 'C' : 'R', w->lane[i].st == AT_COLL ? w->lane[i].site : 0);
		fprintf(stderr, "\n");
	}
}

static void lane_trampoline()
{
	Warp *w = tl_warp;
	w->body();
	w = tl_warp;
	w->lane[w->cur].st = DONE;
	// returning switches to uc_link (the warp's scheduler)
}

void run_warp(Warp &w)
{
	tl_warp = &w;
	for (int i = 0; i < 32; i++)
	{
		Lane &l = w.lane[i];
		l.stack = (char *) malloc(kLaneStack);
		getcontext(&l.ctx);
		l.ctx.uc_stack.ss_sp = l.stack;
		l.ctx.uc_stack.ss_size = kLaneStack;
		l.ctx.uc_link = &w.sched;
		makecontext(&l.ctx, (void (*)()) lane_trampoline, 0);
		l.st = RUNNABLE;
	}
	int rr = 0, last = -1;
	for (;;)
	{
		int pick = -1;
		for (int i = 0; i < 32; i++)
		{
			const int c = (rr + i) & 31;
			if (w.lane[c].st == RUNNABLE)
			{
				pick = c;
				break;
			}
		}
		if (pick >= 0)
		{
			if (pick == last) sched_yield();  // a lone spinning lane: give the other warps' threads the core
			last = pick;
			w.cur = pick;
			rr = pick + 1;
			swapcontext(&w.sched, &w.lane[pick].ctx);
			continue;
		}
		int live = 0;
		for (int i = 0; i < 32; i++) live += (w.lane[i].st != DONE);
		if (live == 0) break;
		// every live lane waits at a collective: exchange and release.  The kernels of this repo only use full-mask
		// collectives in warp-uniform control flow, so all waiting lanes must have arrived at the SAME call: lanes of
		// one warp meeting at different collectives is divergence the hardware would not reconcile the way this
		// scheduler does.
		{
			int site = -1;
			for (int i = 0; i < 32; i++)
			{
				if (w.lane[i].st != AT_COLL) continue;
				if (site < 0) site = w.lane[i].site;
				if (w.lane[i].site != site)
				{
					fprintf(stderr, "emu: lanes of one warp wait at different collectives (source lines %d and %d): divergent use of a full-mask collective\n", site, w.lane[i].site);
					abort();
				}
			}
		}
		if (w.kind == K_CTA_BAR) pthread_barrier_wait(&w.cta->bars[w.bar_id & 15]);
		unsigned cta_or = 0;
		if (w.kind == K_CTA_OR)
		{
			// __syncthreads_or: OR over the warp, then over the CTA (two barriers: publish, then everybody has read)
			unsigned mine = 0;
			for (int i = 0; i < 32; i++)
				if (w.lane[i].st == AT_COLL && w.lane[i].xchg) mine = 1;
			const int ph = w.or_phase;
			w.or_phase ^= 1;
			if (mine) __atomic_fetch_or(&w.cta->or_acc[ph], 1u, __ATOMIC_SEQ_CST);
			pthread_barrier_wait(&w.cta->bars[0]);
			cta_or = __atomic_load_n(&w.cta->or_acc[ph], __ATOMIC_SEQ_CST);
			if (pthread_barrier_wait(&w.cta->bars[0]) == PTHREAD_BARRIER_SERIAL_THREAD) __atomic_store_n(&w.cta->or_acc[ph], 0u, __ATOMIC_SEQ_CST);
		}
		for (int i = 0; i < 32; i++)
		{
			w.present[i] = (w.lane[i].st == AT_COLL);
			w.snap[i] = (w.kind == K_CTA_OR) ? cta_or : w.lane[i].xchg;
			if (w.lane[i].st == AT_COLL) w.lane[i].st = RUNNABLE;
		}
		rr = 0;
		last = -1;
	}
	for (int i = 0; i < 32; i++) free(w.lane[i].stack);
	tl_warp = nullptr;
}

// (threads per CTA, dynamic shared memory) of the first 4096 launches since the log was last read, and how many there
// were: lets a test see which launch configuration a host path chose (emu_launch_log below)
static std::vector<std::pair<unsigned, size_t>> g_launch_log;
static int										g_launch_count = 0;

void launch(dim3 grid, unsigned block_threads, size_t dyn_smem_bytes, const std::function<void()> &fn)
{
	if (g_launch_log.size() < 4096) g_launch_log.emplace_back(block_threads, dyn_smem_bytes);
	g_launch_count++;
	if (dyn_smem_bytes > kMaxDynamicSmem)
	{
		g_launch_error = 1;  // cudaErrorInvalidValue: the device refuses the launch and runs nothing
		return;
	}
	g_grid_dim = grid;
	g_block_dim = dim3(block_threads);
	{
		const char *m = getenv("PGEMB_EMU_TMA");
		g_tma_late = (m && strcmp(m, "late") == 0) ? 1 : 0;
		const char *j = getenv("PGEMB_EMU_JITTER");
		g_jitter = (j && *j && atoi(j) != 0) ? 1 : 0;
	}
	const unsigned nwarps = (block_threads + 31) / 32;
	static bool handler = false;
	if (!handler)
	{
		handler = true;
		signal(SIGUSR1, dump_state);
	}
	for (unsigned by = 0; by < grid.y; by++)
		for (unsigned bx = 0; bx < grid.x; bx++)
		{
			Cta cta;
			cta.nwarps = nwarps;
			cta.block_idx = dim3(bx, by);
			for (auto &b : cta.bars) pthread_barrier_init(&b, nullptr, nwarps);
			cta.dyn_smem = nullptr;
			if (dyn_smem_bytes)
			{
				cta.dyn_smem = (unsigned char *) aligned_alloc(128, (dyn_smem_bytes + 127) / 128 * 128);
				memset(cta.dyn_smem, 0xAA, dyn_smem_bytes);	// shared memory starts uninitialised on the device too
			}
			std::vector<std::thread> th;
			std::vector<Warp *>		 warps(nwarps);
			for (unsigned wi = 0; wi < nwarps; wi++)
			{
				Warp *w = new Warp();
				warps[wi] = w;
				w->cta = &cta;
				w->body = fn;
				for (int l = 0; l < 32; l++) w->lane[l].tid = dim3(wi * 32 + l);
				if (wi < 64) g_live[wi] = w;
				g_live_n = wi + 1;
				th.emplace_back([w]() { run_warp(*w); });
			}
			for (auto &t : th) t.join();
			g_live_n = 0;
			for (auto *w : warps)
			{
				for (int l = 0; l < 32; l++)
					if (!w->lane[l].cp_pending.empty())
					{
						g_tma_unwaited += (int) w->lane[l].cp_pending.size();
						fprintf(stderr, "emu: %zu cp.async pieces of a thread were never waited for (CTA %u)\n", w->lane[l].cp_pending.size(), bx);
					}
				delete w;
			}
			if (!cta.pending.empty())
			{
				// a bulk copy nobody waited for would land in the shared memory of a CTA that is gone
				g_tma_unwaited += (int) cta.pending.size();
				fprintf(stderr, "emu: %zu bulk copies were still in flight when CTA %u exited\n", cta.pending.size(), bx);
			}
			for (auto &b : cta.bars) pthread_barrier_destroy(&b);
			free(cta.dyn_smem);
		}
}

}  // namespace emu

extern "C" int emu_tma_unwaited() { return emu::g_tma_unwaited; }

// Copies up to `cap` entries of the launch log (oldest first), clears it and returns how many launches there were since
// it was last read.
extern "C" int emu_launch_log(unsigned *threads, size_t *smem, int cap)
{
	const int n = emu::g_launch_count;
	for (int i = 0; i < (int) emu::g_launch_log.size() && i < cap; i++)
	{
		threads[i] = emu::g_launch_log[i].first;
		smem[i] = emu::g_launch_log[i].second;
	}
	emu::g_launch_log.clear();
	emu::g_launch_count = 0;
	return n;
}
