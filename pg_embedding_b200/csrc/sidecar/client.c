/*
 * client.c -- libpgemb_client.so: the backend-side half of the sidecar protocol (ipc.h, include/pgemb_client.h).
 * Plain C, no CUDA, no arithmetic: every call is a request executed by a pgemb_sidecar with libpgemb_b200.so.
 *
 * Reference-shaped exports: hnsw_search (embedding.h:46, hnswalg.cpp:256-277), hnsw_bind_point (embedding.h:47,
 * hnswalg.cpp:279-291), hnsw_dist_func / hnsw_init_dist_func (embedding.h:55-56, distfunc.c:157-174), hnsw_is_deleted
 * (embedding.h:44, embedding.c:948-953) -- same signatures, ownership (results are malloc()ed here, free()d by the
 * caller, embedding.c:327) and failure behaviour (false, never an exception or a longjmp).
 *
 * Replicas (one sidecar per GPU; DESIGN.md section 7: the index fits one GPU, so GPUs are replicas and queries are split):
 * the segment name may be a comma-separated list.  Every request that CHANGES a mirror (attach, records, bind, labels,
 * truncate, drop, build) goes to all sidecars in turn -- binds are deterministic, so the replicas stay bit-identical --
 * reads of a mirror go to the first, and this process's searches go to one replica chosen by its pid.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <fcntl.h>
#include <linux/futex.h>
#include <math.h>
#include <sched.h>
#include <signal.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <time.h>
#include <unistd.h>

#include "../../../include/pgemb_client.h"
#include "ipc.h"

#define PGEMB_INTERRUPTED_COMPLETED 101 /* internal: interrupted, but the request had completed (slot already freed by us) */
#define PGEMB_MAX_REPLICAS 16

typedef struct
{
	PgembIpcHeader *hdr;
	unsigned char  *base;
	size_t			bytes;
} Conn;

static Conn			 g_conn[PGEMB_MAX_REPLICAS];
static int			 g_nconn = 0;
static char			 g_names[1024]; /* the list we connected to last: restarted sidecars re-create their segments under the same names */
static __thread char g_err[256];
static int (*g_interrupt)(void) = NULL; /* e.g. a function returning InterruptPending: polled while a request is pending */

static void set_err(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
}

const char *pgemb_client_last_error(void) { return g_err; }
const char *pgemb_client_segment_name(void) { return g_names; }
int			pgemb_client_replicas(void) { return g_nconn; }
void		pgemb_client_set_interrupt_check(int (*fn)(void)) { g_interrupt = fn; }

static inline uint32_t ld(const uint32_t *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline void	   st(uint32_t *p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static long futex(uint32_t *addr, int op, uint32_t val, const struct timespec *ts) { return syscall(SYS_futex, addr, op, val, ts, NULL, 0); }

static double now_s(void)
{
	struct timespec t;
	clock_gettime(CLOCK_MONOTONIC, &t);
	return (double) t.tv_sec + 1e-9 * (double) t.tv_nsec;
}

static PgembIpcSlot *slot_at(const Conn *c, uint32_t i) { return (PgembIpcSlot *) (c->base + c->hdr->slots_off + (size_t) i * c->hdr->slot_stride); }
static float		*slot_vec(PgembIpcSlot *s) { return (float *) ((unsigned char *) s + pgemb_ipc_payload_vec_off()); }
static label_t		*slot_labels(const Conn *c, PgembIpcSlot *s) { return (label_t *) ((unsigned char *) s + pgemb_ipc_payload_labels_off(c->hdr->max_dim)); }
static dist_t		*slot_dists(const Conn *c, PgembIpcSlot *s)
{
	return (dist_t *) ((unsigned char *) s + pgemb_ipc_payload_dists_off(c->hdr->max_dim, c->hdr->max_ef));
}

static int server_alive(const Conn *c)
{
	if (!c->hdr || !ld(&c->hdr->ready)) return 0;
	const pid_t pid = (pid_t) c->hdr->server_pid;
	return pid > 0 && (kill(pid, 0) == 0 || errno != ESRCH);
}

static void conn_close(Conn *c)
{
	if (c->base) munmap(c->base, c->bytes);
	c->base = NULL;
	c->hdr = NULL;
	c->bytes = 0;
}

/* map one segment and check that a live sidecar serves it */
static int conn_open(Conn *c, const char *name, double deadline)
{
	for (;;)
	{
		const int fd = shm_open(name, O_RDWR, 0600);
		if (fd >= 0)
		{
			struct stat sb;
			if (fstat(fd, &sb) == 0 && (size_t) sb.st_size >= sizeof(PgembIpcHeader))
			{
				void *mem = mmap(NULL, (size_t) sb.st_size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
				if (mem != MAP_FAILED)
				{
					PgembIpcHeader *h = (PgembIpcHeader *) mem;
					if (__atomic_load_n(&h->magic, __ATOMIC_ACQUIRE) == PGEMB_IPC_MAGIC && h->version == PGEMB_IPC_VERSION && ld(&h->ready) &&
						(size_t) sb.st_size >= h->bulk_off + h->bulk_bytes)
					{
						c->hdr = h;
						c->base = (unsigned char *) mem;
						c->bytes = (size_t) sb.st_size;
						if (server_alive(c))
						{
							close(fd);
							return PGEMB_OK;
						}
						c->hdr = NULL;
						c->base = NULL;
					}
					munmap(mem, (size_t) sb.st_size);
				}
			}
			close(fd);
		}
		if (now_s() >= deadline) break;
		usleep(2000);
	}
	set_err("pgemb_client_connect: no sidecar is serving %s", name);
	return PGEMB_ERR_STATE;
}

static int all_alive(void)
{
	if (g_nconn == 0) return 0;
	for (int i = 0; i < g_nconn; i++)
		if (!server_alive(&g_conn[i])) return 0;
	return 1;
}

void pgemb_client_disconnect(void)
{
	for (int i = 0; i < g_nconn; i++) conn_close(&g_conn[i]);
	g_nconn = 0;
}

int pgemb_client_connect(const char *shm_names, int timeout_ms)
{
	if (all_alive()) return PGEMB_OK;
	pgemb_client_disconnect(); /* a sidecar we were mapped to is gone: look for its successor */
	if ((!shm_names || !*shm_names) && g_names[0]) shm_names = g_names;
	if (!shm_names || !*shm_names) shm_names = getenv("PGEMB_SIDECAR_SHM");
	if (!shm_names || !*shm_names)
	{
		set_err("pgemb_client_connect: no segment name (argument or PGEMB_SIDECAR_SHM)");
		return PGEMB_ERR_ARG;
	}
	char list[sizeof(g_names)];
	snprintf(list, sizeof(list), "%s", shm_names);
	const double deadline = now_s() + 1e-3 * (double) (timeout_ms > 0 ? timeout_ms : 0);
	char		*save = NULL;
	int			 n = 0, rc = PGEMB_OK;
	for (char *tok = strtok_r(list, ",", &save); tok && rc == PGEMB_OK; tok = strtok_r(NULL, ",", &save))
	{
		while (*tok == ' ') tok++;
		if (!*tok) continue;
		if (n == PGEMB_MAX_REPLICAS)
		{
			set_err("pgemb_client_connect: more than %d replicas", PGEMB_MAX_REPLICAS);
			rc = PGEMB_ERR_ARG;
			break;
		}
		rc = conn_open(&g_conn[n], tok, deadline);
		if (rc == PGEMB_OK) n++;
	}
	if (rc == PGEMB_OK && n == 0)
	{
		set_err("pgemb_client_connect: empty segment list");
		rc = PGEMB_ERR_ARG;
	}
	if (rc != PGEMB_OK)
	{
		for (int i = 0; i < n; i++) conn_close(&g_conn[i]); /* all or nothing */
		return rc;
	}
	g_nconn = n;
	if (shm_names != g_names) snprintf(g_names, sizeof(g_names), "%s", shm_names);
	return PGEMB_OK;
}

static int ensure_connected(void)
{
	if (all_alive()) return PGEMB_OK;
	return pgemb_client_connect(NULL, 0);
}

/* the replica this process sends its searches to: PGEMB_CLIENT_REPLICA, else chosen by the pid */
static const Conn *search_conn(void)
{
	const char *e = getenv("PGEMB_CLIENT_REPLICA");
	if (e && *e) return &g_conn[(unsigned) atoi(e) % (unsigned) g_nconn];
	return &g_conn[(unsigned) getpid() % (unsigned) g_nconn];
}

/* ---- one request ------------------------------------------------------------------------------------------------ */
static PgembIpcSlot *claim_slot(const Conn *c)
{
	const uint32_t n = c->hdr->n_slots;
	uint32_t	   start = ((uint32_t) getpid() * 2654435761u) % n;
	const double   deadline = now_s() + 10.0;
	for (;;)
	{
		for (uint32_t k = 0; k < n; k++)
		{
			PgembIpcSlot *s = slot_at(c, (start + k) % n);
			uint32_t	  expect = PGEMB_SLOT_FREE;
			if (ld(&s->state) == PGEMB_SLOT_FREE &&
				__atomic_compare_exchange_n(&s->state, &expect, PGEMB_SLOT_CLAIMED, 0, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED))
			{
				/* ownership: the previous user cleared owner_pid before it freed the slot (release_slot, the sidecar's own frees), so
				 * between the CAS above and this store the sidecar's reclaim() sees pid 0 and leaves the slot alone */
				__atomic_store_n(&s->owner_pid, (int32_t) getpid(), __ATOMIC_RELEASE);
				s->status = 0;
				s->n_out = 0;
				s->a0 = s->a1 = s->a2 = s->a3 = 0;
				s->ef = 0;
				s->err[0] = 0;
				st(&s->abandoned, 0);
				return s;
			}
		}
		if (!server_alive(c) || now_s() > deadline)
		{
			set_err("no free request slot (sidecar %s)", server_alive(c) ? "busy" : "gone");
			return NULL;
		}
		sched_yield();
	}
}

/* publish a filled slot, wait for the result; returns the request's status (the slot stays DONE: caller releases it) */
static int submit_wait(const Conn *c, PgembIpcSlot *s)
{
	st(&s->state, PGEMB_SLOT_READY);
	__atomic_fetch_add(&c->hdr->submit_seq, 1u, __ATOMIC_SEQ_CST);
	__atomic_thread_fence(__ATOMIC_SEQ_CST);
	if (ld(&c->hdr->server_sleeping)) futex(&c->hdr->submit_seq, FUTEX_WAKE, 1, NULL);
	/* a served request takes tens of microseconds to milliseconds: poll briefly, then sleep on the slot's futex */
	static double spin_s = -1.0; /* PGEMB_CLIENT_SPIN_US: how long a caller polls before it sleeps (default 50; a latency-critical
								  * deployment with few backends may spin for a whole search, ~600 us, and save the wake-up) */
	if (spin_s < 0.0)
	{
		const char *e = getenv("PGEMB_CLIENT_SPIN_US");
		spin_s = (e && *e) ? 1e-6 * atof(e) : 50e-6;
	}
	const double spin_until = now_s() + spin_s;
	for (;;)
	{
		uint32_t v = ld(&s->state);
		if (v == PGEMB_SLOT_DONE) break;
		if (now_s() < spin_until)
		{
			__builtin_ia32_pause();
			continue;
		}
		struct timespec ts = {0, 50 * 1000 * 1000};
		futex(&s->state, FUTEX_WAIT, v, &ts);
		if (g_interrupt && ld(&s->state) != PGEMB_SLOT_DONE && g_interrupt())
		{
			/* the caller wants out (query cancel): leave the request to the sidecar, never touch the slot again except to free
			 * it if the result arrived in the meantime */
			st(&s->abandoned, 1);
			__atomic_thread_fence(__ATOMIC_SEQ_CST);
			uint32_t  expect = PGEMB_SLOT_DONE;
			const int freed_here = __atomic_compare_exchange_n(&s->state, &expect, (uint32_t) PGEMB_SLOT_FREE, 0, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED);
			set_err("interrupted while waiting for the sidecar");
			/* freed_here: the request had just completed and we dropped its result; otherwise the sidecar completes it,
			 * frees the slot and (for a bulk request) the bulk area */
			return freed_here ? PGEMB_INTERRUPTED_COMPLETED : PGEMB_CLIENT_INTERRUPTED;
		}
		if (ld(&s->state) != PGEMB_SLOT_DONE && !server_alive(c))
		{
			set_err("the sidecar went away while a request was pending");
			/* the slot is lost to this segment; a new sidecar creates a new one */
			return PGEMB_ERR_STATE;
		}
	}
	if (s->status != PGEMB_OK) set_err("%s", s->err);
	return s->status;
}

static int interrupted(int rc) { return rc == PGEMB_CLIENT_INTERRUPTED || rc == PGEMB_INTERRUPTED_COMPLETED; }
/* give a slot back after submit_wait() -- unless the request was abandoned: then the slot is not ours any more */
static void release_slot(PgembIpcSlot *s, int rc)
{
	if (!interrupted(rc) && ld(&s->state) == PGEMB_SLOT_DONE)
	{
		__atomic_store_n(&s->owner_pid, 0, __ATOMIC_RELEASE); /* never leave a stale pid on a FREE slot (see claim_slot) */
		st(&s->state, PGEMB_SLOT_FREE);
	}
}

/* the bulk area is one request's at a time */
static int bulk_acquire(const Conn *c)
{
	const uint32_t me = (uint32_t) getpid();
	const double   deadline = now_s() + 60.0;
	for (;;)
	{
		uint32_t expect = 0;
		if (__atomic_compare_exchange_n(&c->hdr->bulk_lock, &expect, me, 0, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED)) return PGEMB_OK;
		if (!server_alive(c) || now_s() > deadline)
		{
			set_err("bulk area unavailable");
			return PGEMB_ERR_STATE;
		}
		usleep(50);
	}
}
static void bulk_release(const Conn *c) { st(&c->hdr->bulk_lock, 0); }

/* a request without payload on one connection (never re-maps: callers may hold pointers into the segment) */
static int do_request(const Conn *c, PgembClientIndex *h, uint32_t op, uint64_t a0, uint64_t a1, uint64_t a2, uint64_t a3, uint64_t *r0,
					  uint64_t *r1, uint64_t *r2)
{
	int			  rc;
	PgembIpcSlot *s = claim_slot(c);
	if (!s) return PGEMB_ERR_STATE;
	s->op = op;
	s->index_key = h ? h->rel_key : 0;
	s->a0 = a0;
	s->a1 = a1;
	s->a2 = a2;
	s->a3 = a3;
	rc = submit_wait(c, s);
	if (r0) *r0 = s->a0;
	if (r1) *r1 = s->a1;
	if (r2) *r2 = s->a2;
	release_slot(s, rc);
	return rc;
}

/* `all` != 0: the request changes a mirror -> every replica, results from the first; else the first replica only */
static int simple_request(int all, PgembClientIndex *h, uint32_t op, uint64_t a0, uint64_t a1, uint64_t a2, uint64_t a3, uint64_t *r0, uint64_t *r1,
						  uint64_t *r2)
{
	int rc = ensure_connected();
	if (rc) return rc;
	const int n = all ? g_nconn : 1;
	for (int i = 0; i < n && rc == PGEMB_OK; i++)
		rc = do_request(&g_conn[i], h, op, a0, a1, a2, a3, i == 0 ? r0 : NULL, i == 0 ? r1 : NULL, i == 0 ? r2 : NULL);
	return interrupted(rc) ? PGEMB_CLIENT_INTERRUPTED : rc;
}

/* ---- mirror maintenance ------------------------------------------------------------------------------------------ */
int pgemb_client_attach(PgembClientIndex *h, size_t capacity, size_t *size_out, size_t *capacity_out)
{
	if (!h)
	{
		set_err("null index");
		return PGEMB_ERR_ARG;
	}
	int rc = ensure_connected();
	if (rc) return rc;
	for (int i = 0; i < g_nconn && rc == PGEMB_OK; i++)
	{
		const Conn	 *c = &g_conn[i];
		PgembIpcSlot *s = claim_slot(c);
		if (!s) return PGEMB_ERR_STATE;
		s->op = PGEMB_OP_ATTACH;
		s->index_key = h->rel_key;
		s->a0 = capacity;
		memcpy(slot_vec(s), &h->meta, sizeof(HnswMetadata));
		rc = submit_wait(c, s);
		if (rc == PGEMB_OK)
		{
			/* replicas hold the same nodes; should one be behind (a restarted sidecar), report the smallest so that the glue
			 * notices */
			if (size_out && (i == 0 || (size_t) s->a1 < *size_out)) *size_out = (size_t) s->a1;
			if (capacity_out && (i == 0 || (size_t) s->a2 < *capacity_out)) *capacity_out = (size_t) s->a2;
		}
		release_slot(s, rc);
	}
	return interrupted(rc) ? PGEMB_CLIENT_INTERRUPTED : rc;
}

/* move `n` items of `item_bytes` through one connection's bulk area in chunks; to_server: copy in before each request, else copy out after */
static int bulk_transfer_conn(const Conn *c, PgembClientIndex *h, uint32_t op, size_t first, size_t n, size_t item_bytes, uint64_t stride_arg, void *data,
							  int to_server)
{
	if (item_bytes == 0 || item_bytes > c->hdr->bulk_bytes)
	{
		set_err("item larger than the sidecar's bulk area");
		return PGEMB_ERR_ARG;
	}
	const size_t per = c->hdr->bulk_bytes / item_bytes;
	int			 rc = bulk_acquire(c);
	if (rc) return rc;
	unsigned char *bulk = c->base + c->hdr->bulk_off;
	for (size_t done = 0; done < n && rc == PGEMB_OK; done += per)
	{
		const size_t k = (n - done < per) ? (n - done) : per;
		if (to_server) memcpy(bulk, (const unsigned char *) data + done * item_bytes, k * item_bytes);
		if (op == PGEMB_OP_APPEND_RECORDS)
			rc = do_request(c, h, op, k, stride_arg, 0, 0, NULL, NULL, NULL);
		else
			rc = do_request(c, h, op, first + done, k, stride_arg, 0, NULL, NULL, NULL);
		if (rc == PGEMB_OK && !to_server) memcpy((unsigned char *) data + done * item_bytes, bulk, k * item_bytes);
	}
	/* an abandoned request still uses the bulk area: the sidecar lets go of it when that request is done */
	if (rc != PGEMB_CLIENT_INTERRUPTED) bulk_release(c);
	return rc;
}

static int bulk_transfer(PgembClientIndex *h, uint32_t op, size_t first, size_t n, size_t item_bytes, uint64_t stride_arg, void *data, int to_server)
{
	if (!h || (!data && n))
	{
		set_err("null argument");
		return PGEMB_ERR_ARG;
	}
	if (n == 0) return PGEMB_OK;
	int rc = ensure_connected();
	if (rc) return rc;
	const int replicas = to_server ? g_nconn : 1; /* writes reach every replica, reads come from the first */
	for (int i = 0; i < replicas && rc == PGEMB_OK; i++) rc = bulk_transfer_conn(&g_conn[i], h, op, first, n, item_bytes, stride_arg, data, to_server);
	return interrupted(rc) ? PGEMB_CLIENT_INTERRUPTED : rc;
}

int pgemb_client_append_records(PgembClientIndex *h, size_t n, const void *records, size_t record_stride)
{
	return bulk_transfer(h, PGEMB_OP_APPEND_RECORDS, 0, n, record_stride, record_stride, (void *) records, 1);
}

int pgemb_client_export_records(PgembClientIndex *h, size_t first, size_t n, void *records, size_t record_stride)
{
	return bulk_transfer(h, PGEMB_OP_EXPORT_RECORDS, first, n, record_stride, record_stride, records, 0);
}

int pgemb_client_get_links(PgembClientIndex *h, size_t first, size_t n, idx_t *links_out)
{
	if (!h)
	{
		set_err("null index");
		return PGEMB_ERR_ARG;
	}
	return bulk_transfer(h, PGEMB_OP_GET_LINKS, first, n, (h->meta.maxM + 1) * sizeof(idx_t), 0, links_out, 0);
}

int pgemb_client_set_labels(PgembClientIndex *h, size_t first, size_t n, const label_t *labels)
{
	return bulk_transfer(h, PGEMB_OP_SET_LABELS, first, n, sizeof(label_t), 0, (void *) labels, 1);
}

int pgemb_client_size(PgembClientIndex *h, size_t *size_out, size_t *capacity_out)
{
	uint64_t  a = 0, b = 0;
	const int rc = simple_request(0, h, PGEMB_OP_SIZE, 0, 0, 0, 0, &a, &b, NULL);
	if (rc == PGEMB_OK)
	{
		if (size_out) *size_out = (size_t) a;
		if (capacity_out) *capacity_out = (size_t) b;
	}
	return rc;
}

int pgemb_client_truncate(PgembClientIndex *h) { return simple_request(1, h, PGEMB_OP_TRUNCATE, 0, 0, 0, 0, NULL, NULL, NULL); }
int pgemb_client_drop(PgembClientIndex *h) { return simple_request(1, h, PGEMB_OP_DROP, 0, 0, 0, 0, NULL, NULL, NULL); }

int pgemb_client_build(PgembClientIndex *h, size_t first, size_t n, size_t batch_max, int exact, double *seconds_out)
{
	uint64_t  sec_bits = 0;
	const int rc = simple_request(1, h, PGEMB_OP_BUILD, first, n, batch_max, exact ? 1 : 0, NULL, NULL, &sec_bits);
	if (rc == PGEMB_OK && seconds_out) memcpy(seconds_out, &sec_bits, sizeof(double));
	return rc;
}

int pgemb_client_stats(uint64_t *n_batches, uint64_t *n_searches, uint64_t *max_batch)
{
	const int rc = ensure_connected();
	if (rc) return rc;
	uint64_t b = 0, s = 0, m = 0;
	for (int i = 0; i < g_nconn; i++)
	{
		b += __atomic_load_n(&g_conn[i].hdr->n_batches, __ATOMIC_RELAXED);
		s += __atomic_load_n(&g_conn[i].hdr->n_searches, __ATOMIC_RELAXED);
		const uint64_t mi = __atomic_load_n(&g_conn[i].hdr->max_batch, __ATOMIC_RELAXED);
		if (mi > m) m = mi;
	}
	if (n_batches) *n_batches = b;
	if (n_searches) *n_searches = s;
	if (max_batch) *max_batch = m;
	return PGEMB_OK;
}

int pgemb_client_scan_stats(uint64_t *n_calls, uint64_t *n_scans, uint64_t *max_batch)
{
	const int rc = ensure_connected();
	if (rc) return rc;
	uint64_t c = 0, s = 0, m = 0;
	for (int i = 0; i < g_nconn; i++)
	{
		c += __atomic_load_n(&g_conn[i].hdr->n_scan_calls, __ATOMIC_RELAXED);
		s += __atomic_load_n(&g_conn[i].hdr->n_scans, __ATOMIC_RELAXED);
		const uint64_t mi = __atomic_load_n(&g_conn[i].hdr->max_scan_batch, __ATOMIC_RELAXED);
		if (mi > m) m = mi;
	}
	if (n_calls) *n_calls = c;
	if (n_scans) *n_scans = s;
	if (max_batch) *max_batch = m;
	return PGEMB_OK;
}

int pgemb_client_dist_stats(uint64_t *n_calls, uint64_t *n_dists, uint64_t *max_batch)
{
	const int rc = ensure_connected();
	if (rc) return rc;
	uint64_t c = 0, d = 0, m = 0;
	for (int i = 0; i < g_nconn; i++)
	{
		c += __atomic_load_n(&g_conn[i].hdr->n_dist_calls, __ATOMIC_RELAXED);
		d += __atomic_load_n(&g_conn[i].hdr->n_dists, __ATOMIC_RELAXED);
		const uint64_t mi = __atomic_load_n(&g_conn[i].hdr->max_dist_batch, __ATOMIC_RELAXED);
		if (mi > m) m = mi;
	}
	if (n_calls) *n_calls = c;
	if (n_dists) *n_dists = d;
	if (max_batch) *max_batch = m;
	return PGEMB_OK;
}

/* ---- the index-less scan (embedding.c:1022-1062 per row + the executor's sort; knn.out:63-91) ------------------------- */
int pgemb_client_scan_topk(PgembClientIndex *h, const coord_t *query, size_t k, label_t *labels_out, dist_t *dists_out, size_t *n_out)
{
	if (!h || !query || !labels_out || !n_out)
	{
		set_err("pgemb_client_scan_topk: null argument");
		return PGEMB_ERR_ARG;
	}
	int rc = ensure_connected();
	if (rc) return rc;
	const Conn	*c = search_conn();
	const size_t kmax = c->hdr->max_ef < 4096 ? c->hdr->max_ef : 4096;
	if (k < 1 || k > kmax)
	{
		set_err("pgemb_client_scan_topk: k = %zu outside 1 .. %zu (min(4096, the sidecar's --max-ef))", k, kmax);
		return PGEMB_ERR_ARG;
	}
	if (h->meta.dim < 1 || h->meta.dim > c->hdr->max_dim)
	{
		set_err("pgemb_client_scan_topk: dims outside the sidecar's limits");
		return PGEMB_ERR_ARG;
	}
	PgembIpcSlot *s = claim_slot(c);
	if (!s) return PGEMB_ERR_STATE;
	s->op = PGEMB_OP_SCAN;
	s->index_key = h->rel_key;
	s->a0 = k;
	memcpy(slot_vec(s), query, h->meta.dim * sizeof(coord_t));
	rc = submit_wait(c, s);
	if (rc == PGEMB_OK)
	{
		if (s->n_out >= 0 && (size_t) s->n_out <= k)
		{
			const size_t n = (size_t) s->n_out;
			memcpy(labels_out, slot_labels(c, s), n * sizeof(label_t));
			if (dists_out) memcpy(dists_out, slot_dists(c, s), n * sizeof(dist_t));
			*n_out = n;
		}
		else
		{
			set_err("pgemb_client_scan_topk: the sidecar returned %d results for k = %zu", (int) s->n_out, k);
			rc = PGEMB_ERR_STATE;
		}
	}
	release_slot(s, rc);
	return interrupted(rc) ? PGEMB_CLIENT_INTERRUPTED : rc;
}

int pgemb_client_shutdown_server(void) { return simple_request(1, NULL, PGEMB_OP_SHUTDOWN, 0, 0, 0, 0, NULL, NULL, NULL); }

/* ---- the reference's algorithm-side symbols (embedding.h:44-56) -------------------------------------------------------- */
bool hnsw_search(HnswMetadata *meta, const coord_t *point, size_t *n_results, label_t **results)
{
	if (!meta || !point || !n_results || !results) return false;
	PgembClientIndex *h = (PgembClientIndex *) meta; /* embedding.c:706: the metadata is the first member of the handle */
	if (ensure_connected() != PGEMB_OK) return false;
	const Conn	*c = search_conn();
	const size_t ef = meta->efSearch; /* re-read on every call: the caller doubles it (embedding.c:334) */
	if (ef < 1 || ef > c->hdr->max_ef || meta->dim < 1 || meta->dim > c->hdr->max_dim)
	{
		set_err("hnsw_search: efSearch or dims outside the sidecar's limits");
		return false;
	}
	label_t *buf = (label_t *) malloc(ef * sizeof(label_t));
	if (!buf) return false;
	PgembIpcSlot *s = claim_slot(c);
	if (!s)
	{
		free(buf);
		return false;
	}
	s->op = PGEMB_OP_SEARCH;
	s->index_key = h->rel_key;
	s->ef = (uint32_t) ef;
	memcpy(slot_vec(s), point, meta->dim * sizeof(coord_t));
	const int rc = submit_wait(c, s);
	bool	  ok = false;
	if (rc == PGEMB_OK && s->n_out >= 0 && (size_t) s->n_out <= ef)
	{
		memcpy(buf, slot_labels(c, s), (size_t) s->n_out * sizeof(label_t));
		*n_results = (size_t) s->n_out;
		*results = buf;
		ok = true;
	}
	release_slot(s, rc);
	if (!ok) free(buf);
	return ok;
}

bool hnsw_bind_point(HnswMetadata *meta, const coord_t *point, idx_t cur)
{
	(void) point; /* the node's record was shipped to the mirror before this call (embedding.c:619-621 stores it first) */
	if (!meta) return false;
	PgembClientIndex *h = (PgembClientIndex *) meta;
	const int		  rc = simple_request(1, h, PGEMB_OP_BIND, cur, meta->efConstruction, 0, 0, NULL, NULL, NULL);
	if (rc != PGEMB_OK)
	{
		fprintf(stderr, "Catch %s\n", pgemb_client_last_error()); /* hnswalg.cpp:288 */
		return false;
	}
	return true;
}

dist_t hnsw_dist_func(dist_func_t dist, coord_t const *ax, coord_t const *bx, size_t dim)
{
	if (!ax || !bx || ensure_connected() != PGEMB_OK) return NAN;
	const Conn *c = search_conn();
	if (dim < 1 || dim > c->hdr->max_dim) return NAN;
	PgembIpcSlot *s = claim_slot(c);
	if (!s) return NAN;
	s->op = PGEMB_OP_DIST;
	s->index_key = 0;
	s->a0 = dim;
	s->a1 = (uint64_t) dist;
	memcpy(slot_vec(s), ax, dim * sizeof(coord_t));
	memcpy(slot_vec(s) + c->hdr->max_dim, bx, dim * sizeof(coord_t));
	const int rc = submit_wait(c, s);
	float	  out = NAN;
	if (rc == PGEMB_OK)
	{
		const uint32_t bits = (uint32_t) s->a2;
		memcpy(&out, &bits, 4);
	}
	release_slot(s, rc);
	return out;
}

void hnsw_init_dist_func(void) { (void) pgemb_client_connect(NULL, 0); } /* called once from _PG_init (embedding.c:150) */

bool hnsw_is_deleted(label_t label) { return ((label >> 48) & 1u) != 0; } /* embedding.c:44, :948-953 */
