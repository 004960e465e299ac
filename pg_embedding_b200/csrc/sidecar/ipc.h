/*
 * ipc.h -- shared-memory protocol between pgemb_sidecar (the one process that owns the CUDA context and the HBM
 * mirrors of the hnsw relations) and its clients (libpgemb_client.so inside every backend process).
 *
 * Why it exists (SURVEY.md section 7 "Postgres process model", section 8(b) "Handle", 8(f4)): backends are forked
 * processes, a CUDA context does not survive fork(), and HnswIndex is re-created per scan (embedding.c:217,254,574) --
 * so the device index has to live in one GPU-owning process and be keyed by relation.  The reference calls
 * hnsw_search one query at a time (embedding.c:317,335); many backends doing so concurrently is exactly the batch the
 * traversal kernel wants, so the sidecar gathers the requests that are pending at the same time into ONE
 * pgemb_search_batch launch.  Index-less scans (PGEMB_OP_SCAN) are gathered the same way, per (relation, k), into one
 * pgemb_scan_topk call, and one-pair distances (PGEMB_OP_DIST), per (metric, dim), into one pgemb_dist_batch call.
 *
 * One POSIX shared-memory segment:
 *     IpcHeader | IpcSlot[n_slots] (each followed by its payload) | bulk area
 * A request is a slot: a client claims a FREE slot (CAS), fills it, publishes READY and bumps header.submit_seq (a
 * futex the server sleeps on when idle); the server sets BUSY, runs it, writes the result into the same slot, publishes
 * DONE and wakes the futex on slot.state; the client copies the result out and returns the slot to FREE.  A client that has to stop waiting (query cancel) marks
 * the slot `abandoned`; the slot is then freed by whichever side sees DONE last, and its result is dropped.  Bulk data
 * (page records, link lists) travels through the bulk area, which a client holds exclusively (header.bulk_lock) for the
 * duration of one request.
 *
 * Both sides are built with GCC: all shared words are plain uint32_t/uint64_t accessed with __atomic builtins.
 */
#ifndef PGEMB_SIDECAR_IPC_H
#define PGEMB_SIDECAR_IPC_H

#include <stdint.h>
#include <stddef.h>

#define PGEMB_IPC_MAGIC 0x424d4750u /* "PGMB" */
#define PGEMB_IPC_VERSION 3u

enum
{
	PGEMB_SLOT_FREE = 0,
	PGEMB_SLOT_CLAIMED = 1, /* a client is filling it */
	PGEMB_SLOT_READY = 2,	/* published, waiting for the server */
	PGEMB_SLOT_BUSY = 3,	/* the server is working on it */
	PGEMB_SLOT_DONE = 4		/* result available */
};

enum
{
	PGEMB_OP_PING = 1,
	PGEMB_OP_ATTACH = 2,		  /* create-or-look-up the mirror of relation `index_key`; payload: HnswMetadata; a0 = capacity -> a1 = size, a2 = capacity */
	PGEMB_OP_APPEND_RECORDS = 3,  /* a0 = n, a1 = record stride, bulk area holds the records (embedding.c:619-621 layout) */
	PGEMB_OP_SEARCH = 4,		  /* ef, payload: query[dim] -> n_out, labels[n_out] (hnsw_search, hnswalg.cpp:256-277) */
	PGEMB_OP_BIND = 5,			  /* a0 = node id, a1 = efConstruction (hnsw_bind_point, hnswalg.cpp:279-291) */
	PGEMB_OP_GET_LINKS = 6,		  /* a0 = first, a1 = n -> bulk area: n * (maxM+1) u32 */
	PGEMB_OP_EXPORT_RECORDS = 7,  /* a0 = first, a1 = n, a2 = record stride -> bulk area */
	PGEMB_OP_SET_LABELS = 8,	  /* a0 = first, a1 = n, bulk area holds n u64 (vacuum: DELETED_FLAG, embedding.c:912-922) */
	PGEMB_OP_TRUNCATE = 9,
	PGEMB_OP_DROP = 10,
	PGEMB_OP_SIZE = 11,			  /* -> a0 = size, a1 = capacity */
	PGEMB_OP_BUILD = 12,		  /* a0 = first, a1 = n, a2 = batch_max, a3 = 1: exact (bit-identical to row-by-row), 0: bulk */
	PGEMB_OP_DIST = 13,			  /* a0 = dim, a1 = metric, payload: a[dim] b[dim] -> a2 = fp32 bits (hnsw_dist_func) */
	PGEMB_OP_SHUTDOWN = 14,
	PGEMB_OP_SCAN = 15			  /* a0 = k, payload: query[dim] -> n_out, labels[n_out], dists[n_out] (pgemb_scan_topk for one query) */
};

typedef struct
{
	uint32_t magic, version;
	uint32_t n_slots, max_dim, max_ef;
	uint32_t slot_stride;	 /* bytes from one slot to the next (header + payload) */
	uint64_t slots_off;		 /* byte offset of slot 0 */
	uint64_t bulk_off, bulk_bytes;
	uint32_t submit_seq;	 /* futex: bumped by a client after it published a request */
	uint32_t server_sleeping;/* 1 while the server is (about to be) blocked on submit_seq */
	uint32_t ready;			 /* 1 once the server serves requests, 0 again when it leaves */
	int32_t	 server_pid;
	uint32_t bulk_lock;		 /* 0 = free, else the pid of the client that owns the bulk area */
	uint32_t pad0;
	/* counters (server-written) */
	uint64_t n_batches;		 /* pgemb_search_batch launches */
	uint64_t n_searches;	 /* queries served */
	uint64_t max_batch;		 /* largest batch so far */
	uint64_t n_requests;	 /* all requests served */
	uint64_t n_scan_calls;	 /* pgemb_scan_topk calls (scans are not counted in n_batches / n_searches / max_batch) */
	uint64_t n_scans;		 /* scan queries served */
	uint64_t max_scan_batch; /* largest scan batch so far */
	uint64_t n_dist_calls;	 /* pgemb_dist_batch calls (distances are not counted in the search or scan counters) */
	uint64_t n_dists;		 /* distance pairs served */
	uint64_t max_dist_batch; /* largest distance batch so far */
} PgembIpcHeader;

typedef struct
{
	uint32_t state;	   /* PGEMB_SLOT_*; futex the client sleeps on while READY/BUSY */
	uint32_t op;
	int32_t	 status;   /* pgemb_status of the request (0 = OK) */
	int32_t	 owner_pid;
	uint64_t index_key;
	uint64_t a0, a1, a2, a3;
	uint32_t ef;
	int32_t	 n_out;
	uint32_t abandoned; /* set by a client that stopped waiting (query cancel): whoever sees DONE afterwards frees the slot */
	char	 err[164];
	/* payload follows: float vec[2 * max_dim]; uint64_t labels[max_ef]  (8-byte aligned); float dists[max_ef] */
} PgembIpcSlot;

static inline size_t pgemb_ipc_payload_vec_off(void) { return (sizeof(PgembIpcSlot) + 15u) & ~(size_t) 15u; }
static inline size_t pgemb_ipc_payload_labels_off(uint32_t max_dim) { return pgemb_ipc_payload_vec_off() + (((size_t) 2 * max_dim * 4 + 15u) & ~(size_t) 15u); }
static inline size_t pgemb_ipc_payload_dists_off(uint32_t max_dim, uint32_t max_ef) { return pgemb_ipc_payload_labels_off(max_dim) + (size_t) max_ef * 8; }
static inline size_t pgemb_ipc_slot_stride(uint32_t max_dim, uint32_t max_ef)
{
	return (pgemb_ipc_payload_dists_off(max_dim, max_ef) + (size_t) max_ef * 4 + 63u) & ~(size_t) 63u;
}

#endif
