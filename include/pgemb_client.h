/*
 * pgemb_client.h -- what a backend process links against instead of libpgemb_b200.so when the device index is owned
 * by a pgemb_sidecar process (pg_embedding_b200/csrc/sidecar; protocol in csrc/sidecar/ipc.h).
 *
 * libpgemb_client.so contains no CUDA and no arithmetic: every call becomes a request in the sidecar's shared-memory
 * segment and is executed there by libpgemb_b200.so.  It exports
 *
 *   (1) the reference's own algorithm-side symbols, signature for signature (reference embedding.h:44-56), so that on
 *       the reference's link line (Makefile:6) it takes the place of `hnswalg.o distfunc.o` in a forked-backend world:
 *         hnsw_search / hnsw_bind_point / hnsw_dist_func / hnsw_init_dist_func / hnsw_is_deleted
 *       The HnswMetadata* they receive must be the first member of a PgembClientIndex (the reference's own
 *       "opaque with known prefix" convention for HnswIndex, embedding.c:65-75, :706);
 *   (2) the mirror-maintenance calls the glue in embedding.c makes (INTEGRATION.md): attach a relation, ship page
 *       records, read modified link lists back, mark labels deleted, truncate, drop.
 *
 * Concurrent hnsw_search calls of different backends are gathered by the sidecar into one batched traversal launch, and
 * concurrent index-less scans (pgemb_client_scan_topk) into one batched brute-force scan, and concurrent hnsw_dist_func
 * calls into one batched distance launch.
 * All functions returning int return 0 on success and a pgemb_status (include/pgemb_b200.h) otherwise;
 * pgemb_client_last_error() describes the last failure of the calling thread.
 */
#ifndef PGEMB_CLIENT_H
#define PGEMB_CLIENT_H

#include "pgemb_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct
{
	HnswMetadata meta;	  /* MUST be first (embedding.c:65-75) */
	uint64_t	 rel_key; /* identifies the relation across backends, e.g. (dbOid << 32) | relfilenode */
} PgembClientIndex;

/* Map the sidecar's segment (`shm_name` as given to `pgemb_sidecar --shm`, NULL: $PGEMB_SIDECAR_SHM) and wait up to
 * timeout_ms for the sidecar to serve.  Idempotent; the mapping is inherited across fork().
 * Replicas: a comma-separated list ("/pgemb0,/pgemb1", one sidecar per GPU) connects to all of them: requests that change
 * a mirror go to every replica in turn (the replicas stay bit-identical: binds are deterministic), reads of a mirror to
 * the first, and the searches of this process to one replica (pid modulo the count; $PGEMB_CLIENT_REPLICA overrides). */
int			pgemb_client_connect(const char *shm_name, int timeout_ms);
void		pgemb_client_disconnect(void);
const char *pgemb_client_last_error(void);
/* Name of the segment this process is (or was last) connected to; "" if never connected. */
const char *pgemb_client_segment_name(void);
/* Number of sidecars this process is connected to. */
int			pgemb_client_replicas(void);

/* Cancellation: `fn` (e.g. a function returning Postgres' InterruptPending) is polled about every 50 ms while a request is
 * pending; when it returns non-zero the call gives up with PGEMB_CLIENT_INTERRUPTED (the reference-shaped calls return
 * false) and the glue runs CHECK_FOR_INTERRUPTS().  The request itself is completed and dropped by the sidecar. */
#define PGEMB_CLIENT_INTERRUPTED 100
void pgemb_client_set_interrupt_check(int (*fn)(void));

/* Create-or-look-up the device mirror of relation h->rel_key with the options in h->meta (capacity is used on creation).
 * Fails if an existing mirror has other dims / maxM / distance function (the reference's check at embedding.c:594-602).
 * size_out / capacity_out (optional): nodes stored / capacity of the mirror. */
int pgemb_client_attach(PgembClientIndex *h, size_t capacity, size_t *size_out, size_t *capacity_out);
/* n records in the reference's on-page layout [count|links[maxM]|coords[dim]|label], record_stride bytes apart
 * (embedding.c:224-228, :619-621); node ids continue densely (embedding.c:693). */
int pgemb_client_append_records(PgembClientIndex *h, size_t n, const void *records, size_t record_stride);
int pgemb_client_export_records(PgembClientIndex *h, size_t first, size_t n, void *records, size_t record_stride);
/* links_out: n * (maxM + 1) u32, reference order [count, ids...] -- the write-back after hnsw_bind_point. */
int pgemb_client_get_links(PgembClientIndex *h, size_t first, size_t n, idx_t *links_out);
int pgemb_client_set_labels(PgembClientIndex *h, size_t first, size_t n, const label_t *labels);
int pgemb_client_size(PgembClientIndex *h, size_t *size_out, size_t *capacity_out);
int pgemb_client_truncate(PgembClientIndex *h);
int pgemb_client_drop(PgembClientIndex *h);
/* Bind the stored, unbound nodes [first, first+n) in id order: exact != 0 -> pgemb_build_exact (bit-identical to n
 * hnsw_bind_point calls), else pgemb_build_bulk. */
int pgemb_client_build(PgembClientIndex *h, size_t first, size_t n, size_t batch_max, int exact, double *seconds_out);
/* Sidecar counters: search launches, queries served, largest batch (how well concurrent callers were batched). */
int pgemb_client_stats(uint64_t *n_batches, uint64_t *n_searches, uint64_t *max_batch);

/* The index-less plan: what `SELECT ... ORDER BY val <op> q LIMIT k` returns with the index not used (one hnsw_dist_func per
 * row, embedding.c:1022-1062, then the executor's sort; the seq-scan block of test/expected/knn.out:63-91), for ONE query over
 * every row of relation h->rel_key's mirror.  It is pgemb_scan_topk (include/pgemb_b200.h) run by the sidecar:
 *   labels_out[k]  results ascending by (dist, label); labels with DELETED_FLAG are skipped
 *   dists_out[k]   optional (NULL): the matching distances, bit-identical to hnsw_dist_func's
 *   *n_out         number of results (< k when the relation has fewer live rows)
 * 1 <= k <= min(4096, the sidecar's --max-ef), else PGEMB_ERR_ARG before anything is sent.  Like hnsw_search it goes to this
 * process's replica and honours the interrupt check and the dead-sidecar bound.  The scans that backends have pending at
 * the same time for the same (relation, k) are served by one pgemb_scan_topk call: one pass over the table for all of them. */
int pgemb_client_scan_topk(PgembClientIndex *h, const coord_t *query, size_t k, label_t *labels_out, dist_t *dists_out, size_t *n_out);
/* Sidecar scan counters, summed over replicas (largest batch: the maximum): pgemb_scan_topk calls, scans served, largest
 * batch.  Scans are not counted by pgemb_client_stats. */
int pgemb_client_scan_stats(uint64_t *n_calls, uint64_t *n_scans, uint64_t *max_batch);
/* Sidecar distance counters, summed over replicas (largest batch: the maximum): pgemb_dist_batch calls, hnsw_dist_func pairs
 * served, largest batch.  The hnsw_dist_func calls that backends have pending at the same time for the same (metric, dim)
 * are served by one pgemb_dist_batch call, each with the bits of a one-pair call.  Distances are not counted by
 * pgemb_client_stats or pgemb_client_scan_stats. */
int pgemb_client_dist_stats(uint64_t *n_calls, uint64_t *n_dists, uint64_t *max_batch);
/* Ask the sidecar to exit (tests, controlled restarts). */
int pgemb_client_shutdown_server(void);

#ifdef __cplusplus
}
#endif
#endif
