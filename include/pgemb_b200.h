/*
 * pgemb_b200.h -- C ABI of the H100-native (sm_90a) HNSW candidate-scoring path for pg_embedding.
 *
 * Two groups of entry points:
 *
 *  (1) The reference's own boundary, kept symbol-for-symbol so that replacing
 *      `hnswalg.o distfunc.o` on the reference's link line (reference Makefile:6) with
 *      libpgemb_b200.so is the drop-in:                       reference embedding.h:17-56
 *        hnsw_search / hnsw_bind_point / hnsw_dist_func / hnsw_init_dist_func
 *      Types coord_t/dist_t/idx_t/label_t, dist_func_t and HnswMetadata have the reference's
 *      exact layout (embedding.h:17-42).
 *
 *  (2) Bulk entry points the callback-per-node reference interface cannot express
 *      (SURVEY.md section 8(b), last row): device-index lifecycle, node upload / link download,
 *      batched search, device-resident search, batched distances, sequential bind against the
 *      device mirror, bulk build, shard top-k merge.  All plain pointers and sizes.
 *
 * No torch / C++ types cross this boundary.  Every function that can fail returns a pgemb_status
 * (0 = OK) or, for the reference-shaped ones, the reference's bool.  pgemb_last_error() returns a
 * thread-local human-readable message for the last failure.
 *
 * There is NO CPU fallback behind any of these: if no CUDA device is usable they fail
 * (PGEMB_ERR_CUDA) -- see DESIGN.md "No fallback".
 */
#ifndef PGEMB_B200_H
#define PGEMB_B200_H

#include <stdint.h>
#include <stddef.h>
#include <stdbool.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- reference types (embedding.h:17-42) -------------------------------------------------- */

typedef float    coord_t;
typedef float    dist_t;
typedef uint32_t idx_t;
typedef uint64_t label_t;

typedef enum {
	DIST_L2,        /* sqrtf(sum (x-y)^2)          distfunc.c:28-65 (AVX2 variant is the one mirrored) */
	DIST_COSINE,    /* 1 - dot/sqrt(|a|^2 |b|^2)   distfunc.c:133-145 */
	DIST_MANHATTAN  /* sum |x-y|                   distfunc.c:147-155 */
} dist_func_t;

typedef struct
{
	size_t		dim;
	size_t		data_size;
	size_t		offset_data;
	size_t		offset_label;
	size_t		size_data_per_element;
	size_t		elems_per_page;
	size_t		M;
	size_t		maxM;
	size_t		efConstruction;
	size_t		efSearch;
	idx_t		enterpoint_node;
	dist_func_t dist_func;
} HnswMetadata;

/* ---- (1) reference-shaped entry points ----------------------------------------------------- */

/* embedding.h:46 / hnswalg.cpp:256-277.  `meta` must be the first member of a PgembHostIndex
 * (below) -- the same "opaque with known prefix" convention the reference uses for HnswIndex
 * (embedding.c:65-75, :706).  k = meta->efSearch is re-read on every call (embedding.c:334).
 * *results is malloc()ed here and free()d by the caller (embedding.c:327); labels ascending by
 * distance, deleted labels filtered (hnswalg.cpp:245).  Returns false on any failure. */
bool hnsw_search(HnswMetadata* meta, const coord_t *point, size_t* n_results, label_t** results);

/* embedding.h:47 / hnswalg.cpp:279-291.  Precondition as in embedding.c:619-621, :693-695: the node
 * `idx` has already been stored (pgemb_index_append) with zeroed links. */
bool hnsw_bind_point(HnswMetadata* meta, const coord_t *point, idx_t idx);

/* embedding.h:55-56 / distfunc.c:159-174.  One pair, host pointers; evaluated by the CUDA kernel
 * (a 1-pair launch -- use pgemb_dist_batch for throughput).  Returns NaN on CUDA failure. */
dist_t hnsw_dist_func(dist_func_t dist, coord_t const* ax, coord_t const* bx, size_t dim);
void   hnsw_init_dist_func(void);

/* embedding.h:44 / embedding.c:948-953: DELETED_FLAG = bit 48 of the label (HnswLabel.pg.flags). */
bool hnsw_is_deleted(label_t label);

/* ---- (2) bulk / device entry points -------------------------------------------------------- */

typedef int pgemb_status;
enum {
	PGEMB_OK = 0,
	PGEMB_ERR_CUDA = 1,        /* no device / CUDA runtime error */
	PGEMB_ERR_ARG = 2,         /* invalid argument */
	PGEMB_ERR_CAPACITY = 3,    /* index capacity or a kernel limit exceeded */
	PGEMB_ERR_STATE = 4,       /* e.g. "Should be blank" (hnswalg.cpp:171), bad link count (:191) */
	PGEMB_ERR_NOMEM = 5
};

typedef struct pgemb_index pgemb_index; /* opaque device index (HBM mirror of the graph) */

/* Host handle with the reference's prefix convention. */
typedef struct
{
	HnswMetadata meta;   /* MUST be first */
	pgemb_index *dev;
} PgembHostIndex;

const char *pgemb_last_error(void);
const char *pgemb_version(void);
/* Number of usable CUDA devices (0 if none); never throws. */
int pgemb_device_count(void);

/* Fill the derived layout fields of *meta from the reloptions exactly as hnsw_get_index does
 * (embedding.c:222-235) with BLCKSZ=8192 page geometry. Returns PGEMB_ERR_ARG if a record cannot
 * fit a page (embedding.c:229-231). */
pgemb_status pgemb_meta_init(HnswMetadata *meta, size_t dims, size_t m, size_t efConstruction,
                             size_t efSearch, dist_func_t dist);

/* Create an empty device index for up to `capacity` nodes on CUDA device `device`.
 * HBM layout (DESIGN.md section 3): vectors[capacity][row_stride] f32 (16-B aligned rows),
 * links[capacity][maxM+1] u32, labels[capacity] u64, norms[capacity] f32 (cosine only). */
pgemb_status pgemb_index_create(const HnswMetadata *meta, size_t capacity, int device, pgemb_index **out);
void         pgemb_index_destroy(pgemb_index *idx);
size_t       pgemb_index_size(const pgemb_index *idx);
size_t       pgemb_index_capacity(const pgemb_index *idx);
int          pgemb_index_device(const pgemb_index *idx);

/* Append n nodes (host pointers).  coords: n*dim f32; labels: n u64 or NULL (label = id);
 * links: n*(maxM+1) u32 in the reference order [count, ids...] or NULL (zeroed = "stored, not
 * bound", embedding.c:619).  Node ids are dense, in append order (embedding.c:693). */
pgemb_status pgemb_index_append(pgemb_index *idx, size_t n, const coord_t *coords,
                                const label_t *labels, const idx_t *links);
/* Same with device pointers (already resident data, e.g. generated on the GPU). */
pgemb_status pgemb_index_append_device(pgemb_index *idx, size_t n, const coord_t *d_coords,
                                       const label_t *d_labels, const idx_t *d_links, void *stream);
/* Ingest n records in the reference's on-page AoS layout
 * [u32 count | u32 links[maxM] | f32 coords[dim] | u64 label] (embedding.c:224-228, :619-621),
 * `record_stride` bytes apart (>= meta.size_data_per_element). */
pgemb_status pgemb_index_append_records(pgemb_index *idx, size_t n, const void *records, size_t record_stride);
/* Export records [first, first+n) in the same AoS layout (write-back of GPU-modified link lists). */
pgemb_status pgemb_index_export_records(const pgemb_index *idx, size_t first, size_t n, void *records, size_t record_stride);
pgemb_status pgemb_index_get_links(const pgemb_index *idx, size_t first, size_t n, idx_t *links_out);
pgemb_status pgemb_index_set_links(pgemb_index *idx, size_t first, size_t n, const idx_t *links);
pgemb_status pgemb_index_get_labels(const pgemb_index *idx, size_t first, size_t n, label_t *labels_out);
pgemb_status pgemb_index_set_labels(pgemb_index *idx, size_t first, size_t n, const label_t *labels);
/* Drop all nodes (TRUNCATE; test/sql/gh-3.sql). */
pgemb_status pgemb_index_truncate(pgemb_index *idx);
/* Grow the index to hold at least `capacity` nodes (a relation grows page by page, embedding.c:636-691); contents and node ids
 * are preserved, a smaller or equal capacity is a no-op.  On failure the index is unchanged. */
pgemb_status pgemb_index_reserve(pgemb_index *idx, size_t capacity);

/* Batched k-NN search: nq independent hnsw_search calls (hnswalg.cpp:234-277 semantics per query).
 * ef plays the role of meta->efSearch (k == ef, hnswalg.cpp:260,:237).
 * Outputs (host pointers; any may be NULL except n_out):
 *   labels_out[nq*ef]  labels ascending by distance, deleted filtered; unused tail = ~0
 *   dists_out [nq*ef]  the matching distances (extension: the reference returns none)
 *   ids_out   [nq*ef]  the matching internal node ids (extension, for parity checks)
 *   n_out     [nq]     number of results per query (<= ef)
 *   stats_out [nq*4]   per query {distance evals, node expansions, link words read, 0}
 *                      -- the counters SURVEY.md section 8(d) derives algorithmic bytes from. */
pgemb_status pgemb_search_batch(pgemb_index *idx, size_t nq, const coord_t *queries, size_t ef,
                                label_t *labels_out, dist_t *dists_out, idx_t *ids_out,
                                int32_t *n_out, uint32_t *stats_out);
/* Same with everything device-resident and launched on `stream` (cudaStream_t, NULL = default);
 * asynchronous: returns after the launch. */
pgemb_status pgemb_search_batch_device(pgemb_index *idx, size_t nq, const coord_t *d_queries, size_t ef,
                                       label_t *d_labels_out, dist_t *d_dists_out, idx_t *d_ids_out,
                                       int32_t *d_n_out, uint32_t *d_stats_out, void *stream);
/* pgemb_search_batch_device (and every other *_device entry) only LAUNCHES: it does not read the traversal's sticky error flag
 * (1 = link id / count out of range, 2 = tie-overflow buffer exceeded, 4 = a streamed batch never arrived).  Poll it with this
 * call: it synchronises `stream`, returns PGEMB_ERR_STATE with the message if the flag was raised, and clears it.
 * One search may be in flight per index at a time (the per-slot visited sets, the work counter and the flag are the index's):
 * concurrent searches on two streams need two pgemb_index handles (replicas). */
pgemb_status pgemb_index_poll_error(pgemb_index *idx, void *stream);
/* Device time (ms) of the search kernel inside the last pgemb_search_batch* call on this index,
 * measured with CUDA events on the launching stream; <0 if unavailable. */
float pgemb_last_kernel_ms(const pgemb_index *idx);
/* Kernels launched by this library since load (the bench's gpu_launches claim). */
uint64_t pgemb_launch_count(void);

/* Batched distances with the reference's exact arithmetic (distfunc.c), host pointers:
 * out[i] = dist(a[i] or a[0] if broadcast_a, b[i]). */
pgemb_status pgemb_dist_batch(dist_func_t dist, size_t dim, size_t n, const coord_t *a, int broadcast_a,
                              const coord_t *b, dist_t *out);
/* Distances from nq host queries to stored nodes ids[nq*k] of a device index (gather kernel K1).
 * out[q*k + j] is NaN where ids[q*k + j] >= the index's size (no error is raised); the other entries are unaffected. */
pgemb_status pgemb_dist_gather(pgemb_index *idx, size_t nq, const coord_t *queries, size_t k,
                               const idx_t *ids, dist_t *out);

/* Exact (brute-force) k-NN over all stored nodes: what `SELECT ... ORDER BY val <op> q LIMIT k` computes WITHOUT the index
 * (one hnsw_dist_func per row, embedding.c:1022-1062, then the executor's sort; test/expected/knn.out:63-91), batched.
 * Distances bit-identical to the reference's; results ascending by (dist,label); labels with DELETED_FLAG skipped.
 * labels_out[nq*k] (unused tail ~0), dists_out[nq*k] optional, n_out[nq]. Host pointers. */
pgemb_status pgemb_scan_topk(pgemb_index *idx, size_t nq, const coord_t *queries, size_t k, label_t *labels_out,
                             dist_t *dists_out, int32_t *n_out);
/* How pgemb_scan_topk gets there (DESIGN.md section 6, K6): for L2 and cosine the table is first FILTERED by one dense
 * contraction on the tensor cores (wgmma tf32, TMA tensor maps, register accumulators; csrc/scan_umma_kernel.cuh) --
 * a row is dropped only if a rigorous lower bound of its distance exceeds the query's current k-th best exact distance --
 * and the survivors are re-scored with the reference-exact arithmetic, so labels, order and distance bits are those of
 * the exact kernels.  Manhattan (no bilinear form) and small tables use the exact tiled kernel throughout.
 * PGEMB_SCAN_TC=0 disables the filter, =2 forces it.  Counters since load:
 *   out[0] scans through the tensor-core filter   out[1] (query,row) pairs it covered   out[2] candidates re-scored exactly
 *   out[3] scans repeated on the exact kernels because the error-bound tripwire fired
 *   out[4] queries whose candidate list overflowed (re-scored against the whole chunk)   out[5] exact-kernel scans */
void pgemb_scan_counters(uint64_t out[6]);
/* pgemb_scan_topk with DEVICE pointers in and out (queries [nq*dim], labels [nq*k], dists [nq*k] optional, n [nq]); `stream` is
 * synchronised with on entry, the scan has finished when the call returns.  Same results, byte for byte. */
pgemb_status pgemb_scan_topk_device(pgemb_index *idx, size_t nq, const coord_t *d_queries, size_t k, label_t *d_labels_out,
                                    dist_t *d_dists_out, int32_t *d_n_out, void *stream);
/* Test entry: the raw tensor-core products S[q][j] = q . row(r0 + j) (TF32 operands, fp32 accumulate) of the K6 kernel,
 * out[nq * nr], host pointers -- lets a test check descriptors / swizzle / accumulator layout against a float64 product. */
pgemb_status pgemb_debug_umma_product(pgemb_index *idx, size_t nq, const coord_t *queries, size_t r0, size_t nr, float *out);

/* ---- index-scan iteration: the reference's beginscan / gettuple / endscan trio -- embedding.c:249-387; SURVEY.md 8(f2) ----
 * One handle = one scan (`so`): the query, the per-scan efSearch that hnsw_gettuple doubles in place (embedding.c:334) and the
 * TIDs handed out so far.  pgemb_index_scan_next is hnsw_gettuple: the first call searches with efSearch; when the results
 * run out and the last search was full (n == efSearch) it doubles efSearch, searches again and continues with the TIDs not
 * returned before (qsort + bsearch de-duplication exactly as embedding.c:354-363, quirks included -- csrc/capi.cu); it ends
 * when a search returns fewer than efSearch results and they are used up, or finds nothing new (:338).
 *   returns 1: *tid_out = next heap TID (the label's low 48 bits; flags dropped as by the reference's 6-byte memcpy)
 *           0: no more tuples
 *         < 0: -(pgemb_status): "HNSW index search failed" (embedding.c:318, :336)
 * pgemb_index_scan_next_batch hands out up to `max` tuples of the same sequence in one call. */
typedef struct pgemb_index_scan pgemb_index_scan;
pgemb_status pgemb_index_scan_begin(pgemb_index *idx, const coord_t *query, size_t efSearch, pgemb_index_scan **out);
int          pgemb_index_scan_next(pgemb_index_scan *scan, label_t *tid_out);
pgemb_status pgemb_index_scan_next_batch(pgemb_index_scan *scan, size_t max, label_t *tids_out, size_t *n_out);
size_t       pgemb_index_scan_ef(const pgemb_index_scan *scan);        /* current (doubled) efSearch */
uint64_t     pgemb_index_scan_searches(const pgemb_index_scan *scan);  /* hnsw_search calls made so far */
void         pgemb_index_scan_end(pgemb_index_scan *scan);

/* hnsw_bind_point against the device mirror (hnswalg.cpp:225-232): node `id` must be stored and
 * unbound.  Sequential semantics: one call at a time per index. */
pgemb_status pgemb_bind_point(pgemb_index *idx, idx_t id);
/* Convenience: append + bind for n points in id order == n sequential hnsw_add_point calls
 * (embedding.c:606-701).  All n binds run on the device without host round trips. */
pgemb_status pgemb_insert_batch(pgemb_index *idx, size_t n, const coord_t *coords, const label_t *labels);

/* Bulk build (the GPU counterpart of ambuild's row-by-row hnsw_add_point loop, embedding.c:504-548):
 * bind nodes [first, first+n) -- already appended, unbound -- in id order, in BATCHES: every node of a
 * batch runs bindPoint's search (hnswalg.cpp:229) against the graph as it was when the batch started;
 * own lists are then written and back-links (hnswalg.cpp:182-222) applied per target in source-id order.
 * Batch size grows with the graph (<= 1/32 of the bound nodes, capped by batch_max), starting with exact
 * one-by-one binds, so a batch of 1 is exactly one reference insert.  The result is a valid graph in the
 * reference's format built with the reference's heuristics, but NOT bit-identical to a sequential
 * build when batch_max > 1 (nodes of one batch do not see each other) -- see DESIGN.md section 8.
 * seconds_out (optional) receives the wall time including the final synchronisation. */
pgemb_status pgemb_build_bulk(pgemb_index *idx, size_t first, size_t n, size_t batch_max, double *seconds_out);

/* Exact AND parallel build: same preconditions as pgemb_build_bulk, but the result is bit-identical to n
 * sequential hnsw_add_point calls (embedding.c:606-701).  Speculative batches of searches against the graph as of
 * the batch start; the longest prefix whose searches provably equal the sequential ones (no expanded node's link
 * list is modified by an earlier insert of the batch) is connected, the rest is retried.  batch_max <= 4096.
 * stats_out (optional, 3 x u64): batches, searches run, inserts. */
pgemb_status pgemb_build_exact(pgemb_index *idx, size_t first, size_t n, size_t batch_max, double *seconds_out, uint64_t *stats_out);

/* Shard top-k merge (SURVEY.md section 8(e)): for each of nq queries merge n_shards lists of
 * (dist,label) ascending lists of length k (n valid per list in n_in) into the k best by
 * (dist,label) lexicographic order (hnswalg.cpp:236-247 pair order). Device pointers. */
pgemb_status pgemb_merge_topk_device(size_t nq, size_t n_shards, size_t k,
                                     const dist_t *d_dists_in, const label_t *d_labels_in, const int32_t *d_n_in,
                                     dist_t *d_dists_out, label_t *d_labels_out, int32_t *d_n_out, void *stream);

/* The same merge over ONE packed buffer per shard -- [labels u64 nq*k | dists f32 nq*k | counts i32 nq], pgemb_packed_topk_bytes
 * -- i.e. over what a single all-gather of the per-shard results delivers (shard s at d_packed + s * shard_stride_bytes). */
size_t       pgemb_packed_topk_bytes(size_t nq, size_t k);
pgemb_status pgemb_merge_topk_packed_device(size_t nq, size_t n_shards, size_t k, const void *d_packed, size_t shard_stride_bytes,
                                            dist_t *d_dists_out, label_t *d_labels_out, int32_t *d_n_out, void *stream);

/* ---- sharded search without a collective: peers read each other's results over NVLink (DESIGN.md section 7) -------------
 * One pgemb_exchange per rank (= per GPU / shard).  Set-up, once: create; hand the 64-byte handle (other processes) or
 * the buffer pointer (ranks of the same process) of every rank to every rank; attach.  Per step, on every rank with the SAME
 * nq and queries:   pgemb_sharded_search_device  (local traversal -> this rank's result area, then its sequence number is
 * stored into every peer's flag array by 4-byte copies in stream order)   and   pgemb_sharded_merge_device  (ONE kernel that
 * waits for all peers' flags, reads their lists directly from peer memory and merges by (dist,label), hnswalg.cpp:236-247).
 * No NCCL call, no host synchronisation between the two.  ef must equal the k the exchange was created with. */
#define PGEMB_IPC_HANDLE_BYTES 64
typedef struct pgemb_exchange pgemb_exchange;
pgemb_status pgemb_exchange_create(int device, int rank, int world, size_t max_nq, size_t k, pgemb_exchange **out);
void         pgemb_exchange_destroy(pgemb_exchange *ex);
pgemb_status pgemb_exchange_handle(pgemb_exchange *ex, void *handle_out /* PGEMB_IPC_HANDLE_BYTES */);
void        *pgemb_exchange_buffer(pgemb_exchange *ex);
/* handles: world x PGEMB_IPC_HANDLE_BYTES (this rank's own slot is ignored); same_process != 0: each slot starts with the raw
 * device pointer from pgemb_exchange_buffer instead of an IPC handle. */
pgemb_status pgemb_exchange_attach(pgemb_exchange *ex, const void *handles, int same_process);
pgemb_status pgemb_sharded_search_device(pgemb_index *idx, pgemb_exchange *ex, size_t nq, const coord_t *d_queries, size_t ef, void *stream);
/* the brute-force scan (pgemb_scan_topk_device) as the local step instead of the traversal: BASELINE configs[4], every rank scans
 * its id range for the whole query batch; k must equal the exchange's k */
pgemb_status pgemb_sharded_scan_device(pgemb_index *idx, pgemb_exchange *ex, size_t nq, const coord_t *d_queries, size_t k, void *stream);
pgemb_status pgemb_sharded_merge_device(pgemb_exchange *ex, size_t nq, label_t *d_labels_out, dist_t *d_dists_out, int32_t *d_n_out, void *stream);
float        pgemb_exchange_last_merge_ms(pgemb_exchange *ex);
int          pgemb_exchange_error(pgemb_exchange *ex);

#ifdef __cplusplus
}
#endif
#endif /* PGEMB_B200_H */
