// capi.cu -- host side of the C ABI declared in include/pgemb_b200.h.
//
// Mirrors the reference's host-facing contract for the hot path (embedding.h:44-56): hnsw_search,
// hnsw_bind_point, hnsw_dist_func, hnsw_init_dist_func keep their names, argument meaning, ownership
// (malloc'd results freed by the caller, embedding.c:327) and error behaviour (bool false, no C++
// exception crosses -- hnswalg.cpp:258-276), and adds the bulk/device entry points a GPU needs.
// There is no CPU implementation of any of it in this library: without a usable CUDA device every
// entry point fails with PGEMB_ERR_CUDA.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "aux_kernels.cuh"
#include "bind_kernel.cuh"
#include "common.cuh"
#include "scan_tile_kernel.cuh"
#include "scan_umma_kernel.cuh"
#include "search_kernel.cuh"

using namespace pgemb;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static std::atomic<uint64_t>	g_launches{0};

static pgemb_status fail(pgemb_status st, const std::string &msg)
{
	g_last_error = msg;
	return st;
}

#define CU_TRY(expr)                                                                                             \
	do {                                                                                                         \
		cudaError_t _e = (expr);                                                                                 \
		if (_e != cudaSuccess)                                                                                   \
			return fail(PGEMB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                     \
	} while (0)

// Runs f(std::integral_constant<int, M_...>{}) for the runtime metric and returns its status: a kernel launched inside takes
// decltype(m)::value.  with_tc_metric covers only the metrics that have a tensor-core path, so that no M_MAN instance of
// those kernels is compiled.
template <typename F> static pgemb_status with_metric(int metric, F &&f)
{
	if (metric == DIST_L2) return f(std::integral_constant<int, M_L2>{});
	if (metric == DIST_COSINE) return f(std::integral_constant<int, M_COS>{});
	if (metric == DIST_MANHATTAN) return f(std::integral_constant<int, M_MAN>{});
	return fail(PGEMB_ERR_ARG, "unknown distance function");
}

template <typename F> static pgemb_status with_tc_metric(int metric, F &&f)
{
	if (metric == DIST_L2) return f(std::integral_constant<int, M_L2>{});
	if (metric == DIST_COSINE) return f(std::integral_constant<int, M_COS>{});
	return fail(PGEMB_ERR_ARG, "no tensor-core path for this metric");
}

extern "C" const char *pgemb_last_error(void) { return g_last_error.c_str(); }
extern "C" const char *pgemb_version(void) { return "pg_embedding_b200 0.2 (sm_90a)"; }
extern "C" uint64_t	   pgemb_launch_count(void) { return g_launches.load(); }

extern "C" int pgemb_device_count(void)
{
	int			n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess)
	{
		cudaGetLastError();
		return 0;
	}
	return n;
}

// ------------------------------------------------------------------------------------------------
// metadata (embedding.c:222-235)
// ------------------------------------------------------------------------------------------------
extern "C" pgemb_status pgemb_meta_init(HnswMetadata *meta, size_t dims, size_t m, size_t efConstruction, size_t efSearch,
										dist_func_t dist)
{
	if (!meta || dims == 0) return fail(PGEMB_ERR_ARG, "HNSW index requires 'dims' to be specified");  // embedding.c:219-221
	if (efConstruction < 1 || efSearch < 1) return fail(PGEMB_ERR_ARG, "efconstruction/efsearch must be >= 1");
	if ((int) dist < 0 || (int) dist > 2) return fail(PGEMB_ERR_ARG, "unknown distance function");
	memset(meta, 0, sizeof(*meta));
	meta->dim = dims;
	meta->M = m;
	meta->maxM = m * 2;
	meta->data_size = dims * sizeof(coord_t);
	meta->offset_data = (meta->maxM + 1) * sizeof(idx_t);
	meta->offset_label = meta->offset_data + meta->data_size;
	meta->size_data_per_element = meta->offset_label + sizeof(label_t);
	// BLCKSZ 8192, MAXALIGN(SizeOfPageHeaderData) 24, sizeof(HnswPageOpaque) 4, sizeof(ItemIdData) 4
	meta->elems_per_page = (8192 - 24 - 4) / (meta->size_data_per_element + 4);
	meta->efConstruction = efConstruction;
	meta->efSearch = efSearch;
	meta->dist_func = dist;
	meta->enterpoint_node = 0;
	if (meta->elems_per_page == 0) return fail(PGEMB_ERR_ARG, "Element doesn't fit in Postgres page");  // embedding.c:229-231
	return PGEMB_OK;
}

extern "C" bool hnsw_is_deleted(label_t label) { return ((label >> 48) & 1u) != 0; }

// ------------------------------------------------------------------------------------------------
// the device index
// ------------------------------------------------------------------------------------------------

struct pgemb_index
{
	HnswMetadata meta;
	int			 device = 0;
	int			 sm_count = 0;
	size_t		 capacity = 0, n = 0;
	uint32_t	 row_f = 0, link_stride = 0;
	float		*d_vectors = nullptr;
	uint32_t	*d_links = nullptr;
	uint64_t	*d_labels = nullptr;
	float		*d_norms = nullptr;
	cudaStream_t stream = nullptr;
	cudaEvent_t	 ev0 = nullptr, ev1 = nullptr;
	static constexpr int kMaxChunks = 16;
	cudaStream_t s_in = nullptr;  // copy stream of the host-pointer batch API
	cudaEvent_t	 ev_in = nullptr;  // the traversal's stream waits on it for the queries (or the first `avail`) to land
	unsigned int *h_avail = nullptr;  // pinned: values the copy stream publishes to the running kernel
	bool		 ev_valid = false;
	// search workspace
	uint32_t	  ws_slots = 0, ws_ef = 0, vis_words = 0, vlog_cap = 0;
	uint32_t	 *d_visited = nullptr, *d_vlog = nullptr, *d_vhash = nullptr;
	uint32_t	  ws_vh = 0;  // allocated hash entries per slot
	size_t		  l2_persist_max = 0, l2_window_max = 0;
	bool		  l2_limit_dropped = false;	 // the scan path gave the persisting-L2 set-aside back (scan_filter_pass)
	// link lists that came from the caller have not been checked for repeated ids yet / result of the last check
	bool links_checked = true, links_distinct = true;
	uint64_t	 *d_ovf = nullptr;
	uint32_t	 *d_seq_ids = nullptr;	 // ids of a run of sequential binds (pgemb_insert_batch)
	size_t		  seq_ids_cap = 0;
	uint64_t	 *d_resg = nullptr;	 // result buffers of the huge-ef traversal variant ([slots][2 * ef])
	size_t		  resg_keys = 0;
	unsigned int *d_counter = nullptr;
	int			 *d_error = nullptr;
	// staging for the host-pointer API
	void  *d_stage = nullptr;
	size_t stage_bytes = 0;
	// pinned landing area of the small-batch host path: results + error flag arrive by truly asynchronous copies, one synchronisation
	char  *h_land = nullptr;
	size_t land_bytes = 0;
	// bind workspace
	BindWorkspace bind_ws;
	size_t norms_n = 0;	 // rows [0, norms_n) have their squared norm in d_norms (cosine: all; L2: filled lazily by the tensor-core scan)
	// what the last traversal launch configured, so that an identical launch skips the attribute / occupancy / L2-window driver calls
	const void *last_fn = nullptr;
	uint32_t	last_smem = 0;
	const void *last_l2_base = nullptr;
	size_t		last_l2_bytes = 0;
	cudaStream_t last_l2_stream = nullptr;
};

static pgemb_status set_device(const pgemb_index *idx)
{
	CU_TRY(cudaSetDevice(idx->device));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_create(const HnswMetadata *meta, size_t capacity, int device, pgemb_index **out)
{
	if (!meta || !out) return fail(PGEMB_ERR_ARG, "null argument");
	if (meta->dim == 0 || meta->dim > 65535) return fail(PGEMB_ERR_ARG, "dims out of range (1..65535; stored as uint16 on pages, embedding.c:494)");
	if (meta->maxM != meta->M * 2) return fail(PGEMB_ERR_ARG, "maxM must be 2*M (embedding.c:224)");
	if (meta->maxM > 4096) return fail(PGEMB_ERR_ARG, "maxM > 4096 unsupported");
	if ((int) meta->dist_func < 0 || (int) meta->dist_func > 2) return fail(PGEMB_ERR_ARG, "unknown distance function");
	if (capacity == 0 || capacity >= (1ull << 31)) return fail(PGEMB_ERR_ARG, "capacity must be in [1, 2^31)");
	int ndev = 0;
	CU_TRY(cudaGetDeviceCount(&ndev));
	if (device < 0 || device >= ndev) return fail(PGEMB_ERR_CUDA, "no such CUDA device");
	CU_TRY(cudaSetDevice(device));
	pgemb_index *idx = new (std::nothrow) pgemb_index();
	if (!idx) return fail(PGEMB_ERR_NOMEM, "out of host memory");
	idx->meta = *meta;
	idx->device = device;
	idx->capacity = capacity;
	idx->row_f = (uint32_t) ((meta->dim + 3) & ~(size_t) 3);
	idx->link_stride = (uint32_t) ((meta->maxM + 1 + 3) & ~(size_t) 3);
	cudaError_t e;
	// from here on a failure must not leak the half-built index
#define CU_TRY_IDX(expr)                                                                                  \
	if ((e = (expr)) != cudaSuccess)                                                                      \
	{                                                                                                     \
		pgemb_index_destroy(idx);                                                                         \
		return fail(PGEMB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e));                   \
	}
#define ALLOC(ptr, bytes)                                                                                 \
	if ((e = cudaMalloc((void **) &(ptr), (bytes))) != cudaSuccess)                                       \
	{                                                                                                     \
		pgemb_index_destroy(idx);                                                                         \
		return fail(PGEMB_ERR_NOMEM, std::string("cudaMalloc " #ptr ": ") + cudaGetErrorString(e));       \
	}
	cudaDeviceProp prop;
	CU_TRY_IDX(cudaGetDeviceProperties(&prop, device));
	idx->sm_count = prop.multiProcessorCount;
	idx->l2_persist_max = (size_t) prop.persistingL2CacheMaxSize;
	idx->l2_window_max = (size_t) prop.accessPolicyMaxWindowSize;
	ALLOC(idx->d_vectors, capacity * idx->row_f * sizeof(float));
	ALLOC(idx->d_links, capacity * idx->link_stride * sizeof(uint32_t));
	ALLOC(idx->d_labels, capacity * sizeof(uint64_t));
	ALLOC(idx->d_norms, capacity * sizeof(float));
	ALLOC(idx->d_counter, sizeof(unsigned int) * 4);
	ALLOC(idx->d_error, sizeof(int));
	CU_TRY_IDX(cudaMemset(idx->d_error, 0, sizeof(int)));
	CU_TRY_IDX(cudaStreamCreateWithFlags(&idx->stream, cudaStreamNonBlocking));
	CU_TRY_IDX(cudaEventCreate(&idx->ev0));
	CU_TRY_IDX(cudaEventCreate(&idx->ev1));
#undef ALLOC
#undef CU_TRY_IDX
	*out = idx;
	return PGEMB_OK;
}

extern "C" void pgemb_index_destroy(pgemb_index *idx)
{
	if (!idx) return;
	cudaSetDevice(idx->device);
	cudaDeviceSynchronize();
	cudaFree(idx->d_vectors);
	cudaFree(idx->d_links);
	cudaFree(idx->d_labels);
	cudaFree(idx->d_norms);
	cudaFree(idx->d_visited);
	cudaFree(idx->d_vlog);
	cudaFree(idx->d_vhash);
	cudaFree(idx->d_ovf);
	cudaFree(idx->d_resg);
	cudaFree(idx->d_seq_ids);
	cudaFree(idx->d_counter);
	cudaFree(idx->d_error);
	cudaFree(idx->d_stage);
	if (idx->h_land) cudaFreeHost(idx->h_land);
	bind_ws_free(idx->bind_ws);
	if (idx->stream) cudaStreamDestroy(idx->stream);
	if (idx->s_in) cudaStreamDestroy(idx->s_in);
	if (idx->h_avail) cudaFreeHost(idx->h_avail);
	if (idx->ev_in) cudaEventDestroy(idx->ev_in);
	if (idx->ev0) cudaEventDestroy(idx->ev0);
	if (idx->ev1) cudaEventDestroy(idx->ev1);
	delete idx;
}

extern "C" size_t pgemb_index_size(const pgemb_index *idx) { return idx ? idx->n : 0; }
extern "C" size_t pgemb_index_capacity(const pgemb_index *idx) { return idx ? idx->capacity : 0; }
extern "C" int	  pgemb_index_device(const pgemb_index *idx) { return idx ? idx->device : -1; }

static pgemb_status ensure_stage(pgemb_index *idx, size_t bytes)
{
	if (idx->stage_bytes >= bytes) return PGEMB_OK;
	if (idx->d_stage) cudaFree(idx->d_stage);
	idx->d_stage = nullptr;
	idx->stage_bytes = 0;
	size_t want = bytes + bytes / 4 + 4096;
	CU_TRY(cudaMalloc(&idx->d_stage, want));
	idx->stage_bytes = want;
	return PGEMB_OK;
}

// Arrays carved out of one staging buffer, back to back in the order listed, each starting 256-byte aligned.  `bytes` is
// what the buffer must hold; place() points every array at its part of the buffer.
struct StageLayout
{
	struct Part
	{
		template <typename T> Part(T *&p, size_t n) : ptr((void **) &p), size(n) {}
		void **ptr;
		size_t size;
	};
	static size_t up(size_t x) { return (x + 255) & ~(size_t) 255; }
	std::vector<Part> parts;
	size_t			  bytes = 0;
	StageLayout(std::initializer_list<Part> l) : parts(l) { for (const Part &p : parts) bytes += up(p.size); }
	void place(void *base) const
	{
		char *b = (char *) base;
		for (const Part &p : parts)
		{
			*p.ptr = b;
			b += up(p.size);
		}
	}
};

static pgemb_status compute_norms(pgemb_index *idx, size_t first, size_t n, cudaStream_t s)
{
	if (idx->meta.dist_func != DIST_COSINE || n == 0) return PGEMB_OK;
	const uint32_t threads = 128;
	const uint32_t blocks = (uint32_t) ((n * 4 + threads - 1) / threads);
	PGEMB_LAUNCH(norms_kernel, blocks, threads, 0, s, idx->d_vectors, idx->row_f, (uint32_t) idx->meta.dim, (uint32_t) first, (uint32_t) n,
											idx->d_norms);
	g_launches++;
	CU_TRY(cudaGetLastError());
	idx->norms_n = first + n;
	return PGEMB_OK;
}

static pgemb_status append_common(pgemb_index *idx, size_t n, const coord_t *coords, const label_t *labels, const idx_t *links,
								  cudaMemcpyKind kind, cudaStream_t s)
{
	if (!idx || (!coords && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (idx->n + n > idx->capacity) return fail(PGEMB_ERR_CAPACITY, "index capacity exceeded");
	if (n == 0) return PGEMB_OK;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t first = idx->n;
	const size_t dim = idx->meta.dim, maxM1 = idx->meta.maxM + 1;
	// rows: zero the padding, then a pitched copy dim -> row_f
	if (idx->row_f != dim) CU_TRY(cudaMemsetAsync(idx->d_vectors + first * idx->row_f, 0, n * idx->row_f * sizeof(float), s));
	CU_TRY(cudaMemcpy2DAsync(idx->d_vectors + first * idx->row_f, idx->row_f * sizeof(float), coords, dim * sizeof(float),
							 dim * sizeof(float), n, kind, s));
	CU_TRY(cudaMemsetAsync(idx->d_links + first * idx->link_stride, 0, n * idx->link_stride * sizeof(uint32_t), s));
	if (links)
	{
		CU_TRY(cudaMemcpy2DAsync(idx->d_links + first * idx->link_stride, idx->link_stride * sizeof(uint32_t), links,
								 maxM1 * sizeof(uint32_t), maxM1 * sizeof(uint32_t), n, kind, s));
		idx->links_checked = false;
	}
	if (labels)
		CU_TRY(cudaMemcpyAsync(idx->d_labels + first, labels, n * sizeof(uint64_t), kind, s));
	else
	{
		std::vector<uint64_t> tmp;
		try
		{
			tmp.resize(n);
		}
		catch (const std::bad_alloc &)
		{
			return fail(PGEMB_ERR_NOMEM, "out of host memory");
		}
		for (size_t i = 0; i < n; i++) tmp[i] = first + i;
		CU_TRY(cudaMemcpyAsync(idx->d_labels + first, tmp.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
		CU_TRY(cudaStreamSynchronize(s));
	}
	st = compute_norms(idx, first, n, s);
	if (st) return st;
	idx->n += n;
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_append(pgemb_index *idx, size_t n, const coord_t *coords, const label_t *labels,
										   const idx_t *links)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	pgemb_status st = append_common(idx, n, coords, labels, links, cudaMemcpyHostToDevice, idx->stream);
	if (st) return st;
	CU_TRY(cudaStreamSynchronize(idx->stream));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_append_device(pgemb_index *idx, size_t n, const coord_t *d_coords, const label_t *d_labels,
												  const idx_t *d_links, void *stream)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	return append_common(idx, n, d_coords, d_labels, d_links, cudaMemcpyDeviceToDevice, (cudaStream_t) stream);
}

extern "C" pgemb_status pgemb_index_append_records(pgemb_index *idx, size_t n, const void *records, size_t record_stride)
{
	if (!idx || (!records && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (record_stride < idx->meta.size_data_per_element || (record_stride & 3)) return fail(PGEMB_ERR_ARG, "bad record stride");
	if (idx->n + n > idx->capacity) return fail(PGEMB_ERR_CAPACITY, "index capacity exceeded");
	if (n == 0) return PGEMB_OK;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t chunk = 1u << 16;
	for (size_t done = 0; done < n; done += chunk)
	{
		const size_t m = (n - done < chunk) ? (n - done) : chunk;
		st = ensure_stage(idx, m * record_stride);
		if (st) return st;
		CU_TRY(cudaMemcpyAsync(idx->d_stage, (const char *) records + done * record_stride, m * record_stride, cudaMemcpyHostToDevice,
							   idx->stream));
		const uint32_t threads = 128, blocks = (uint32_t) ((m * 32 + threads - 1) / threads);
		PGEMB_LAUNCH(records_unpack_kernel, blocks, threads, 0, idx->stream, (const unsigned char *) idx->d_stage, record_stride, (uint32_t) m,
																   (uint32_t) (idx->n + done), (uint32_t) idx->meta.dim,
																   (uint32_t) idx->meta.maxM, idx->row_f, idx->link_stride,
																   idx->d_vectors, idx->d_links, idx->d_labels);
		g_launches++;
		CU_TRY(cudaGetLastError());
		CU_TRY(cudaStreamSynchronize(idx->stream));
	}
	st = compute_norms(idx, idx->n, n, idx->stream);
	if (st) return st;
	CU_TRY(cudaStreamSynchronize(idx->stream));
	idx->n += n;
	idx->links_checked = false;
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_export_records(const pgemb_index *cidx, size_t first, size_t n, void *records, size_t record_stride)
{
	pgemb_index *idx = const_cast<pgemb_index *>(cidx);
	if (!idx || (!records && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (record_stride < idx->meta.size_data_per_element || (record_stride & 3)) return fail(PGEMB_ERR_ARG, "bad record stride");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (n == 0) return PGEMB_OK;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t chunk = 1u << 16;
	for (size_t done = 0; done < n; done += chunk)
	{
		const size_t m = (n - done < chunk) ? (n - done) : chunk;
		st = ensure_stage(idx, m * record_stride);
		if (st) return st;
		CU_TRY(cudaMemsetAsync(idx->d_stage, 0, m * record_stride, idx->stream));
		const uint32_t threads = 128, blocks = (uint32_t) ((m * 32 + threads - 1) / threads);
		PGEMB_LAUNCH(records_pack_kernel, blocks, threads, 0, idx->stream, (unsigned char *) idx->d_stage, record_stride, (uint32_t) m,
																 (uint32_t) (first + done), (uint32_t) idx->meta.dim,
																 (uint32_t) idx->meta.maxM, idx->row_f, idx->link_stride, idx->d_vectors,
																 idx->d_links, idx->d_labels);
		g_launches++;
		CU_TRY(cudaGetLastError());
		CU_TRY(cudaMemcpyAsync((char *) records + done * record_stride, idx->d_stage, m * record_stride, cudaMemcpyDeviceToHost,
							   idx->stream));
		CU_TRY(cudaStreamSynchronize(idx->stream));
	}
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_get_links(const pgemb_index *idx, size_t first, size_t n, idx_t *links_out)
{
	if (!idx || (!links_out && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (n == 0) return PGEMB_OK;
	CU_TRY(cudaSetDevice(idx->device));
	const size_t maxM1 = idx->meta.maxM + 1;
	CU_TRY(cudaMemcpy2DAsync(links_out, maxM1 * sizeof(uint32_t), idx->d_links + first * idx->link_stride,
							 idx->link_stride * sizeof(uint32_t), maxM1 * sizeof(uint32_t), n, cudaMemcpyDeviceToHost, idx->stream));
	CU_TRY(cudaStreamSynchronize(idx->stream));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_set_links(pgemb_index *idx, size_t first, size_t n, const idx_t *links)
{
	if (!idx || (!links && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (n == 0) return PGEMB_OK;
	CU_TRY(cudaSetDevice(idx->device));
	const size_t maxM1 = idx->meta.maxM + 1;
	CU_TRY(cudaMemcpy2DAsync(idx->d_links + first * idx->link_stride, idx->link_stride * sizeof(uint32_t), links,
							 maxM1 * sizeof(uint32_t), maxM1 * sizeof(uint32_t), n, cudaMemcpyHostToDevice, idx->stream));
	CU_TRY(cudaStreamSynchronize(idx->stream));
	idx->links_checked = false;
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_get_labels(const pgemb_index *idx, size_t first, size_t n, label_t *labels_out)
{
	if (!idx || (!labels_out && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (n == 0) return PGEMB_OK;
	CU_TRY(cudaSetDevice(idx->device));
	CU_TRY(cudaMemcpyAsync(labels_out, idx->d_labels + first, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, idx->stream));
	CU_TRY(cudaStreamSynchronize(idx->stream));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_set_labels(pgemb_index *idx, size_t first, size_t n, const label_t *labels)
{
	if (!idx || (!labels && n)) return fail(PGEMB_ERR_ARG, "null argument");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (n == 0) return PGEMB_OK;
	CU_TRY(cudaSetDevice(idx->device));
	CU_TRY(cudaMemcpyAsync(idx->d_labels + first, labels, n * sizeof(uint64_t), cudaMemcpyHostToDevice, idx->stream));
	CU_TRY(cudaStreamSynchronize(idx->stream));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_reserve(pgemb_index *idx, size_t capacity)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	if (capacity <= idx->capacity) return PGEMB_OK;
	if (capacity >= (1ull << 31)) return fail(PGEMB_ERR_ARG, "capacity must be in [1, 2^31)");
	pgemb_status st = set_device(idx);
	if (st) return st;
	float	 *nv = nullptr, *nn = nullptr;
	uint32_t *nl = nullptr;
	uint64_t *nb = nullptr;
	cudaError_t e = cudaMalloc((void **) &nv, capacity * idx->row_f * sizeof(float));
	if (e == cudaSuccess) e = cudaMalloc((void **) &nl, capacity * idx->link_stride * sizeof(uint32_t));
	if (e == cudaSuccess) e = cudaMalloc((void **) &nb, capacity * sizeof(uint64_t));
	if (e == cudaSuccess) e = cudaMalloc((void **) &nn, capacity * sizeof(float));
	cudaStream_t s = idx->stream;
	const size_t n = idx->n;
	if (e == cudaSuccess && n) e = cudaMemcpyAsync(nv, idx->d_vectors, n * idx->row_f * sizeof(float), cudaMemcpyDeviceToDevice, s);
	if (e == cudaSuccess && n) e = cudaMemcpyAsync(nl, idx->d_links, n * idx->link_stride * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s);
	if (e == cudaSuccess && n) e = cudaMemcpyAsync(nb, idx->d_labels, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s);
	if (e == cudaSuccess && n) e = cudaMemcpyAsync(nn, idx->d_norms, n * sizeof(float), cudaMemcpyDeviceToDevice, s);
	if (e == cudaSuccess) e = cudaStreamSynchronize(s);
	if (e != cudaSuccess)
	{
		cudaFree(nv);
		cudaFree(nl);
		cudaFree(nb);
		cudaFree(nn);
		cudaGetLastError();
		return fail(e == cudaErrorMemoryAllocation ? PGEMB_ERR_NOMEM : PGEMB_ERR_CUDA, std::string("pgemb_index_reserve: ") + cudaGetErrorString(e));
	}
	cudaFree(idx->d_vectors);
	cudaFree(idx->d_links);
	cudaFree(idx->d_labels);
	cudaFree(idx->d_norms);
	idx->d_vectors = nv;
	idx->d_links = nl;
	idx->d_labels = nb;
	idx->d_norms = nn;
	idx->capacity = capacity;  // the per-slot visited bitmaps and the build's stamps are sized by capacity: re-made on next use
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_index_truncate(pgemb_index *idx)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	idx->n = 0;
	idx->norms_n = 0;
	idx->links_checked = idx->links_distinct = true;
	return PGEMB_OK;
}

// ------------------------------------------------------------------------------------------------
// search launch configuration (DESIGN.md section 6)
// ------------------------------------------------------------------------------------------------
static int env_int(const char *name, int dflt)
{
	const char *v = getenv(name);
	return (v && *v) ? atoi(v) : dflt;
}

// shared-memory layout + slots/rings per CTA: search_config.h (shared with the host emulation harness in tests/emu)
static pgemb_status make_config(const pgemb_index *idx, uint32_t ef, SearchConfig *c, bool coop, bool res_global)
{
	SearchShape sh;
	sh.res_global = res_global;
	sh.metric = (int) idx->meta.dist_func;
	sh.dim = (uint32_t) idx->meta.dim;
	sh.row_f = idx->row_f;
	sh.link_stride = idx->link_stride;
	sh.maxM = (uint32_t) idx->meta.maxM;
	sh.ef = ef;
	sh.sm_count = (uint32_t) idx->sm_count;
	// long L2 rows (>= 4 KB, e.g. 1536-d): 8 lanes per row, rings of 4 rows -> twice as many rings per SM (measured on the
	// configs[3] row shape: 0.67 -> 0.80 of the HBM roofline, profiles/README.md round 2); PGEMB_L2_TPR8=0 disables
	sh.tpr = (!res_global && sh.metric == DIST_L2 && env_int("PGEMB_L2_TPR8", 1) != 0 && idx->row_f * 4u >= (uint32_t) env_int("PGEMB_L2_TPR8_MIN_BYTES", 4096)) ? 8u : 4u;
	SearchTuning tu;
	tu.duty = env_int("PGEMB_RING_DUTY_PCT", 50) / 100.0;
	tu.want_warps = env_int("PGEMB_WARPS", 0);
	tu.want_rings = env_int("PGEMB_RINGS", 0);
	tu.want_coop_warps = env_int("PGEMB_COOP_WARPS", 0);
	tu.smem_visited = env_int("PGEMB_SMEM_VISITED", 4096);  // latency mode: entries of the shared-memory visited set (0 = keep it at L2)
	switch (make_search_config(sh, tu, coop, c))
	{
		case 0: return PGEMB_OK;
		case 1: return fail(PGEMB_ERR_CAPACITY, "search working set does not fit shared memory (dims/ef/maxM too large)");
		default: return fail(PGEMB_ERR_CAPACITY, "PGEMB_WARPS/PGEMB_RINGS do not fit shared memory");
	}
}

// Visited-set sizing: an open-addressing table of vh entries per slot (kept at most half full by the
// kernel, which then migrates to the exact bitmap).  A search touches ~20*ef nodes on typical data.
static uint32_t visited_hash_entries(const pgemb_index *idx, uint32_t ef)
{
	uint64_t want = (uint64_t) ef * (uint64_t) env_int("PGEMB_VH_PER_EF", 64);
	if (want < 4096) want = 4096;
	uint32_t h = 4096;
	while (h < want && h < (1u << 20)) h <<= 1;
	const uint64_t bitmap_bytes = ((uint64_t) idx->capacity + 31) / 32 * 4;
	if (env_int("PGEMB_VISITED_HASH", 1) == 0 || bitmap_bytes <= (uint64_t) h * 4) return 0;  // the bitmap is the smaller structure
	return h;
}

// vhs: entries of the latency mode's shared-memory visited set (0 = none).  Both hash sets are reset -- and migrated to the
// bitmap -- from the slot's log, so the log must hold half a table (the kernel migrates before a table passes half full).
static pgemb_status ensure_workspace(pgemb_index *idx, uint32_t slots, uint32_t ef, uint32_t vh, uint32_t vhs)
{
	const uint32_t vis_words = (uint32_t) ((idx->capacity + 31) / 32);
	const uint32_t min_log = (vh > vhs ? vh : vhs) / 2;
	if (idx->ws_slots < slots || idx->vis_words != vis_words || idx->ws_vh < vh || idx->vlog_cap < min_log)
	{
		cudaFree(idx->d_visited);
		cudaFree(idx->d_vlog);
		cudaFree(idx->d_vhash);
		idx->d_visited = nullptr;
		idx->d_vlog = nullptr;
		idx->d_vhash = nullptr;
		if (slots < idx->ws_slots) slots = idx->ws_slots;
		if (vh < idx->ws_vh) vh = idx->ws_vh;
		idx->ws_slots = 0;
		idx->vlog_cap = (uint32_t) (idx->capacity < 32768 ? idx->capacity : 32768);
		if (idx->vlog_cap < vh / 2) idx->vlog_cap = vh / 2;
		if (idx->vlog_cap < min_log) idx->vlog_cap = min_log;
		CU_TRY(cudaMalloc((void **) &idx->d_visited, (size_t) slots * vis_words * 4));
		CU_TRY(cudaMemset(idx->d_visited, 0, (size_t) slots * vis_words * 4));
		CU_TRY(cudaMalloc((void **) &idx->d_vlog, (size_t) slots * idx->vlog_cap * 4));
		CU_TRY(cudaMalloc((void **) &idx->d_vhash, (size_t) slots * (vh ? vh : 1) * 4));
		CU_TRY(cudaMemset(idx->d_vhash, 0xff, (size_t) slots * (vh ? vh : 1) * 4));
		idx->ws_slots = slots;
		idx->ws_vh = vh;
		idx->vis_words = vis_words;
		cudaFree(idx->d_ovf);
		idx->d_ovf = nullptr;
		idx->ws_ef = 0;
		if (idx->l2_persist_max > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, idx->l2_persist_max * 3 / 4);
		cudaGetLastError();
	}
	if (idx->ws_ef < ef || !idx->d_ovf)
	{
		cudaFree(idx->d_ovf);
		idx->d_ovf = nullptr;
		CU_TRY(cudaMalloc((void **) &idx->d_ovf, (size_t) idx->ws_slots * ef * 8));
		idx->ws_ef = ef;
	}
	return PGEMB_OK;
}

// Every decision of one traversal launch, made from the index, the batch size, ef and the PGEMB_* knobs (read on every call).
struct SearchPlan
{
	uint32_t	 ef = 0;
	bool		 coop = false;		  // latency mode: a whole CTA cooperates on each query (search_kernel.cuh, COOP)
	bool		 res_global = false;  // the result queues live in global memory (d_resg)
	SearchConfig cfg;				  // slot-capped for res_global
	search_fn_t	 fn = nullptr;
	uint32_t	 vh = 0;  // visited-hash entries per slot (0: the bitmap alone)
	uint32_t	 grid = 0;
	bool		 pairs = false;	 // test both halves of a link list at once, if no list repeats an id
	uint32_t	 prefetch_links = 1;
	bool		 l2_window = false;	 // keep the per-slot hash sets resident in L2
	bool		 fast_small = true;	 // skip the driver calls that would only restate what the last launch configured
};

static pgemb_status plan_search(const pgemb_index *idx, size_t nq, size_t ef, SearchPlan *pl)
{
	pl->ef = (uint32_t) ef;
	pl->res_global = env_int("PGEMB_RES_GLOBAL", 0) != 0;
	// fewer queries than SMs: latency mode
	pl->coop = !pl->res_global && nq <= (size_t) idx->sm_count && env_int("PGEMB_COOP", 1) != 0;
	pgemb_status st = make_config(idx, pl->ef, &pl->cfg, pl->coop, pl->res_global);
	if (st == PGEMB_ERR_CAPACITY && !pl->res_global)
	{
		// 2 x ef result keys no longer fit a CTA's shared memory: the traversal variant that keeps them in global memory
		// (throughput-mode kernel, 4 lanes per row) -- slower per hop, but efSearch doubling must not fail (embedding.c:334)
		pl->res_global = true;
		pl->coop = false;
		st = make_config(idx, pl->ef, &pl->cfg, false, true);
	}
	if (st) return st;
	// small batches are spread over all SMs (the slots steal queries from one counter), not packed into few CTAs
	pl->grid = (uint32_t) (nq < (size_t) idx->sm_count ? nq : (size_t) idx->sm_count);
	pl->vh = visited_hash_entries(idx, pl->ef);
	if (pl->res_global)
	{
		// per-slot global state is O(ef): cap the slots so that the workspace stays within ~4 GB
		const uint64_t per_slot = (uint64_t) ef * 24u + (uint64_t) pl->vh * 4u + ((uint64_t) idx->capacity + 31) / 32 * 4u;
		const uint64_t max_slots = ((uint64_t) 4 << 30) / (per_slot ? per_slot : 1);
		uint32_t	   w = (uint32_t) (max_slots / (pl->grid ? pl->grid : 1));
		if (w < 1) w = 1;
		if (w < pl->cfg.warps) pl->cfg.warps = w;
		pl->cfg.slots = pl->cfg.warps * (uint32_t) idx->sm_count;
	}
	pl->fn = pick_search_kernel((int) idx->meta.dist_func, pl->coop, pl->cfg.tpr, pl->res_global);
	if (!pl->fn) return fail(PGEMB_ERR_ARG, "no kernel for this metric");
	// latency mode: both 32-id halves of a link list are test-and-set concurrently (one round trip instead of two dependent
	// ones) -- legal only when no list repeats an id, which holds for every list the bind kernels write and is checked once
	// for lists that came from the caller.  (Throughput mode: measured slower, 0.82 vs 0.85 of the roofline -- not used there.)
	pl->pairs = pl->coop && env_int("PGEMB_VISITED_PAIRS", 1) != 0;
	pl->prefetch_links = (uint32_t) env_int("PGEMB_PREFETCH", 1);
	pl->l2_window = pl->vh && idx->l2_window_max > 0 && env_int("PGEMB_L2_PERSIST", 1);
	pl->fast_small = env_int("PGEMB_FAST_SMALL", 1) != 0;
	return PGEMB_OK;
}

// The device state a launch of `pl` needs: the kernel's shared-memory attribute and residency, the workspace, the global result
// queues, the link-list check and the L2 window.
static pgemb_status prepare_search(pgemb_index *idx, const SearchPlan &pl, cudaStream_t s)
{
	if (!(pl.fast_small && idx->last_fn == (const void *) pl.fn && idx->last_smem == pl.cfg.smem))
	{
		CU_TRY(cudaFuncSetAttribute(pl.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) pl.cfg.smem));
		int occ = 0;
		CU_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, pl.fn, (int) pl.cfg.warps * 32, pl.cfg.smem));
		if (occ < 1) return fail(PGEMB_ERR_CAPACITY, "search kernel cannot be resident (shared memory / registers)");
		idx->last_fn = (const void *) pl.fn;
		idx->last_smem = pl.cfg.smem;
	}
	const pgemb_status st = ensure_workspace(idx, pl.cfg.slots, pl.ef, pl.vh, pl.cfg.vhs_entries);
	if (st) return st;
	const size_t keys = (size_t) pl.cfg.slots * 2 * pl.ef;
	if (pl.res_global && idx->resg_keys < keys)
	{
		cudaFree(idx->d_resg);
		idx->d_resg = nullptr;
		idx->resg_keys = 0;
		if (cudaMalloc((void **) &idx->d_resg, keys * 8) != cudaSuccess)
		{
			cudaGetLastError();
			return fail(PGEMB_ERR_NOMEM, "out of device memory for the result queues of this efSearch");
		}
		idx->resg_keys = keys;
	}
	if (pl.pairs && !idx->links_checked)
	{
		// caller-provided link lists: one pass to learn whether any list repeats an id (sticky until truncate)
		const uint32_t nn = (uint32_t) idx->n;
		int			   dup = 0;
		CU_TRY(cudaMemsetAsync(idx->d_counter + 3, 0, sizeof(int), s));
		if (nn) PGEMB_LAUNCH(links_distinct_kernel, (nn + 3) / 4, 128, 0, s, idx->d_links, idx->link_stride, (uint32_t) idx->meta.maxM, 0u, nn, (int *) (idx->d_counter + 3));
		g_launches++;
		CU_TRY(cudaMemcpyAsync(&dup, idx->d_counter + 3, sizeof(int), cudaMemcpyDeviceToHost, s));
		CU_TRY(cudaStreamSynchronize(s));
		idx->links_distinct = idx->links_distinct && dup == 0;
		idx->links_checked = true;
	}
	if (pl.l2_window)
	{
		if (idx->l2_limit_dropped)
		{
			if (idx->l2_persist_max > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, idx->l2_persist_max * 3 / 4);
			cudaGetLastError();
			idx->l2_limit_dropped = false;
		}
		// keep the per-slot visited sets (hit on every hop by L2 atomics) resident while rows stream through L2 -- unless the
		// stream already carries exactly this window
		size_t bytes = (size_t) pl.cfg.slots * pl.vh * 4;
		if (bytes > idx->l2_window_max) bytes = idx->l2_window_max;
		if (!(pl.fast_small && idx->last_l2_base == (const void *) idx->d_vhash && idx->last_l2_bytes == bytes && idx->last_l2_stream == s))
		{
			cudaStreamAttrValue av = {};
			av.accessPolicyWindow.base_ptr = idx->d_vhash;
			av.accessPolicyWindow.num_bytes = bytes;
			av.accessPolicyWindow.hitRatio = 1.0f;
			av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
			av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
			if (cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
			idx->last_l2_base = idx->d_vhash;
			idx->last_l2_bytes = bytes;
			idx->last_l2_stream = s;
		}
	}
	return PGEMB_OK;
}

// What one traversal launch searches and where its results go (device pointers): caller vectors (`queries`, rows of dim floats;
// timed for pgemb_last_kernel_ms) or stored nodes (`node_ids`: the build paths, raw mode, not timed).  `n` is required.
struct SearchRequest
{
	SearchRequest(size_t nq, size_t ef, const float *queries, int32_t *n) : nq(nq), ef(ef), queries(queries), n(n) {}
	SearchRequest(size_t nq, size_t ef, const uint32_t *node_ids, int32_t *n) : nq(nq), ef(ef), node_ids(node_ids), n(n) {}
	size_t				nq, ef;
	const float		   *queries = nullptr;
	const uint32_t	   *node_ids = nullptr;
	label_t			   *labels = nullptr;
	dist_t			   *dists = nullptr;
	idx_t			   *ids = nullptr;
	int32_t			   *n = nullptr;
	uint32_t		   *stats = nullptr;
	const unsigned int *avail = nullptr;  // a batch streamed in next to the kernel (SearchParams::avail)
	uint32_t		   *exp = nullptr, *exp_n = nullptr;  // pgemb_build_exact: each search's expansions (validate_kernel)
	uint32_t			exp_cap = 0;
};

// One traversal launch: argument checks, plan_search, prepare_search, the parameter block, the launch.
static pgemb_status launch_search(pgemb_index *idx, const SearchRequest &r, cudaStream_t s)
{
	if (!idx || !r.n) return fail(PGEMB_ERR_ARG, "null argument");
	if (r.ef < 1 || r.ef > (1u << 27)) return fail(PGEMB_ERR_ARG, "ef out of range");
	if (r.nq == 0) return PGEMB_OK;
	if (r.nq >= (1ull << 31)) return fail(PGEMB_ERR_ARG, "too many queries in one batch");
	pgemb_status st = set_device(idx);
	if (st) return st;
	SearchPlan pl;
	st = plan_search(idx, r.nq, r.ef, &pl);
	if (st) return st;
	st = prepare_search(idx, pl, s);
	if (st) return st;
	const bool stored = r.node_ids != nullptr;
	SearchParams p;
	memset(&p, 0, sizeof(p));
	p.vectors = idx->d_vectors;
	p.links = idx->d_links;
	p.labels = idx->d_labels;
	p.norms = idx->d_norms;
	p.n_items = (uint32_t) idx->n;
	p.dim = (uint32_t) idx->meta.dim;
	p.row_f = idx->row_f;
	p.link_stride = idx->link_stride;
	p.maxM = (uint32_t) idx->meta.maxM;
	p.entry = idx->meta.enterpoint_node;
	p.queries = r.queries;
	p.query_ids = r.node_ids;
	p.nq = (uint32_t) r.nq;
	p.q_stride = stored ? 0u : p.dim;
	p.ef = pl.ef;
	p.raw_mode = stored ? 1u : 0u;
	p.labels_out = r.labels;
	p.dists_out = r.dists;
	p.ids_out = r.ids;
	p.n_out = r.n;
	p.stats_out = r.stats;
	p.visited = idx->d_visited;
	p.vlog = idx->d_vlog;
	p.ovf = idx->d_ovf;
	p.res_g = pl.res_global ? idx->d_resg : nullptr;
	p.vis_words = idx->vis_words;
	p.vlog_cap = idx->vlog_cap;
	p.vhash = idx->d_vhash;
	p.vh_size = pl.vh;
	{
		uint32_t lg = 0;
		while ((1u << lg) < pl.vh) lg++;
		p.vh_shift = 32u - lg;
	}
	p.counter = idx->d_counter;
	p.avail = r.avail;
	p.exp_out = r.exp;
	p.exp_cap = r.exp_cap;
	p.exp_n_out = r.exp_n;
	p.error_flag = idx->d_error;
	apply_config(p, pl.cfg, idx->row_f);
	p.prefetch_links = pl.prefetch_links;
	p.visited_pairs = (pl.pairs && idx->links_distinct) ? 1u : 0u;
	CU_TRY(cudaMemsetAsync(idx->d_counter, 0, sizeof(unsigned int), s));
	if (!stored) CU_TRY(cudaEventRecord(idx->ev0, s));
	PGEMB_LAUNCH(pl.fn, pl.grid, pl.cfg.warps * 32, pl.cfg.smem, s, p);
	g_launches++;
	CU_TRY(cudaGetLastError());
	if (!stored)
	{
		CU_TRY(cudaEventRecord(idx->ev1, s));
		idx->ev_valid = true;
	}
	return PGEMB_OK;
}

static pgemb_status check_device_error(pgemb_index *idx, cudaStream_t s)
{
	int err = 0;
	CU_TRY(cudaMemcpyAsync(&err, idx->d_error, sizeof(int), cudaMemcpyDeviceToHost, s));
	CU_TRY(cudaStreamSynchronize(s));
	if (err != 0)
	{
		CU_TRY(cudaMemsetAsync(idx->d_error, 0, sizeof(int), s));
		return fail(PGEMB_ERR_STATE, err == 1 ? "corrupt graph: link id / count out of range"
											  : (err == 2 ? "tie-overflow buffer exceeded"
														  : (err == 4 ? "query batch never arrived on the device" : "bind failed (reference would throw)")));
	}
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_search_batch_device(pgemb_index *idx, size_t nq, const coord_t *d_queries, size_t ef,
												  label_t *d_labels_out, dist_t *d_dists_out, idx_t *d_ids_out, int32_t *d_n_out,
												  uint32_t *d_stats_out, void *stream)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	SearchRequest r(nq, ef, d_queries, d_n_out);
	r.labels = d_labels_out;
	r.dists = d_dists_out;
	r.ids = d_ids_out;
	r.stats = d_stats_out;
	return launch_search(idx, r, (cudaStream_t) stream);
}

struct HostOut { void *host; const void *dev; size_t bytes; };  // a caller's buffer (nullptr: not wanted), its part of the staging buffer

// Enqueues the caller's queries to d_q on `s` (fast_small) or on the copy stream, streamed in chunks next to the kernel (*avail:
// the count of queries landed so far) or whole before the launch.  *reader: the stream that reads the caller's buffer.
static pgemb_status copy_queries_in(pgemb_index *idx, size_t nq, const coord_t *queries, float *d_q, bool fast_small, cudaStream_t s,
									cudaStream_t *reader, const unsigned int **avail)
{
	const size_t dim = idx->meta.dim;
	if (fast_small)
	{
		CU_TRY(cudaMemcpyAsync(d_q, queries, nq * dim * sizeof(float), cudaMemcpyHostToDevice, s));
		return PGEMB_OK;
	}
	if (!idx->s_in)
	{
		CU_TRY(cudaStreamCreateWithFlags(&idx->s_in, cudaStreamNonBlocking));
		CU_TRY(cudaEventCreateWithFlags(&idx->ev_in, cudaEventDisableTiming));
		CU_TRY(cudaMallocHost((void **) &idx->h_avail, sizeof(unsigned int) * pgemb_index::kMaxChunks));
	}
	*reader = idx->s_in;
	// Streaming the batch in behind the running kernel needs kernels and copies to overlap.  Tools that serialise or replay
	// kernel launches (Nsight Compute, compute-sanitizer: both arrive through CUDA_INJECTION64_PATH; CUDA_LAUNCH_BLOCKING=1)
	// get the plain copy-then-launch order.  PGEMB_STREAM_QUERIES=0/1 overrides.
	const char	 *force = getenv("PGEMB_STREAM_QUERIES"), *inj = getenv("CUDA_INJECTION64_PATH");
	const bool	  streamed = (force && *force) ? atoi(force) != 0 : !(inj && *inj) && env_int("CUDA_LAUNCH_BLOCKING", 0) == 0;
	unsigned int *d_avail = idx->d_counter + 2;
	size_t		  nchunks = streamed ? (nq + 4095) / 4096 : 1;
	if (nchunks > (size_t) pgemb_index::kMaxChunks) nchunks = pgemb_index::kMaxChunks;
	const size_t per = (nq + nchunks - 1) / nchunks;
	CU_TRY(cudaMemsetAsync(d_avail, 0, sizeof(unsigned int), idx->s_in));
	if (streamed)
	{
		// the kernel may start as soon as `avail` reads 0 ...
		CU_TRY(cudaEventRecord(idx->ev_in, idx->s_in));
		CU_TRY(cudaStreamWaitEvent(s, idx->ev_in, 0));
		*avail = d_avail;
	}
	for (size_t c = 0, q0 = 0; q0 < nq; c++, q0 += per)
	{
		const size_t qn_ = (q0 + per <= nq) ? per : (nq - q0);
		cudaError_t	 ce = cudaMemcpyAsync(d_q + q0 * dim, queries + q0 * dim, qn_ * dim * sizeof(float), cudaMemcpyHostToDevice, idx->s_in);
		idx->h_avail[c] = (unsigned int) (q0 + qn_);
		if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_avail, &idx->h_avail[c], sizeof(unsigned int), cudaMemcpyHostToDevice, idx->s_in);
		if (ce != cudaSuccess) return fail(PGEMB_ERR_CUDA, std::string("pgemb_search_batch: copying the queries in failed: ") + cudaGetErrorString(ce));
	}
	if (!streamed)
	{
		// ... or, not streamed, only after the whole batch has landed
		CU_TRY(cudaEventRecord(idx->ev_in, idx->s_in));
		CU_TRY(cudaStreamWaitEvent(s, idx->ev_in, 0));
	}
	return PGEMB_OK;
}

// Ends a host-pointer search whose traversal is enqueued on `s`: the results go to the caller's buffers, the copy stream is
// drained and the kernel's sticky error flag is read.  outs[0] .. outs[4] are back to back in the staging buffer.
static pgemb_status search_hand_off(pgemb_index *idx, const HostOut (&outs)[5], bool fast_small, cudaStream_t s, cudaStream_t reader)
{
	// the outputs are one contiguous range of the staging buffer [labels | dists | ids | counts | stats]: after a small batch ONE
	// copy into pinned memory + the 4-byte error flag, then one synchronisation (a copy into the caller's pageable buffers would
	// block the host once per copy)
	const char	*d_first = (const char *) outs[0].dev;
	const size_t range = (size_t) ((const char *) outs[4].dev - d_first) + StageLayout::up(outs[4].bytes);
	if (fast_small && range + 64 <= ((size_t) 4 << 20))
	{
		if (idx->land_bytes < range + 64)
		{
			if (idx->h_land) cudaFreeHost(idx->h_land);
			idx->h_land = nullptr;
			idx->land_bytes = 0;
			CU_TRY(cudaMallocHost((void **) &idx->h_land, range + 64 + 65536));
			idx->land_bytes = range + 64 + 65536;
		}
		int *h_err = (int *) (idx->h_land + ((range + 15) & ~(size_t) 15));
		CU_TRY(cudaMemcpyAsync(idx->h_land, d_first, range, cudaMemcpyDeviceToHost, s));
		CU_TRY(cudaMemcpyAsync(h_err, idx->d_error, sizeof(int), cudaMemcpyDeviceToHost, s));
		CU_TRY(cudaStreamSynchronize(s));
		for (const HostOut &o : outs)
			if (o.host) memcpy(o.host, idx->h_land + ((const char *) o.dev - d_first), o.bytes);
		if (*h_err != 0) return check_device_error(idx, s);	 // reads, reports and clears the flag
		return PGEMB_OK;
	}
	for (const HostOut &o : outs)
		if (o.host) CU_TRY(cudaMemcpyAsync(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost, s));
	if (reader != s) CU_TRY(cudaStreamSynchronize(reader));
	return check_device_error(idx, s);
}

extern "C" pgemb_status pgemb_search_batch(pgemb_index *idx, size_t nq, const coord_t *queries, size_t ef, label_t *labels_out,
										   dist_t *dists_out, idx_t *ids_out, int32_t *n_out, uint32_t *stats_out)
{
	if (!idx || !queries || !n_out) return fail(PGEMB_ERR_ARG, "null argument");
	if (nq == 0) return PGEMB_OK;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t lb = nq * ef * sizeof(uint64_t), db = nq * ef * sizeof(float), ib = nq * ef * sizeof(uint32_t);
	const size_t nb = nq * sizeof(int32_t), sb = nq * 4 * sizeof(uint32_t);
	float		*d_q = nullptr, *d_d = nullptr;
	uint64_t	*d_l = nullptr;
	uint32_t	*d_i = nullptr, *d_s = nullptr;
	int32_t		*d_n = nullptr;
	const StageLayout stage{{d_q, nq * idx->meta.dim * sizeof(float)}, {d_l, lb}, {d_d, db}, {d_i, ib}, {d_n, nb}, {d_s, sb}};
	st = ensure_stage(idx, stage.bytes);
	if (st) return st;
	stage.place(idx->d_stage);
	cudaStream_t s = idx->stream, reader = s;
	// the outputs the caller asked for, in staging order
	const HostOut outs[5] = {{labels_out, d_l, lb}, {dists_out, d_d, db}, {ids_out, d_i, ib}, {n_out, d_n, nb}, {stats_out, d_s, sb}};
	SearchRequest r(nq, ef, d_q, d_n);
	r.labels = labels_out ? d_l : nullptr;
	r.dists = dists_out ? d_d : nullptr;
	r.ids = ids_out ? d_i : nullptr;
	r.stats = stats_out ? d_s : nullptr;
	// ONE traversal launch; the query batch is streamed in next to it: the copy stream moves chunk after chunk
	// H2D and publishes "queries available" after each, the kernel's slots wait for their query to land
	// (SearchParams::avail).  So the PCIe transfer hides behind the traversal instead of preceding it.
	// The copies are ENQUEUED FIRST: they then make progress whether or not the launch call returns at once, so a
	// blocking launch (CUDA_LAUNCH_BLOCKING, a profiler or sanitizer serialising kernels) cannot leave the kernel
	// waiting for data that was never queued.  Under such a tool (detected by its injection variable) the batch is
	// simply copied before the launch: replayed kernels must not depend on a concurrent copy.
	// A handful of queries (the reference-shaped hnsw_search: one) are not worth the streaming protocol: copy, launch, copy back
	// on ONE stream, one synchronisation.
	const bool fast_small = env_int("PGEMB_FAST_SMALL", 1) != 0 && nq <= 64;
	st = copy_queries_in(idx, nq, queries, d_q, fast_small, s, &reader, &r.avail);
	if (!st) st = launch_search(idx, r, s);
	if (!st) st = search_hand_off(idx, outs, fast_small, s, reader);
	if (st) cudaStreamSynchronize(reader);	// the caller's query buffer must not be read after we return
	return st;
}

// The device-pointer entry points are asynchronous and do not read the kernel's sticky error flag; a caller that wants to know
// (corrupt graph, tie-overflow, a batch that never arrived) polls it here -- synchronises `stream`, returns and clears the flag.
extern "C" pgemb_status pgemb_index_poll_error(pgemb_index *idx, void *stream)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	pgemb_status st = set_device(idx);
	if (st) return st;
	return check_device_error(idx, (cudaStream_t) stream);
}

extern "C" float pgemb_last_kernel_ms(const pgemb_index *idx)
{
	if (!idx || !idx->ev_valid) return -1.0f;
	float ms = -1.0f;
	if (cudaSetDevice(idx->device) != cudaSuccess) return -1.0f;
	if (cudaEventSynchronize(idx->ev1) != cudaSuccess) return -1.0f;
	if (cudaEventElapsedTime(&ms, idx->ev0, idx->ev1) != cudaSuccess) return -1.0f;
	return ms;
}

// ------------------------------------------------------------------------------------------------
// distances (distfunc.c:157-174; embedding.c:1022-1062)
// ------------------------------------------------------------------------------------------------
static pgemb_status launch_pairs(int metric, const float *d_a, const float *d_b, uint32_t dim, uint32_t n, int broadcast_a, float *d_out,
								 cudaStream_t s)
{
	const uint32_t threads = 128;
	const uint32_t lanes = (metric == DIST_L2) ? 8 : 4;
	const uint32_t blocks = (uint32_t) (((size_t) n * lanes + threads - 1) / threads);
	return with_metric(metric, [&](auto m) -> pgemb_status {
		PGEMB_LAUNCH(dist_pairs_kernel<decltype(m)::value>, blocks, threads, 0, s, d_a, d_b, dim, dim, dim, n, broadcast_a, d_out);
		g_launches++;
		CU_TRY(cudaGetLastError());
		return PGEMB_OK;
	});
}

// hnsw_dist_func has no handle to hang a buffer on (distfunc.c:171: two pointers and a length), so the staging area of the
// pair-distance entry points is process-wide: one device buffer on the current device, grown on demand, reused by every call
// (round 1 paid three cudaMalloc + three cudaFree per pair).  One caller at a time (a Postgres backend is single-threaded;
// other hosts serialise on the mutex).
static struct
{
	std::mutex mu;
	void	  *d = nullptr;
	size_t	   bytes = 0;
	int		   device = -1;
} g_pair_stage;

extern "C" pgemb_status pgemb_dist_batch(dist_func_t dist, size_t dim, size_t n, const coord_t *a, int broadcast_a, const coord_t *b,
										 dist_t *out)
{
	if ((!a || !b || !out) && n) return fail(PGEMB_ERR_ARG, "null argument");
	if (dim == 0 || dim > 65535) return fail(PGEMB_ERR_ARG, "dims out of range");
	if (n == 0) return PGEMB_OK;
	if (n >= (1ull << 28)) return fail(PGEMB_ERR_ARG, "batch too large");
	int dev = 0;
	CU_TRY(cudaGetDevice(&dev));
	const size_t ab = (broadcast_a ? 1 : n) * dim * sizeof(float), bb = n * dim * sizeof(float), ob = n * sizeof(float);
	float		*d_a = nullptr, *d_b = nullptr, *d_o = nullptr;
	const StageLayout stage{{d_a, ab}, {d_b, bb}, {d_o, ob}};
	std::lock_guard<std::mutex> lock(g_pair_stage.mu);
	if (g_pair_stage.device != dev || g_pair_stage.bytes < stage.bytes)
	{
		if (g_pair_stage.d)
		{
			if (g_pair_stage.device >= 0 && g_pair_stage.device != dev)
			{
				cudaSetDevice(g_pair_stage.device);
				cudaFree(g_pair_stage.d);
				cudaSetDevice(dev);
			}
			else
				cudaFree(g_pair_stage.d);
		}
		g_pair_stage.d = nullptr;
		g_pair_stage.bytes = 0;
		const size_t want = stage.bytes + stage.bytes / 2 + 65536;
		if (cudaMalloc(&g_pair_stage.d, want) != cudaSuccess)
		{
			cudaGetLastError();
			g_pair_stage.d = nullptr;
			return fail(PGEMB_ERR_NOMEM, "out of device memory for the distance batch");
		}
		g_pair_stage.bytes = want;
		g_pair_stage.device = dev;
	}
	stage.place(g_pair_stage.d);
	CU_TRY(cudaMemcpyAsync(d_a, a, ab, cudaMemcpyHostToDevice, 0));
	CU_TRY(cudaMemcpyAsync(d_b, b, bb, cudaMemcpyHostToDevice, 0));
	pgemb_status st = launch_pairs((int) dist, d_a, d_b, (uint32_t) dim, (uint32_t) n, broadcast_a, d_o, 0);
	if (st) return st;
	CU_TRY(cudaMemcpyAsync(out, d_o, ob, cudaMemcpyDeviceToHost, 0));
	CU_TRY(cudaStreamSynchronize(0));
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_dist_gather(pgemb_index *idx, size_t nq, const coord_t *queries, size_t k, const idx_t *ids, dist_t *out)
{
	if (!idx || ((!queries || !ids || !out) && nq && k)) return fail(PGEMB_ERR_ARG, "null argument");
	if (nq == 0 || k == 0) return PGEMB_OK;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t dim = idx->meta.dim;
	const size_t qb = nq * dim * 4, ib = nq * k * 4, ob = nq * k * 4;
	float		*d_q = nullptr, *d_o = nullptr;
	uint32_t	*d_i = nullptr;
	const StageLayout stage{{d_q, qb}, {d_i, ib}, {d_o, ob}};
	st = ensure_stage(idx, stage.bytes);
	if (st) return st;
	stage.place(idx->d_stage);
	cudaStream_t s = idx->stream;
	CU_TRY(cudaMemcpyAsync(d_q, queries, qb, cudaMemcpyHostToDevice, s));
	CU_TRY(cudaMemcpyAsync(d_i, ids, ib, cudaMemcpyHostToDevice, s));
	const int	   metric = (int) idx->meta.dist_func;
	const uint32_t threads = 128, lanes = (metric == DIST_L2) ? 8 : 4;
	const uint32_t blocks = (uint32_t) ((nq * k * lanes + threads - 1) / threads);
	st = with_metric(metric, [&](auto m) -> pgemb_status {
		PGEMB_LAUNCH(dist_gather_kernel<decltype(m)::value>, blocks, threads, 0, s, idx->d_vectors, idx->d_norms, idx->row_f, (uint32_t) dim,
					 (uint32_t) idx->n, d_q, (uint32_t) dim, (uint32_t) nq, (uint32_t) k, d_i, d_o);
		return PGEMB_OK;
	});
	if (st) return st;
	g_launches++;
	CU_TRY(cudaGetLastError());
	CU_TRY(cudaMemcpyAsync(out, d_o, ob, cudaMemcpyDeviceToHost, s));
	CU_TRY(cudaStreamSynchronize(s));
	return PGEMB_OK;
}

// ------------------------------------------------------------------------------------------------
// exact scan: the brute-force operator path (embedding.c:1022-1062; SURVEY.md 8(f3) / K6)
// ------------------------------------------------------------------------------------------------
// counters of the scan paths since load: [0] scans through the tensor-core filter, [1] (query,row) pairs it covered,
// [2] candidates re-scored exactly, [3] scans repeated on the exact kernels because the error-bound tripwire fired,
// [4] queries whose candidate list overflowed (re-scored against the whole chunk), [5] scans on the exact kernels only
static std::atomic<uint64_t> g_scan_tc{0}, g_scan_pairs{0}, g_scan_rescored{0}, g_scan_fallbacks{0}, g_scan_overflow{0}, g_scan_exact{0};
extern "C" void pgemb_scan_counters(uint64_t out[6])
{
	out[0] = g_scan_tc.load();
	out[1] = g_scan_pairs.load();
	out[2] = g_scan_rescored.load();
	out[3] = g_scan_fallbacks.load();
	out[4] = g_scan_overflow.load();
	out[5] = g_scan_exact.load();
}

// TF32 error bound of the filter, relative to |q||v|: both operands cut to 10 mantissa bits (2^-10 each, truncation or
// rounding), fp32 accumulation of `dim` products in the tensor core (2^-21 per term is generous), 50 % slack on top.
// PGEMB_SCAN_TC_REL_PPM overrides (parts per million).
static float scan_tc_rel(size_t dim)
{
	float	  rel = 1.5f * (2.0f / 1024.0f + (float) dim / 2097152.0f);
	const int ppm = env_int("PGEMB_SCAN_TC_REL_PPM", 0);
	if (ppm > 0) rel = (float) ppm * 1e-6f;
	return rel;
}

// squared norms of rows [norms_n, n) (cosine has them from the append; L2 computes them on the first tensor-core scan)
static pgemb_status ensure_row_norms(pgemb_index *idx, cudaStream_t s)
{
	if (idx->norms_n >= idx->n) return PGEMB_OK;
	const size_t first = idx->norms_n, n = idx->n - first;
	PGEMB_LAUNCH(norms_kernel, (uint32_t) ((n * 4 + 127) / 128), 128, 0, s, idx->d_vectors, idx->row_f, (uint32_t) idx->meta.dim, (uint32_t) first, (uint32_t) n,
				 idx->d_norms);
	g_launches++;
	CU_TRY(cudaGetLastError());
	idx->norms_n = idx->n;
	return PGEMB_OK;
}

#ifndef PGEMB_HOST_EMULATION
// cuTensorMapEncodeTiled through the runtime's driver entry point: no link-time dependency on libcuda
typedef CUresult (*tmap_encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
								   const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static tmap_encode_fn tmap_encoder()
{
	static tmap_encode_fn fn = nullptr;
	static bool			  tried = false;
	if (tried) return fn;
	tried = true;
	void						   *p = nullptr;
	cudaDriverEntryPointQueryResult qr;
	if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (tmap_encode_fn) p;
	else cudaGetLastError();
	return fn;
}
// [rows][row_f] fp32, K-major boxes of 32 floats x box_rows rows, 128-byte swizzle, out-of-range elements read as zero
static pgemb_status make_tmap(CUtensorMap *m, const float *base, uint32_t row_f, size_t rows, uint32_t box_rows)
{
	tmap_encode_fn enc = tmap_encoder();
	if (!enc) return fail(PGEMB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
	const cuuint64_t gdim[2] = {(cuuint64_t) row_f, (cuuint64_t) rows};
	const cuuint64_t gstr[1] = {(cuuint64_t) row_f * 4};
	const cuuint32_t box[2] = {kUmmaBK, box_rows};
	const cuuint32_t estr[2] = {1, 1};
	const CUresult	 r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *) base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
							 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) return fail(PGEMB_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int) r) + ")");
	return PGEMB_OK;
}
#endif

// one launch of the tensor-core filter over rows [r0, r0 + nr) for the nq staged queries (d_q: [nq][row_f], zero padded)
static pgemb_status launch_scan_filter(pgemb_index *idx, int metric, const float *d_q, const float *d_qn, uint32_t nq, uint32_t r0, uint32_t nr, float rel,
									   const float2 *d_qconst, uint32_t *d_cand_rows, float *d_cand_s, uint32_t *d_cand_n, uint32_t cap, float *d_dbg,
									   cudaStream_t s)
{
	ScanFilterParams p;
	memset(&p, 0, sizeof(p));
	p.nq = nq;
	p.r0 = r0;
	p.nr = nr;
	p.kblocks = (idx->row_f + kUmmaBK - 1) / kUmmaBK;
	p.n_qtiles = (nq + kUmmaTQ - 1) / kUmmaTQ;
	p.n_rtiles = (nr + kUmmaTR - 1) / kUmmaTR;
	p.qconst = d_qconst;
	p.vnorm2 = idx->d_norms;
	p.cand_rows = d_cand_rows;
	p.cand_s = d_cand_s;
	p.cand_n = d_cand_n;
	p.cap = cap;
	p.dbg_s = d_dbg;
#ifdef PGEMB_HOST_EMULATION
	(void) s;
	(void) d_qn;
	return with_tc_metric(metric, [&](auto m) -> pgemb_status {
		scan_filter_emulated<decltype(m)::value>(d_q, idx->row_f, idx->d_vectors, idx->row_f, (uint32_t) idx->meta.dim, rel, d_qn, p);
		g_launches++;
		return PGEMB_OK;
	});
#else
	(void) rel;
	(void) d_qn;
	CUtensorMap	 tq, tv;
	pgemb_status st = make_tmap(&tq, d_q, idx->row_f, nq, kUmmaTQ);
	if (st) return st;
	st = make_tmap(&tv, idx->d_vectors, idx->row_f, idx->n, kUmmaTR);
	if (st) return st;
	const uint32_t tiles = p.n_qtiles * p.n_rtiles;
	const uint32_t grid = tiles < (uint32_t) idx->sm_count ? tiles : (uint32_t) idx->sm_count;
	return with_tc_metric(metric, [&](auto m) -> pgemb_status {
		CU_TRY(cudaFuncSetAttribute(scan_filter_wgmma_kernel<decltype(m)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) kUmmaSmem));
		scan_filter_wgmma_kernel<decltype(m)::value><<<grid, kUmmaThreads, kUmmaSmem, s>>>(tq, tv, p);
		g_launches++;
		CU_TRY(cudaGetLastError());
		return PGEMB_OK;
	});
#endif
}

// Every decision of one scan call, from the index, the batch and the PGEMB_SCAN_* knobs.  The knobs are read on every call,
// so that a caller can switch them between calls.
struct ScanPlan
{
	int	   metric;		  // the query's operator (DIST_*): any of the three, whatever the index's own metric is
	bool   tc;			  // tensor-core filter + exact re-scoring; else the exact kernels alone
	bool   tiled;		  // exact pass: scan_tile_kernel (same bits as scan_dist_kernel, rows read once per query tile)
	int	   l2reset;		  // filter pass: what to give back of a traversal's L2 persistence window (scan_filter_pass)
	float  rel;			  // filter pass: error bound relative to |q||v|
	size_t chunk;		  // exact pass: rows per distance / select launch pair
	size_t c0, cap;		  // filter pass: first chunk (every row of it is a candidate), candidate list length per query
	size_t growth, cmax;  // filter pass: chunk growth factor, largest chunk
};

static ScanPlan plan_scan(const pgemb_index *idx, int metric, size_t nq, size_t k, bool allow_tc)
{
	ScanPlan p;
	// PGEMB_SCAN_TC: 0 = exact kernels only, 1 (default) = tensor-core filter for L2 / cosine when the table has at least
	// PGEMB_SCAN_TC_MIN_ROWS (default 4096) rows, 2 = always (tests).
	const int mode = env_int("PGEMB_SCAN_TC", 1);
	p.metric = metric;
	p.tc = allow_tc && metric != DIST_MANHATTAN && mode > 0 && (mode >= 2 || idx->n >= (size_t) env_int("PGEMB_SCAN_TC_MIN_ROWS", 4096));
	p.tiled = env_int("PGEMB_SCAN_TILED", 1) != 0;
	// PGEMB_SCAN_L2RESET: 0 = leave as is, 1 = reset lines + window, 2 (default) = also drop the set-aside limit until the next
	// traversal configures it again
	p.l2reset = env_int("PGEMB_SCAN_L2RESET", 2);
	p.rel = scan_tc_rel(idx->meta.dim);
	int lg = env_int("PGEMB_SCAN_CHUNK_LOG2", 0);
	p.chunk = (lg >= 8 && lg <= 20) ? (size_t) 1 << lg : (size_t) 1 << 14;
	while (p.chunk > 256 && nq * p.chunk * 4 > ((size_t) 256 << 20)) p.chunk >>= 1;
	// tensor-core path: first chunk establishes the threshold (every row of it is a candidate), then x2 per chunk (PGEMB_SCAN_TC_GROWTH)
	lg = env_int("PGEMB_SCAN_TC_CHUNK0_LOG2", 0);
	p.c0 = (lg >= 5 && lg <= 20) ? (size_t) 1 << lg : ((2 * k > 256 ? 2 * k : 256) + 255) / 256 * 256;
	const int cap = env_int("PGEMB_SCAN_TC_CAP", 0);
	p.cap = cap > 0 ? (size_t) cap : (2 * p.c0 > 4096 ? 2 * p.c0 : 4096);
	p.growth = (size_t) env_int("PGEMB_SCAN_TC_GROWTH", 2);	// measured (profiles/r2_call10_scan_growth_sweep.log): 2 / 3 / 4 / 8 -> 6.7 / 7.7 / 8.0 / 8.6 ms per 1024 x 1M x 768 scan at k 64
	if (p.growth < 2) p.growth = 2;
	// chunks stop growing at 2^20 rows (PGEMB_SCAN_TC_CHUNK_MAX_LOG2): the candidate lists are sized for what passes the filter in
	// one chunk, and a table of tens of millions of rows must not end in one chunk of half the table
	lg = env_int("PGEMB_SCAN_TC_CHUNK_MAX_LOG2", 0);
	p.cmax = (lg >= 8 && lg <= 30) ? (size_t) 1 << lg : (size_t) 1 << 20;
	return p;
}

// The arrays of one scan in the staging buffer.  q: [nq][row_f] queries; dist: [nq][chunk] distances of the exact pass;
// td, tl, tn: running top-k (order keys, labels, counts); sd, sl: select / re-score scratch of the same shape; qn: query squared
// norms; cn, qc, cr, cs: candidate counts, filter constants, candidate rows, candidate products; cnt: [0] re-scored,
// [1] tripwire, [2] overflowed queries
struct ScanBuffers
{
	float	 *q = nullptr, *dist = nullptr, *qn = nullptr, *cs = nullptr;
	uint32_t *td = nullptr, *sd = nullptr, *tn = nullptr, *cn = nullptr, *cr = nullptr, *cnt = nullptr;
	uint64_t *tl = nullptr, *sl = nullptr;
	float2	 *qc = nullptr;
};

// nq queries into d_q at row_f stride, zero padded (the TMA tensor map reads whole 16-byte units)
static pgemb_status stage_queries(const pgemb_index *idx, float *d_q, const coord_t *queries, size_t nq, cudaMemcpyKind kind, cudaStream_t s)
{
	const size_t rf = idx->row_f, dim = idx->meta.dim;
	if (rf != dim) CU_TRY(cudaMemsetAsync(d_q, 0, nq * rf * 4, s));
	CU_TRY(cudaMemcpy2DAsync(d_q, rf * 4, queries, dim * 4, dim * 4, nq, kind, s));
	return PGEMB_OK;
}

// K6: tensor-core filter + exact re-scoring over the whole table in geometrically growing chunks (scan_umma_kernel.cuh)
static pgemb_status scan_filter_pass(pgemb_index *idx, const ScanPlan &p, const ScanBuffers &b, size_t nq, size_t k, cudaStream_t s)
{
	// The filter lives on L2 reuse (the table streams from HBM once, the other query tiles re-read it from L2).  A traversal
	// on this index leaves an L2 persistence window behind (the per-slot visited sets, prepare_search): give those lines and
	// the set-aside back before scanning.
	if (p.l2reset > 0 && idx->last_l2_base != nullptr)
	{
		cudaStreamAttrValue av;
		memset(&av, 0, sizeof(av));
		av.accessPolicyWindow.num_bytes = 0;
		if (cudaStreamSetAttribute(idx->last_l2_stream ? idx->last_l2_stream : s, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
		if (cudaCtxResetPersistingL2Cache() != cudaSuccess) cudaGetLastError();
		if (p.l2reset > 1 && cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0) != cudaSuccess) cudaGetLastError();
		idx->last_l2_base = nullptr;
		idx->l2_limit_dropped = p.l2reset > 1;
	}
	pgemb_status st = ensure_row_norms(idx, s);
	if (st) return st;
	const int	 metric = p.metric;
	const size_t N = idx->n, dim = idx->meta.dim, rf = idx->row_f;
	CU_TRY(cudaMemsetAsync(b.cnt, 0, 16, s));
	st = with_tc_metric(metric, [&](auto m) -> pgemb_status {
		PGEMB_LAUNCH(scan_qconst_init_kernel<decltype(m)::value>, (uint32_t) ((nq + 127) / 128), 128, 0, s, b.qn, (uint32_t) nq, p.rel, b.qc, b.cn);
		return PGEMB_OK;
	});
	if (st) return st;
	g_launches++;
	size_t csize = p.c0;
	for (size_t r0 = 0; r0 < N;)
	{
		size_t nr = N - r0 < csize ? N - r0 : csize;
		if (N - r0 - nr < nr / 8) nr = N - r0;	// do not leave a sliver for an extra launch pair
		st = launch_scan_filter(idx, metric, b.q, b.qn, (uint32_t) nq, (uint32_t) r0, (uint32_t) nr, p.rel, b.qc, b.cr, b.cs, b.cn, (uint32_t) p.cap, nullptr, s);
		if (st) return st;
		st = with_tc_metric(metric, [&](auto m) -> pgemb_status {
			PGEMB_LAUNCH(scan_rescore_kernel<decltype(m)::value>, (uint32_t) nq, 128, 0, s, idx->d_vectors, idx->row_f, (uint32_t) dim, idx->d_norms, b.q,
						 (uint32_t) rf, b.qn, idx->d_labels, (uint32_t) nq, (uint32_t) r0, (uint32_t) nr, (uint32_t) k, p.rel, b.cr, b.cs, b.cn, (uint32_t) p.cap,
						 b.td, b.tl, b.tn, b.sd, b.sl, b.qc, b.cnt);
			return PGEMB_OK;
		});
		if (st) return st;
		g_launches++;
		CU_TRY(cudaGetLastError());
		r0 += nr;
		csize *= p.growth;
		if (csize > p.cmax) csize = p.cmax > p.c0 ? p.cmax : p.c0;
	}
	g_scan_tc++;
	g_scan_pairs += (uint64_t) nq * N;
	return PGEMB_OK;
}

// the exact kernels: per chunk of rows, every (query, row) distance, then its fold into the running top-k
static pgemb_status scan_exact_pass(pgemb_index *idx, const ScanPlan &p, const ScanBuffers &b, size_t nq, size_t k, cudaStream_t s)
{
	const int	   metric = p.metric;
	const size_t   N = idx->n, dim = idx->meta.dim, rf = idx->row_f;
	const uint32_t lanes = (metric == DIST_L2) ? 8 : 4;
	if (metric == DIST_COSINE)
	{
		// the cosine epilogue divides by the row norms: a mirror of another metric computes them on its first cosine scan
		const pgemb_status st = ensure_row_norms(idx, s);
		if (st) return st;
	}
	g_scan_exact++;
	for (size_t r0 = 0; r0 < N; r0 += p.chunk)
	{
		const size_t   nr = (N - r0 < p.chunk) ? (N - r0) : p.chunk;
		const uint32_t threads = 128;
		const uint32_t blocks = (uint32_t) ((nq * nr * lanes + threads - 1) / threads);
		const pgemb_status st = with_metric(metric, [&](auto m) -> pgemb_status {
			constexpr uint32_t tq = ScanTile<decltype(m)::value>::TQ;
			if (p.tiled)
				PGEMB_LAUNCH(scan_tile_kernel<decltype(m)::value>, dim3((uint32_t) ((nq + tq - 1) / tq), (uint32_t) ((nr + kScanTileRows - 1) / kScanTileRows)),
							 kScanThreads, 0, s, idx->d_vectors, idx->d_norms, idx->row_f, (uint32_t) dim, b.q, (uint32_t) rf, b.qn, (uint32_t) nq,
							 (uint32_t) r0, (uint32_t) nr, b.dist);
			else
				PGEMB_LAUNCH(scan_dist_kernel<decltype(m)::value>, blocks, threads, 0, s, idx->d_vectors, idx->d_norms, idx->row_f, (uint32_t) dim, b.q,
							 (uint32_t) rf, (uint32_t) nq, (uint32_t) r0, (uint32_t) nr, b.dist);
			return PGEMB_OK;
		});
		if (st) return st;
		PGEMB_LAUNCH(scan_select_kernel, (uint32_t) ((nq + 3) / 4), 128, 0, s, b.dist, idx->d_labels, (uint32_t) nq, (uint32_t) r0, (uint32_t) nr, (uint32_t) k,
					 b.td, b.tl, b.tn, b.sd, b.sl);
		g_launches += 2;
		CU_TRY(cudaGetLastError());
	}
	return PGEMB_OK;
}

// The results in the caller's layout (scan_finish_kernel), then the tripwire counters into cnt[4] if asked for, and one
// synchronisation.  Device pointers receive the results directly.  For host pointers the kernel writes into the select /
// re-score scratch and the candidate counts, which have the outputs' shapes and are dead after the last pass, and the
// results are copied from there.
static pgemb_status scan_hand_off(const ScanBuffers &b, size_t nq, size_t k, label_t *labels_out, dist_t *dists_out, int32_t *n_out, bool device_io,
								  uint32_t *cnt, cudaStream_t s)
{
	label_t *lo = device_io ? labels_out : b.sl;
	dist_t	*dout = (device_io || !dists_out) ? dists_out : (dist_t *) b.sd;
	int32_t *no = device_io ? n_out : (int32_t *) b.cn;
	PGEMB_LAUNCH(scan_finish_kernel, (uint32_t) ((nq * k + 255) / 256), 256, 0, s, b.td, b.tl, b.tn, (uint32_t) nq, (uint32_t) k, lo, dout, no);
	g_launches++;
	CU_TRY(cudaGetLastError());
	if (!device_io)
	{
		CU_TRY(cudaMemcpyAsync(labels_out, lo, nq * k * 8, cudaMemcpyDeviceToHost, s));
		if (dists_out) CU_TRY(cudaMemcpyAsync(dists_out, dout, nq * k * 4, cudaMemcpyDeviceToHost, s));
		CU_TRY(cudaMemcpyAsync(n_out, no, nq * 4, cudaMemcpyDeviceToHost, s));
	}
	if (cnt) CU_TRY(cudaMemcpyAsync(cnt, b.cnt, 16, cudaMemcpyDeviceToHost, s));
	CU_TRY(cudaStreamSynchronize(s));
	return PGEMB_OK;
}

// One group of queries: stage them, run one pass over the table, hand the results over.  *tc_violation: the tensor-core
// filter saw a product outside its assumed error bound.
static pgemb_status scan_topk_impl(pgemb_index *idx, int metric, size_t nq, const coord_t *queries, size_t k, label_t *labels_out, dist_t *dists_out,
								   int32_t *n_out, bool allow_tc, bool *tc_violation, bool device_io)
{
	*tc_violation = false;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const ScanPlan p = plan_scan(idx, metric, nq, k, allow_tc);
	cudaStream_t   s = idx->stream;
	const size_t   qb = nq * idx->row_f * 4, db = p.tc ? 0 : nq * p.chunk * 4, kd = nq * k * 4, kl = nq * k * 8, nb = nq * 4;
	const size_t   cb = p.tc ? nq * p.cap * 4 : 0;
	ScanBuffers	   b;
	const StageLayout stage{{b.q, qb}, {b.dist, db}, {b.td, kd}, {b.sd, kd}, {b.tl, kl}, {b.sl, kl}, {b.tn, nb},
							{b.qn, nb}, {b.cn, nb}, {b.qc, nq * 8}, {b.cr, cb}, {b.cs, cb}, {b.cnt, 16}};
	st = ensure_stage(idx, stage.bytes + 256);
	if (st) return st;
	stage.place(idx->d_stage);
	st = stage_queries(idx, b.q, queries, nq, device_io ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s);
	if (st) return st;
	CU_TRY(cudaMemsetAsync(b.tn, 0, nb, s));
	if (p.tc || (p.tiled && metric == DIST_COSINE))
	{
		PGEMB_LAUNCH(norms_kernel, (uint32_t) ((nq * 4 + 127) / 128), 128, 0, s, b.q, idx->row_f, (uint32_t) idx->meta.dim, 0u, (uint32_t) nq, b.qn);
		g_launches++;
		CU_TRY(cudaGetLastError());
	}
	st = p.tc ? scan_filter_pass(idx, p, b, nq, k, s) : scan_exact_pass(idx, p, b, nq, k, s);
	if (st) return st;
	uint32_t cnt[4] = {0, 0, 0, 0};
	st = scan_hand_off(b, nq, k, labels_out, dists_out, n_out, device_io, p.tc ? cnt : nullptr, s);
	if (st) return st;
	if (p.tc)
	{
		g_scan_rescored += cnt[0];
		g_scan_overflow += cnt[2];
		*tc_violation = cnt[1] != 0;
	}
	return PGEMB_OK;
}

static pgemb_status scan_topk_groups(pgemb_index *idx, int metric, size_t nq, const coord_t *queries, size_t k, label_t *labels_out, dist_t *dists_out,
									 int32_t *n_out, bool device_io)
{
	if (!idx || ((!queries || !labels_out || !n_out) && nq)) return fail(PGEMB_ERR_ARG, "null argument");
	if (metric < 0 || metric > 2) return fail(PGEMB_ERR_ARG, "unknown distance function");
	if (nq == 0) return PGEMB_OK;
	if (k < 1 || k > 4096) return fail(PGEMB_ERR_ARG, "k out of range (1..4096)");
	if (nq > (1u << 20)) return fail(PGEMB_ERR_ARG, "too many queries in one scan batch");
	// query groups: the candidate lists of the tensor-core path are sized per group
	const size_t group = 4096;
	for (size_t q0 = 0; q0 < nq; q0 += group)
	{
		const size_t gq = nq - q0 < group ? nq - q0 : group;
		bool		 viol = false;
		pgemb_status st = scan_topk_impl(idx, metric, gq, queries + q0 * idx->meta.dim, k, labels_out + q0 * k, dists_out ? dists_out + q0 * k : nullptr, n_out + q0,
										 true, &viol, device_io);
		if (st == PGEMB_OK && viol)
		{
			// the tensor-core filter saw a product outside its assumed error bound: its result is not trusted
			g_scan_fallbacks++;
			fprintf(stderr, "pgemb_scan_topk: tensor-core error bound exceeded, repeating the scan on the exact kernels\n");
			st = scan_topk_impl(idx, metric, gq, queries + q0 * idx->meta.dim, k, labels_out + q0 * k, dists_out ? dists_out + q0 * k : nullptr, n_out + q0, false, &viol,
								device_io);
		}
		if (st) return st;
	}
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_scan_topk_op(pgemb_index *idx, dist_func_t metric, size_t nq, const coord_t *queries, size_t k, label_t *labels_out,
										   dist_t *dists_out, int32_t *n_out)
{
	return scan_topk_groups(idx, (int) metric, nq, queries, k, labels_out, dists_out, n_out, false);
}

extern "C" pgemb_status pgemb_scan_topk(pgemb_index *idx, size_t nq, const coord_t *queries, size_t k, label_t *labels_out, dist_t *dists_out,
										int32_t *n_out)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null argument");
	return pgemb_scan_topk_op(idx, idx->meta.dist_func, nq, queries, k, labels_out, dists_out, n_out);
}

// The same scan with DEVICE pointers in and out (the caller's stream is only synchronised with: the scan runs on the index's own
// stream and has finished when the call returns).  For callers whose queries and results live in HBM already: the sharded scan.
extern "C" pgemb_status pgemb_scan_topk_op_device(pgemb_index *idx, dist_func_t metric, size_t nq, const coord_t *d_queries, size_t k, label_t *d_labels_out,
												  dist_t *d_dists_out, int32_t *d_n_out, void *stream)
{
	if (idx && stream)
	{
		pgemb_status st = set_device(idx);
		if (st) return st;
		CU_TRY(cudaStreamSynchronize((cudaStream_t) stream));  // the queries may have been produced on it
	}
	return scan_topk_groups(idx, (int) metric, nq, d_queries, k, d_labels_out, d_dists_out, d_n_out, true);
}

extern "C" pgemb_status pgemb_scan_topk_device(pgemb_index *idx, size_t nq, const coord_t *d_queries, size_t k, label_t *d_labels_out, dist_t *d_dists_out,
											   int32_t *d_n_out, void *stream)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null argument");
	return pgemb_scan_topk_op_device(idx, idx->meta.dist_func, nq, d_queries, k, d_labels_out, d_dists_out, d_n_out, stream);
}

// Debug / test entry: the raw tensor-core products S[q][j] = q . row(r0 + j) of the K6 kernel (TF32 operands, fp32
// accumulate), so that a test can check the wgmma descriptors, the swizzled TMA tiles and the accumulator layout against a
// float64 product directly.  Host pointers; out[nq * nr].
extern "C" pgemb_status pgemb_debug_umma_product(pgemb_index *idx, size_t nq, const coord_t *queries, size_t r0, size_t nr, float *out)
{
	if (!idx || ((!queries || !out) && nq && nr)) return fail(PGEMB_ERR_ARG, "null argument");
	if (nq == 0 || nr == 0) return PGEMB_OK;
	if (r0 + nr > idx->n) return fail(PGEMB_ERR_ARG, "range beyond index size");
	if (idx->meta.dist_func == DIST_MANHATTAN) return fail(PGEMB_ERR_ARG, "manhattan has no tensor-core path");
	if (nq * nr > ((size_t) 1 << 28)) return fail(PGEMB_ERR_ARG, "debug product too large");
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t rf = idx->row_f, dim = idx->meta.dim;
	float		*d_q = nullptr, *d_qn = nullptr, *d_s = nullptr;
	const StageLayout stage{{d_q, nq * rf * 4}, {d_qn, nq * 4}, {d_s, nq * nr * 4}};
	st = ensure_stage(idx, stage.bytes + 256);
	if (st) return st;
	stage.place(idx->d_stage);
	cudaStream_t s = idx->stream;
	st = stage_queries(idx, d_q, queries, nq, cudaMemcpyHostToDevice, s);
	if (st) return st;
	CU_TRY(cudaMemsetAsync(d_s, 0, nq * nr * 4, s));
	st = ensure_row_norms(idx, s);
	if (st) return st;
	st = launch_scan_filter(idx, (int) idx->meta.dist_func, d_q, d_qn, (uint32_t) nq, (uint32_t) r0, (uint32_t) nr, scan_tc_rel(dim), nullptr, nullptr, nullptr, nullptr,
							0, d_s, s);
	if (st) return st;
	CU_TRY(cudaMemcpyAsync(out, d_s, nq * nr * 4, cudaMemcpyDeviceToHost, s));
	CU_TRY(cudaStreamSynchronize(s));
	return PGEMB_OK;
}

extern "C" void hnsw_init_dist_func(void)
{
	// distfunc.c:159-169 picks the CPU SIMD variant here; the CUDA path has a single variant per metric
	// (the AVX2 summation order).  Touch the runtime so that later calls do not pay context creation.
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) cudaGetLastError();
}

extern "C" dist_t hnsw_dist_func(dist_func_t dist, coord_t const *ax, coord_t const *bx, size_t dim)
{
	float		 out = NAN;
	pgemb_status st = pgemb_dist_batch(dist, dim, 1, ax, 0, bx, &out);
	if (st != PGEMB_OK) return NAN;
	return out;
}

// ------------------------------------------------------------------------------------------------
// reference-shaped search / bind
// ------------------------------------------------------------------------------------------------
extern "C" bool hnsw_search(HnswMetadata *meta, const coord_t *point, size_t *n_results, label_t **results)
{
	if (!meta || !point || !n_results || !results) return false;
	PgembHostIndex *h = reinterpret_cast<PgembHostIndex *>(meta);
	if (!h->dev) { g_last_error = "hnsw_search: no device index attached to this HnswMetadata"; return false; }
	const size_t ef = meta->efSearch;  // re-read every call: the caller doubles it (embedding.c:334)
	if (ef < 1) return false;
	label_t *buf = (label_t *) malloc(ef * sizeof(label_t));
	if (!buf) return false;
	int32_t		 n = 0;
	pgemb_status st = pgemb_search_batch(h->dev, 1, point, ef, buf, nullptr, nullptr, &n, nullptr);
	if (st != PGEMB_OK)
	{
		free(buf);
		return false;
	}
	*results = buf;
	*n_results = (size_t) n;
	return true;
}

extern "C" pgemb_status pgemb_bind_point(pgemb_index *idx, idx_t id)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	if ((size_t) id >= idx->n) return fail(PGEMB_ERR_ARG, "bind: node not stored");
	pgemb_status st = set_device(idx);
	if (st) return st;
	st = bind_points(idx, id, 1);
	if (st) return st;
	return check_device_error(idx, idx->stream);
}

extern "C" pgemb_status pgemb_insert_batch(pgemb_index *idx, size_t n, const coord_t *coords, const label_t *labels)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	const size_t first = idx->n;
	pgemb_status st = pgemb_index_append(idx, n, coords, labels, nullptr);
	if (st) return st;
	st = bind_points(idx, (idx_t) first, n);
	if (st) return st;
	return check_device_error(idx, idx->stream);
}

extern "C" bool hnsw_bind_point(HnswMetadata *meta, const coord_t *point, idx_t cur)
{
	(void) point;  // the node's coordinates were stored by the caller before this call (embedding.c:619-621)
	if (!meta) return false;
	PgembHostIndex *h = reinterpret_cast<PgembHostIndex *>(meta);
	if (!h->dev) { g_last_error = "hnsw_bind_point: no device index attached"; return false; }
	h->dev->meta.efConstruction = meta->efConstruction;
	pgemb_status st = pgemb_bind_point(h->dev, cur);
	if (st != PGEMB_OK)
	{
		fprintf(stderr, "Catch %s\n", pgemb_last_error());  // hnswalg.cpp:288
		return false;
	}
	return true;
}

// ------------------------------------------------------------------------------------------------
// index-scan iteration (SURVEY.md 8(f2)): hnsw_beginscan / hnsw_gettuple / hnsw_endscan, embedding.c:249-387
// ------------------------------------------------------------------------------------------------
// The reference's scan keeps the TIDs returned so far, and when they run out while the last search was "full"
// (n == efSearch) it doubles efSearch IN PLACE, searches again and appends the TIDs it has not returned yet
// (embedding.c:329-366).  Restated statement by statement -- including the two quirks a caller can observe:
//   * `if (n_results <= so->n_results) return false` compares the NEW search's count with the ACCUMULATED count (:338);
//   * the de-duplication bsearch runs over so->n_results entries while so->n_results GROWS (:357-363): sorted prefix +
//     unsorted suffix, so a probe can miss a TID that is in the prefix and the scan returns that tuple twice.  The probe
//     sequence is glibc's bsearch (l = 0, u = n, idx = (l + u) / 2).
// A TID is the label's low 6 bytes (memcpy of sizeof(ItemPointerData), :324/:361); ItemPointerCompare orders by block number
// ((bi_hi << 16) | bi_lo), then ip_posid.  The checker's restatement of the same loop is oracle/scan_iter.c.
struct pgemb_index_scan
{
	pgemb_index			 *idx = nullptr;
	std::vector<float>	  key;
	size_t				  ef = 0;		 // so->hnsw->meta.efSearch: per-scan copy (embedding.c:254), doubled in place
	std::vector<uint64_t> results;		 // TIDs (flags stripped), in the order they are handed out
	size_t				  curr = 0;
	bool				  no_more = true;  // embedding.c:258
	uint64_t			  searches = 0;
};

static inline int tid_compare(uint64_t a, uint64_t b)
{
	const uint32_t ba = (uint32_t) (((a & 0xffffu) << 16) | ((a >> 16) & 0xffffu)), bb = (uint32_t) (((b & 0xffffu) << 16) | ((b >> 16) & 0xffffu));
	if (ba != bb) return ba < bb ? -1 : 1;
	const uint32_t pa = (uint32_t) ((a >> 32) & 0xffffu), pb = (uint32_t) ((b >> 32) & 0xffffu);
	if (pa != pb) return pa < pb ? -1 : 1;
	return 0;
}

extern "C" pgemb_status pgemb_index_scan_begin(pgemb_index *idx, const coord_t *query, size_t efSearch, pgemb_index_scan **out)
{
	if (!idx || !query || !out) return fail(PGEMB_ERR_ARG, "null argument");
	if (efSearch < 1) return fail(PGEMB_ERR_ARG, "efsearch must be >= 1");
	pgemb_index_scan *so = new (std::nothrow) pgemb_index_scan();
	if (!so) return fail(PGEMB_ERR_NOMEM, "out of host memory");
	try
	{
		so->key.assign(query, query + idx->meta.dim);
	}
	catch (const std::bad_alloc &)
	{
		delete so;
		return fail(PGEMB_ERR_NOMEM, "out of host memory");
	}
	so->idx = idx;
	so->ef = efSearch;
	*out = so;
	return PGEMB_OK;
}

// one hnsw_search with the scan's current efSearch; labels -> TIDs
static pgemb_status scan_search(pgemb_index_scan *so, std::vector<uint64_t> &tids)
{
	std::vector<uint64_t> lab;
	try
	{
		lab.resize(so->ef);
	}
	catch (const std::bad_alloc &)
	{
		return fail(PGEMB_ERR_NOMEM, "out of host memory");
	}
	int32_t		 n = 0;
	pgemb_status st = pgemb_search_batch(so->idx, 1, so->key.data(), so->ef, lab.data(), nullptr, nullptr, &n, nullptr);
	so->searches++;
	if (st) return st;
	tids.assign(lab.begin(), lab.begin() + n);
	for (auto &t : tids) t &= 0xffffffffffffull;
	return PGEMB_OK;
}

extern "C" int pgemb_index_scan_next(pgemb_index_scan *so, label_t *tid_out)
{
	if (!so || !tid_out)
	{
		fail(PGEMB_ERR_ARG, "null argument");
		return -PGEMB_ERR_ARG;
	}
	try
	{
		std::vector<uint64_t> res;
		if (so->curr == 0)
		{
			pgemb_status st = scan_search(so, res);
			if (st) return -st;	 // "HNSW index search failed" (embedding.c:318)
			so->results = res;
			so->no_more = res.size() < so->ef;
		}
		if (so->curr >= so->results.size())
		{
			if (so->no_more) return 0;
			if (so->ef > ((size_t) 1 << 40)) return 0;	// efSearch cannot overflow before every node has been returned
			so->ef *= 2;  // embedding.c:334
			pgemb_status st = scan_search(so, res);
			if (st) return -st;
			if (res.size() <= so->results.size()) return 0;	 // "No new results found"
			so->no_more = res.size() < so->ef;
			size_t n_results = so->results.size();
			so->results.resize(n_results + res.size());
			std::sort(so->results.begin(), so->results.begin() + n_results, [](uint64_t a, uint64_t b) { return tid_compare(a, b) < 0; });
			for (uint64_t t : res)
			{
				size_t l = 0, u = n_results;
				bool   found = false;
				while (l < u)
				{
					const size_t i = (l + u) / 2;
					const int	 c = tid_compare(t, so->results[i]);
					if (c < 0) u = i;
					else if (c > 0) l = i + 1;
					else { found = true; break; }
				}
				if (!found) so->results[n_results++] = t;
			}
			so->results.resize(n_results);
		}
		*tid_out = so->results[so->curr++];
		return 1;
	}
	catch (const std::bad_alloc &)
	{
		fail(PGEMB_ERR_NOMEM, "out of host memory");
		return -PGEMB_ERR_NOMEM;
	}
}

extern "C" pgemb_status pgemb_index_scan_next_batch(pgemb_index_scan *so, size_t max, label_t *tids_out, size_t *n_out)
{
	if (!so || (!tids_out && max) || !n_out) return fail(PGEMB_ERR_ARG, "null argument");
	size_t n = 0;
	while (n < max)
	{
		const int r = pgemb_index_scan_next(so, &tids_out[n]);
		if (r < 0) return (pgemb_status) -r;
		if (r == 0) break;
		n++;
	}
	*n_out = n;
	return PGEMB_OK;
}

extern "C" size_t pgemb_index_scan_ef(const pgemb_index_scan *so) { return so ? so->ef : 0; }
extern "C" uint64_t pgemb_index_scan_searches(const pgemb_index_scan *so) { return so ? so->searches : 0; }
extern "C" void pgemb_index_scan_end(pgemb_index_scan *so) { delete so; }

// ------------------------------------------------------------------------------------------------
// K4 driver: sequential binds (hnsw_bind_point semantics, hnswalg.cpp:225-232) without host round trips
// ------------------------------------------------------------------------------------------------
static pgemb_status ensure_bind_ws(pgemb_index *idx, size_t points, size_t ef)
{
	BindWorkspace &w = idx->bind_ws;
	const size_t   M = idx->meta.M ? idx->meta.M : 1;
	if (w.cap_points >= points && w.cap_ef >= ef && w.cap_m >= M) return PGEMB_OK;
	bind_ws_free(w);
	CU_TRY(cudaMalloc((void **) &w.d_qids, points * sizeof(uint32_t)));
	CU_TRY(cudaMalloc((void **) &w.d_cand_ids, points * ef * sizeof(uint32_t)));
	CU_TRY(cudaMalloc((void **) &w.d_cand_d, points * ef * sizeof(float)));
	CU_TRY(cudaMalloc((void **) &w.d_cand_n, points * sizeof(int32_t)));
	CU_TRY(cudaMalloc((void **) &w.d_pairs, points * M * sizeof(uint64_t)));
	CU_TRY(cudaMalloc((void **) &w.d_pairs_sorted, points * M * sizeof(uint64_t)));
	w.cub_bytes = 0;
	cub::DeviceRadixSort::SortKeys(nullptr, w.cub_bytes, w.d_pairs, w.d_pairs_sorted, (int) (points * M));
	CU_TRY(cudaMalloc(&w.d_cub, w.cub_bytes + 256));
	w.cap_points = points;
	w.cap_ef = ef;
	w.cap_m = M;
	return PGEMB_OK;
}

static GraphView graph_view(pgemb_index *idx)
{
	GraphView g;
	g.vectors = idx->d_vectors;
	g.norms = idx->d_norms;
	g.links = idx->d_links;
	g.row_f = idx->row_f;
	g.link_stride = idx->link_stride;
	g.dim = (uint32_t) idx->meta.dim;
	g.M = (uint32_t) idx->meta.M;
	g.maxM = (uint32_t) idx->meta.maxM;
	g.error_flag = idx->d_error;
	return g;
}

// Select: each of `count` new nodes whose candidate lists sit in bind_ws slots [0,count) picks its neighbours and writes its
// (target, source) pairs to bind_ws.d_pairs.  `staged`: the heuristic with its operands staged in shared memory.
static pgemb_status launch_select(pgemb_index *idx, const uint32_t *d_new_ids, size_t count, size_t ef, bool staged, cudaStream_t s)
{
	BindWorkspace  &w = idx->bind_ws;
	const GraphView g = graph_view(idx);
	const size_t	sel_smem = select_smem_bytes(ef, idx->meta.M, idx->row_f, staged);
	return with_metric((int) idx->meta.dist_func, [&](auto m) -> pgemb_status {
		const auto fn = staged ? select_kernel<decltype(m)::value, true> : select_kernel<decltype(m)::value, false>;
		if (sel_smem > 48 * 1024) CU_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sel_smem));
		PGEMB_LAUNCH(fn, (uint32_t) count, kBindThreads, sel_smem, s, g, d_new_ids, w.d_cand_ids, w.d_cand_d, w.d_cand_n, (uint32_t) ef, w.d_pairs);
		g_launches++;
		CU_TRY(cudaGetLastError());
		return PGEMB_OK;
	});
}

// Back-links of the pairs of the first `count` selected nodes: sorted by (target, source), so that every target takes its new
// neighbours in source-id order -- the sequential order.
static pgemb_status launch_backlinks(pgemb_index *idx, size_t count, cudaStream_t s)
{
	BindWorkspace  &w = idx->bind_ws;
	const GraphView g = graph_view(idx);
	const size_t	maxM1 = idx->meta.maxM + 1;
	const size_t	bl_smem = maxM1 * 8 * 2 + (idx->meta.maxM ? idx->meta.maxM : 1) * 8 + maxM1 * 4;
	// m = 0: no node selects a neighbour, so select_kernel wrote no pair slot -- not even a "none" marker -- and there is nothing to apply
	if (idx->meta.M == 0) return PGEMB_OK;
	const uint32_t	n_pairs = (uint32_t) (count * idx->meta.M);
	const uint64_t *sorted = w.d_pairs;
	if (count > 1)
	{
		size_t bytes = w.cub_bytes;
		CU_TRY(cub::DeviceRadixSort::SortKeys(w.d_cub, bytes, w.d_pairs, w.d_pairs_sorted, (int) n_pairs, 0, 64, s));
		g_launches++;
		sorted = w.d_pairs_sorted;
	}
	return with_metric((int) idx->meta.dist_func, [&](auto m) -> pgemb_status {
		if (bl_smem > 48 * 1024) CU_TRY(cudaFuncSetAttribute(backlink_kernel<decltype(m)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bl_smem));
		PGEMB_LAUNCH(backlink_kernel<decltype(m)::value>, n_pairs, kBindThreads, bl_smem, s, g, sorted, n_pairs);
		g_launches++;
		CU_TRY(cudaGetLastError());
		return PGEMB_OK;
	});
}

// Connect `count` new nodes whose candidate lists sit in bind_ws slots [0,count): select + back-links.
static pgemb_status launch_connect(pgemb_index *idx, const uint32_t *d_new_ids, size_t count, size_t ef, cudaStream_t s)
{
	// a handful of inserts (hnsw_bind_point: one): the heuristic with its operands staged in shared memory -- the kept rows
	// must fit next to the key arrays (M = 32 at 768-d: 100 KB); batches keep the small-footprint kernel (many CTAs per SM)
	const size_t M = idx->meta.M ? idx->meta.M : 1;
	const bool	 staged = count <= 8 && M <= 256 && select_smem_bytes(ef, M, idx->row_f, true) <= 200 * 1024 && env_int("PGEMB_SELECT_STAGED", 1) != 0;
	pgemb_status st = launch_select(idx, d_new_ids, count, ef, staged, s);
	if (st) return st;
	return launch_backlinks(idx, count, s);
}

// Search `count` stored nodes (their ids at d_ids) with ef = efc into bind_ws slots [0,count); with_expansions: also record each
// search's expansions for validate_kernel.
static pgemb_status search_stored(pgemb_index *idx, const uint32_t *d_ids, size_t count, size_t efc, cudaStream_t s, bool with_expansions)
{
	BindWorkspace &w = idx->bind_ws;
	SearchRequest  r(count, efc, d_ids, w.d_cand_n);
	r.dists = w.d_cand_d;
	r.ids = w.d_cand_ids;
	if (with_expansions)
	{
		r.exp = w.d_exp;
		r.exp_n = w.d_exp_n;
		r.exp_cap = BindWorkspace::kExpCap;
	}
	return launch_search(idx, r, s);
}

__global__ void iota_kernel(uint32_t *out, uint32_t start, uint32_t n);

pgemb_status bind_points(pgemb_index *idx, idx_t first, size_t n)
{
	if (n == 0) return PGEMB_OK;
	if ((size_t) first + n > idx->n) return fail(PGEMB_ERR_ARG, "bind: nodes not stored");
	const size_t efc = idx->meta.efConstruction;
	if (efc < 1) return fail(PGEMB_ERR_ARG, "efConstruction must be >= 1");
	cudaStream_t s = idx->stream;
	// one bind at a time uses ONE slot of the bind workspace (candidates, pairs); only the ids are per point
	pgemb_status st = ensure_bind_ws(idx, 1, efc);
	if (st) return st;
	if (idx->seq_ids_cap < n)
	{
		cudaFree(idx->d_seq_ids);
		idx->d_seq_ids = nullptr;
		idx->seq_ids_cap = 0;
		CU_TRY(cudaMalloc((void **) &idx->d_seq_ids, n * sizeof(uint32_t)));
		idx->seq_ids_cap = n;
	}
	PGEMB_LAUNCH(iota_kernel, (uint32_t) ((n + 255) / 256), 256, 0, s, idx->d_seq_ids, (uint32_t) first, (uint32_t) n);
	g_launches++;
	CU_TRY(cudaGetLastError());
	// strictly sequential: node i sees the links written for nodes < i (embedding.c:624-629 serialises writers)
	for (size_t i = 0; i < n; i++)
	{
		if (first + i == 0) continue;  // hnswalg.cpp:227-228
		st = search_stored(idx, idx->d_seq_ids + i, 1, efc, s, false);
		if (st) return st;
		st = launch_connect(idx, idx->d_seq_ids + i, 1, efc, s);
		if (st) return st;
	}
	return PGEMB_OK;
}

// device time of a build from start() to finish(); the two events go away on every return path
struct BuildTimer
{
	cudaEvent_t e0 = nullptr, e1 = nullptr;
	cudaError_t start(cudaStream_t s)
	{
		cudaError_t e = cudaEventCreate(&e0);
		if (e == cudaSuccess) e = cudaEventCreate(&e1);
		return e != cudaSuccess ? e : cudaEventRecord(e0, s);
	}
	// the build is enqueued: waits for it, returns the kernels' sticky error and its device seconds in *seconds_out
	pgemb_status finish(pgemb_index *idx, cudaStream_t s, double *seconds_out)
	{
		CU_TRY(cudaEventRecord(e1, s));
		const pgemb_status st = check_device_error(idx, s);
		float ms = 0.f;
		cudaEventElapsedTime(&ms, e0, e1);
		if (seconds_out) *seconds_out = ms * 1e-3;
		return st;
	}
	~BuildTimer()
	{
		if (e0) cudaEventDestroy(e0);
		if (e1) cudaEventDestroy(e1);
	}
};

__global__ void iota_kernel(uint32_t *out, uint32_t start, uint32_t n)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = start + i;
}

extern "C" pgemb_status pgemb_build_bulk(pgemb_index *idx, size_t first, size_t n, size_t batch_max, double *seconds_out)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "build: nodes not stored");
	if (batch_max < 1) batch_max = 1;
	if (batch_max > (1u << 16)) batch_max = 1u << 16;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t efc = idx->meta.efConstruction;
	if (efc < 1) return fail(PGEMB_ERR_ARG, "efConstruction must be >= 1");
	cudaStream_t s = idx->stream;
	st = ensure_bind_ws(idx, batch_max, efc);
	if (st) return st;
	BindWorkspace &w = idx->bind_ws;
	BuildTimer	   timer;
	CU_TRY(timer.start(s));
	size_t pos = first;
	const size_t end = first + n;
	while (pos < end)
	{
		size_t B = pos / 32;  // nodes bound so far = pos
		if (B < 1) B = 1;
		if (B > batch_max) B = batch_max;
		if (B > end - pos) B = end - pos;
		if (pos == 0)
		{
			pos = 1;  // node 0 has nothing to connect to (hnswalg.cpp:227-228)
			continue;
		}
		PGEMB_LAUNCH(iota_kernel, (uint32_t) ((B + 255) / 256), 256, 0, s, w.d_qids, (uint32_t) pos, (uint32_t) B);
		g_launches++;
		st = search_stored(idx, w.d_qids, B, efc, s, false);
		if (st) return st;
		st = launch_connect(idx, w.d_qids, B, efc, s);
		if (st) return st;
		pos += B;
	}
	return timer.finish(idx, s, seconds_out);
}

// Exact AND parallel build: the result is bit-identical to n sequential hnsw_add_point calls (embedding.c:606-701).
// Speculative batches: all inserts of a batch search the graph as it was before the batch (one launch); the
// longest prefix whose searches provably equal the sequential ones (validate_kernel) is connected -- own lists
// + back-links per target in source-id order, which is the sequential order -- and the batch restarts at the
// first conflicting insert.  The first insert of a batch is always valid, so the build always progresses.
// Measured and dropped (profiles/r2_call16_exact_repair.log): redoing each conflicting insert alone and re-validating the rest of
// the batch against its true back-link targets -- bit-identical too (446 fuzzed configurations), but every repair costs a whole
// search latency, which is what a fresh speculative round costs while accepting ~37 inserts: 207-795 us per insert at N ~ 1M
// against 172 us for this restart scheme.
extern "C" pgemb_status pgemb_build_exact(pgemb_index *idx, size_t first, size_t n, size_t batch_max, double *seconds_out,
										  uint64_t *stats_out /* [3]: batches, searches run, inserts */)
{
	if (!idx) return fail(PGEMB_ERR_ARG, "null index");
	if (first + n > idx->n) return fail(PGEMB_ERR_ARG, "build: nodes not stored");
	if (batch_max < 1) batch_max = 1;
	if (batch_max > 4096) batch_max = 4096;
	pgemb_status st = set_device(idx);
	if (st) return st;
	const size_t efc = idx->meta.efConstruction;
	if (efc < 1) return fail(PGEMB_ERR_ARG, "efConstruction must be >= 1");
	cudaStream_t s = idx->stream;
	st = ensure_bind_ws(idx, batch_max, efc);
	if (st) return st;
	BindWorkspace &w = idx->bind_ws;
	const uint32_t ecap = BindWorkspace::kExpCap;
	if (!w.d_exp || w.stamp_cap < idx->capacity)
	{
		cudaFree(w.d_exp); cudaFree(w.d_exp_n); cudaFree(w.d_stamp); cudaFree(w.d_first);
		w.d_exp = w.d_exp_n = w.d_stamp = w.d_first = nullptr;
		CU_TRY(cudaMalloc((void **) &w.d_exp, w.cap_points * (size_t) ecap * 4));
		CU_TRY(cudaMalloc((void **) &w.d_exp_n, w.cap_points * 4));
		CU_TRY(cudaMalloc((void **) &w.d_stamp, idx->capacity * 4));
		CU_TRY(cudaMalloc((void **) &w.d_first, 4));
		CU_TRY(cudaMemset(w.d_stamp, 0xff, idx->capacity * 4));
		w.stamp_cap = idx->capacity;
	}
	const size_t M = idx->meta.M ? idx->meta.M : 1;
	BuildTimer	 timer;
	CU_TRY(timer.start(s));
	size_t	 pos = first;
	const size_t end = first + n;
	size_t	 B = 1;
	uint64_t batches = 0, searches = 0;
	while (pos < end)
	{
		if (pos == 0)
		{
			pos = 1;  // node 0 has nothing to connect to (hnswalg.cpp:227-228)
			continue;
		}
		if (B > batch_max) B = batch_max;
		if (B > end - pos) B = end - pos;
		PGEMB_LAUNCH(iota_kernel, (uint32_t) ((B + 255) / 256), 256, 0, s, w.d_qids, (uint32_t) pos, (uint32_t) B);
		g_launches++;
		st = search_stored(idx, w.d_qids, B, efc, s, true);
		if (st) return st;
		batches++;
		searches += B;
		size_t acc = B;
		// the small-footprint select at every batch size (launch_connect stages batches of up to 8)
		st = launch_select(idx, w.d_qids, B, efc, false, s);
		if (st) return st;
		const uint32_t n_pairs_all = (uint32_t) (B * M);
		// m = 0: no back-links, so no search of the batch can conflict with an earlier insert (and no pair slot was written)
		if (B > 1 && idx->meta.M > 0)
		{
			uint32_t hfirst = (uint32_t) B;
			CU_TRY(cudaMemcpyAsync(w.d_first, &hfirst, 4, cudaMemcpyHostToDevice, s));
			PGEMB_LAUNCH(stamp_targets_kernel, (n_pairs_all + 255) / 256, 256, 0, s, w.d_pairs, n_pairs_all, w.d_stamp);
			PGEMB_LAUNCH(validate_kernel, (uint32_t) ((B * 32 + 255) / 256), 256, 0, s, w.d_exp, w.d_exp_n, ecap, w.d_qids, (uint32_t) B, w.d_stamp, w.d_first);
			PGEMB_LAUNCH(clear_stamps_kernel, (n_pairs_all + 255) / 256, 256, 0, s, w.d_pairs, n_pairs_all, w.d_stamp);
			g_launches += 3;
			CU_TRY(cudaMemcpyAsync(&hfirst, w.d_first, 4, cudaMemcpyDeviceToHost, s));
			CU_TRY(cudaStreamSynchronize(s));
			acc = hfirst < B ? hfirst : B;
			if (acc < 1) acc = 1;
			if (acc < B)
			{
				PGEMB_LAUNCH(zero_links_kernel, (uint32_t) (B - acc), 64, 0, s, idx->d_links, idx->link_stride, w.d_qids + acc, (uint32_t) (B - acc));
				g_launches++;
			}
		}
		// back-links of the accepted prefix
		st = launch_backlinks(idx, acc, s);
		if (st) return st;
		pos += acc;
		// Speculative searches are nearly free (one launch, one warp each, latency-bound), so the batch only
		// shrinks while the graph is tiny (every search expands most of it and everything conflicts).
		B = (acc == B) ? B * 2 : (acc * 8 > batch_max ? batch_max : acc * 8 + 1);
		// a batch that would only slightly exceed one query per SM is cut to one query per SM, so that the speculative
		// searches run in latency mode (a CTA per search: shorter round) -- the accepted prefix is far shorter than the
		// batch anyway (measured: 209 -> 183 us per insert at N ~ 1M).  Same result by construction (any batch size gives
		// the sequential graph).
		if (env_int("PGEMB_EXACT_CLAMP_SMS", 1) != 0 && B > (size_t) idx->sm_count && B <= 3 * (size_t) idx->sm_count) B = (size_t) idx->sm_count;
	}
	if (stats_out)
	{
		stats_out[0] = batches;
		stats_out[1] = searches;
		stats_out[2] = n;
	}
	return timer.finish(idx, s, seconds_out);
}

// ------------------------------------------------------------------------------------------------
// shard merge (K5) and the peer-memory exchange (SURVEY.md 8(e))
// ------------------------------------------------------------------------------------------------
static pgemb_status launch_merge(size_t nq, size_t n_shards, size_t k, const ShardLists &in, const uint32_t *d_flags, uint32_t seq, uint32_t self,
								 dist_t *d_dists_out, label_t *d_labels_out, int32_t *d_n_out, int *d_error, cudaStream_t s)
{
	const uint32_t threads = 128;
	const uint32_t blocks = (uint32_t) ((nq * 32 + threads - 1) / threads);
	PGEMB_LAUNCH(merge_topk_lists_kernel, blocks, threads, 0, s, (uint32_t) nq, (uint32_t) n_shards, (uint32_t) k, in, d_flags, seq, self, d_dists_out,
				 d_labels_out, d_n_out, d_error);
	g_launches++;
	CU_TRY(cudaGetLastError());
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_merge_topk_device(size_t nq, size_t n_shards, size_t k, const dist_t *d_dists_in, const label_t *d_labels_in,
												const int32_t *d_n_in, dist_t *d_dists_out, label_t *d_labels_out, int32_t *d_n_out,
												void *stream)
{
	if (nq == 0) return PGEMB_OK;
	if (!d_dists_in || !d_labels_in || !d_n_in || !d_dists_out || !d_labels_out || !d_n_out) return fail(PGEMB_ERR_ARG, "null argument");
	if (n_shards == 0 || k == 0) return fail(PGEMB_ERR_ARG, "n_shards and k must be > 0");
	if (n_shards > kMaxShards) return fail(PGEMB_ERR_ARG, "at most 16 shards");
	ShardLists in;
	memset(&in, 0, sizeof(in));
	for (size_t s = 0; s < n_shards; s++)  // input layout: [shard][query][k]
	{
		in.dist[s] = d_dists_in + s * nq * k;
		in.lab[s] = d_labels_in + s * nq * k;
		in.cnt[s] = d_n_in + s * nq;
	}
	return launch_merge(nq, n_shards, k, in, nullptr, 0, 0, d_dists_out, d_labels_out, d_n_out, nullptr, (cudaStream_t) stream);
}

// One packed result buffer per rank: [labels u64 nq*k | dists f32 nq*k | counts i32 nq] -- what ONE all-gather moves.
struct PackedTopk
{
	uint64_t *labels;
	float	 *dists;
	int32_t	 *counts;
};

static PackedTopk packed_topk(const void *base, size_t nq, size_t k)
{
	char *b = (char *) base;
	return {(uint64_t *) b, (float *) (b + nq * k * 8), (int32_t *) (b + nq * k * 12)};
}

// a packed buffer as one input of the merge kernel
static void set_shard(ShardLists &in, size_t shard, const void *base, size_t nq, size_t k)
{
	const PackedTopk p = packed_topk(base, nq, k);
	in.lab[shard] = p.labels;
	in.dist[shard] = p.dists;
	in.cnt[shard] = p.counts;
}

extern "C" size_t pgemb_packed_topk_bytes(size_t nq, size_t k) { return nq * k * 12 + nq * 4; }

extern "C" pgemb_status pgemb_merge_topk_packed_device(size_t nq, size_t n_shards, size_t k, const void *d_packed, size_t shard_stride_bytes,
													   dist_t *d_dists_out, label_t *d_labels_out, int32_t *d_n_out, void *stream)
{
	if (nq == 0) return PGEMB_OK;
	if (!d_packed || !d_dists_out || !d_labels_out || !d_n_out) return fail(PGEMB_ERR_ARG, "null argument");
	if (n_shards == 0 || k == 0 || n_shards > kMaxShards) return fail(PGEMB_ERR_ARG, "n_shards must be in 1..16 and k > 0");
	if (shard_stride_bytes < pgemb_packed_topk_bytes(nq, k) || (shard_stride_bytes & 7)) return fail(PGEMB_ERR_ARG, "bad shard stride");
	ShardLists in;
	memset(&in, 0, sizeof(in));
	for (size_t s = 0; s < n_shards; s++) set_shard(in, s, (const char *) d_packed + s * shard_stride_bytes, nq, k);
	return launch_merge(nq, n_shards, k, in, nullptr, 0, 0, d_dists_out, d_labels_out, d_n_out, nullptr, (cudaStream_t) stream);
}

// ---- peer-memory exchange: no collective at all ------------------------------------------------------------------
// Every rank owns one buffer: two result areas (step parity) in the packed layout above + a flag word per peer.  A step is
//   pgemb_sharded_search_device   the local search writes its top-k into this rank's area of the step's parity; then, in
//                                 stream order, the rank's sequence number is stored into EVERY peer's flag array (4-byte
//                                 copies by the copy engine over NVLink: no kernel, no collective);
//   pgemb_sharded_merge_device    ONE kernel: waits until all peers' flags show this step, then reads the peers' lists
//                                 straight from their memory (peer-mapped / CUDA-IPC pointers) and merges.
// Two parities are enough: a peer that is still reading my area of step s cannot have published s + 1, and my search of
// step s + 2 (which overwrites that area) is stream-ordered after my merge of s + 1, which waited for that flag.
struct pgemb_exchange
{
	int		 device = 0, rank = 0, world = 1;
	size_t	 max_nq = 0, k = 0;
	size_t	 area_bytes = 0, off_flags = 0, total_bytes = 0;
	char	*d_buf = nullptr;
	char	*peer[kMaxShards] = {};
	bool	 peer_ipc[kMaxShards] = {};
	bool	 attached = false;
	uint32_t seq = 0;
	uint32_t *h_seq = nullptr;	// pinned ring: the values the flag copies read
	int		 *d_error = nullptr;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	bool	 ev_valid = false;
};

extern "C" pgemb_status pgemb_exchange_create(int device, int rank, int world, size_t max_nq, size_t k, pgemb_exchange **out)
{
	if (!out) return fail(PGEMB_ERR_ARG, "null argument");
	if (world < 1 || world > (int) kMaxShards || rank < 0 || rank >= world) return fail(PGEMB_ERR_ARG, "rank/world out of range (world <= 16)");
	if (max_nq == 0 || k == 0) return fail(PGEMB_ERR_ARG, "max_nq and k must be > 0");
	CU_TRY(cudaSetDevice(device));
	pgemb_exchange *ex = new (std::nothrow) pgemb_exchange();
	if (!ex) return fail(PGEMB_ERR_NOMEM, "out of host memory");
	ex->device = device;
	ex->rank = rank;
	ex->world = world;
	ex->max_nq = max_nq;
	ex->k = k;
	ex->area_bytes = (pgemb_packed_topk_bytes(max_nq, k) + 255) & ~(size_t) 255;
	ex->off_flags = 2 * ex->area_bytes;
	ex->total_bytes = ex->off_flags + 256;
	cudaError_t e = cudaMalloc((void **) &ex->d_buf, ex->total_bytes);
	if (e == cudaSuccess) e = cudaMemset(ex->d_buf, 0, ex->total_bytes);
	if (e == cudaSuccess) e = cudaMallocHost((void **) &ex->h_seq, 64 * sizeof(uint32_t));
	if (e == cudaSuccess) e = cudaMalloc((void **) &ex->d_error, sizeof(int));
	if (e == cudaSuccess) e = cudaMemset(ex->d_error, 0, sizeof(int));
	if (e == cudaSuccess) e = cudaEventCreate(&ex->ev0);
	if (e == cudaSuccess) e = cudaEventCreate(&ex->ev1);
	if (e == cudaSuccess) e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
	{
		pgemb_exchange_destroy(ex);
		return fail(PGEMB_ERR_CUDA, std::string("pgemb_exchange_create: ") + cudaGetErrorString(e));
	}
	ex->peer[rank] = ex->d_buf;
	*out = ex;
	return PGEMB_OK;
}

extern "C" void pgemb_exchange_destroy(pgemb_exchange *ex)
{
	if (!ex) return;
	cudaSetDevice(ex->device);
	cudaDeviceSynchronize();
#ifndef PGEMB_HOST_EMULATION
	for (int r = 0; r < ex->world; r++)
		if (r != ex->rank && ex->peer[r] && ex->peer_ipc[r]) cudaIpcCloseMemHandle(ex->peer[r]);
#endif
	cudaFree(ex->d_buf);
	cudaFree(ex->d_error);
	if (ex->h_seq) cudaFreeHost(ex->h_seq);
	if (ex->ev0) cudaEventDestroy(ex->ev0);
	if (ex->ev1) cudaEventDestroy(ex->ev1);
	cudaGetLastError();
	delete ex;
}

// 64-byte handle of this rank's buffer for the other PROCESSES (exchange it out of band: torch.distributed all_gather, a pipe ...)
extern "C" pgemb_status pgemb_exchange_handle(pgemb_exchange *ex, void *handle_out)
{
	if (!ex || !handle_out) return fail(PGEMB_ERR_ARG, "null argument");
#ifdef PGEMB_HOST_EMULATION
	memset(handle_out, 0, PGEMB_IPC_HANDLE_BYTES);
	memcpy(handle_out, &ex->d_buf, sizeof(void *));
#else
	static_assert(sizeof(cudaIpcMemHandle_t) == PGEMB_IPC_HANDLE_BYTES, "CUDA IPC handle size");
	CU_TRY(cudaSetDevice(ex->device));
	cudaIpcMemHandle_t h;
	CU_TRY(cudaIpcGetMemHandle(&h, ex->d_buf));
	memcpy(handle_out, &h, sizeof(h));
#endif
	return PGEMB_OK;
}

// the raw device pointer, for attaching ranks that live in the SAME process (one process driving several GPUs)
extern "C" void *pgemb_exchange_buffer(pgemb_exchange *ex) { return ex ? ex->d_buf : nullptr; }

extern "C" pgemb_status pgemb_exchange_attach(pgemb_exchange *ex, const void *handles, int same_process)
{
	if (!ex || !handles) return fail(PGEMB_ERR_ARG, "null argument");
	CU_TRY(cudaSetDevice(ex->device));
	for (int r = 0; r < ex->world; r++)
	{
		if (r == ex->rank) continue;
		const char *h = (const char *) handles + (size_t) r * PGEMB_IPC_HANDLE_BYTES;
		if (same_process)
		{
			void *ptr = nullptr;
			memcpy(&ptr, h, sizeof(void *));
			if (!ptr) return fail(PGEMB_ERR_ARG, "null peer buffer");
#ifndef PGEMB_HOST_EMULATION
			cudaPointerAttributes at;
			CU_TRY(cudaPointerGetAttributes(&at, ptr));
			if (at.device != ex->device)
			{
				const cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
				if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(PGEMB_ERR_CUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
				cudaGetLastError();
			}
#endif
			ex->peer[r] = (char *) ptr;
			ex->peer_ipc[r] = false;
		}
		else
		{
#ifdef PGEMB_HOST_EMULATION
			return fail(PGEMB_ERR_ARG, "the host emulation has no other processes");
#else
			cudaIpcMemHandle_t hh;
			memcpy(&hh, h, sizeof(hh));
			void *ptr = nullptr;
			CU_TRY(cudaIpcOpenMemHandle(&ptr, hh, cudaIpcMemLazyEnablePeerAccess));
			ex->peer[r] = (char *) ptr;
			ex->peer_ipc[r] = true;
#endif
		}
	}
	ex->attached = true;
	return PGEMB_OK;
}

// the result area of step `seq` in `buf` (this rank's buffer or a peer's): the step's parity picks one of the two
static char *step_area(const pgemb_exchange *ex, char *buf, uint32_t seq) { return buf + (size_t) (seq & 1u) * ex->area_bytes; }

// arguments of a local step; `k_name` is what the entry point calls its k
static pgemb_status check_local_step(const pgemb_index *idx, const pgemb_exchange *ex, size_t nq, size_t k, const char *k_name)
{
	if (!idx || !ex) return fail(PGEMB_ERR_ARG, "null argument");
	if (ex->world > 1 && !ex->attached) return fail(PGEMB_ERR_STATE, "pgemb_exchange_attach has not been called");
	if (k != ex->k) return fail(PGEMB_ERR_ARG, std::string(k_name) + " differs from the exchange's k");
	if (nq == 0 || nq > ex->max_nq) return fail(PGEMB_ERR_ARG, "nq out of range for this exchange");
	if (idx->device != ex->device) return fail(PGEMB_ERR_ARG, "index and exchange live on different devices");
	return PGEMB_OK;
}

// The local step has been enqueued: advance the sequence number and store it into every peer's flag array, after the step in
// stream order.
static pgemb_status publish_step(pgemb_exchange *ex, cudaStream_t s)
{
	ex->seq += 1;
	uint32_t *src = &ex->h_seq[ex->seq & 63u];
	*src = ex->seq;
	for (int r = 0; r < ex->world; r++)
	{
		if (r == ex->rank) continue;
		CU_TRY(cudaMemcpyAsync(ex->peer[r] + ex->off_flags + (size_t) ex->rank * 4, src, 4, cudaMemcpyHostToDevice, s));
	}
	return PGEMB_OK;
}

extern "C" pgemb_status pgemb_sharded_search_device(pgemb_index *idx, pgemb_exchange *ex, size_t nq, const coord_t *d_queries, size_t ef, void *stream)
{
	pgemb_status st = check_local_step(idx, ex, nq, ef, "ef");
	if (st) return st;
	const PackedTopk out = packed_topk(step_area(ex, ex->d_buf, ex->seq + 1), nq, ex->k);
	SearchRequest r(nq, ef, d_queries, out.counts);
	r.labels = out.labels;
	r.dists = out.dists;
	st = launch_search(idx, r, (cudaStream_t) stream);
	if (st) return st;
	return publish_step(ex, (cudaStream_t) stream);
}

// The brute-force scan as the local step of a sharded exchange (BASELINE configs[4]: every rank scans its id range for the whole
// query batch): results land in this rank's result area, then the step is published to the peers exactly as a traversal's is.
extern "C" pgemb_status pgemb_sharded_scan_device(pgemb_index *idx, pgemb_exchange *ex, size_t nq, const coord_t *d_queries, size_t k, void *stream)
{
	pgemb_status st = check_local_step(idx, ex, nq, k, "k");
	if (st) return st;
	const PackedTopk out = packed_topk(step_area(ex, ex->d_buf, ex->seq + 1), nq, ex->k);
	st = pgemb_scan_topk_device(idx, nq, d_queries, k, out.labels, out.dists, out.counts, stream);
	if (st) return st;
	return publish_step(ex, (cudaStream_t) stream);
}

extern "C" pgemb_status pgemb_sharded_merge_device(pgemb_exchange *ex, size_t nq, label_t *d_labels_out, dist_t *d_dists_out, int32_t *d_n_out, void *stream)
{
	if (!ex || !d_labels_out || !d_dists_out || !d_n_out) return fail(PGEMB_ERR_ARG, "null argument");
	if (nq == 0 || nq > ex->max_nq) return fail(PGEMB_ERR_ARG, "nq out of range for this exchange");
	if (ex->seq == 0) return fail(PGEMB_ERR_STATE, "no search step to merge");
	CU_TRY(cudaSetDevice(ex->device));
	cudaStream_t s = (cudaStream_t) stream;
	ShardLists	 in;
	memset(&in, 0, sizeof(in));
	for (int r = 0; r < ex->world; r++) set_shard(in, (size_t) r, step_area(ex, ex->peer[r], ex->seq), nq, ex->k);
	CU_TRY(cudaEventRecord(ex->ev0, s));
	pgemb_status st = launch_merge(nq, (size_t) ex->world, ex->k, in, ex->world > 1 ? (const uint32_t *) (ex->d_buf + ex->off_flags) : nullptr, ex->seq,
								   (uint32_t) ex->rank, d_dists_out, d_labels_out, d_n_out, ex->d_error, s);
	if (st) return st;
	CU_TRY(cudaEventRecord(ex->ev1, s));
	ex->ev_valid = true;
	return PGEMB_OK;
}

// device time (ms) of the last wait+merge kernel (includes waiting for the slowest peer); <0 if unavailable
extern "C" float pgemb_exchange_last_merge_ms(pgemb_exchange *ex)
{
	if (!ex || !ex->ev_valid) return -1.0f;
	float ms = -1.0f;
	if (cudaSetDevice(ex->device) != cudaSuccess || cudaEventSynchronize(ex->ev1) != cudaSuccess || cudaEventElapsedTime(&ms, ex->ev0, ex->ev1) != cudaSuccess) return -1.0f;
	return ms;
}

// 0 = fine; 5 = a peer never published its step within the kernel's patience
extern "C" int pgemb_exchange_error(pgemb_exchange *ex)
{
	if (!ex) return -1;
	int err = 0;
	if (cudaSetDevice(ex->device) != cudaSuccess || cudaMemcpy(&err, ex->d_error, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
	return err;
}
