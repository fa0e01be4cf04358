/*
 * graphsage_b200.h - C-ABI of libgraphsage_b200.so (sm_90a, H100).
 *
 * The reference (williamleif/GraphSAGE) has NO FFI boundary: its hot path is python
 * classes composing TensorFlow library ops.  Each entry point below therefore names the
 * TF op sequence (reference file:line) it replaces; the python classes that keep the
 * reference's surface (graphsage_b200/{neigh_samplers,aggregators,models}.py) bind these
 * through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - Pointers are DEVICE pointers unless the name ends in _host.  Row-major.  "pitch"/"ld"
 *     are in ELEMENTS.  The library never synchronises: every call only enqueues work on `stream`
 *     (a cudaStream_t passed as void*).  It never allocates device memory either, with one exception:
 *     gs_shard_alloc/gs_shard_free (cudaMalloc'd buffers that can be exported through CUDA IPC).
 *   - Return value: 0 = OK, <0 = gs_status error; gs_last_error_string() (thread-local, host)
 *     describes the last failure.  No exceptions cross the boundary.
 *   - There is no CPU fallback: without a CUDA device every compute entry returns GS_ERR_CUDA.
 */
#ifndef GRAPHSAGE_B200_H_
#define GRAPHSAGE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_ABI_VERSION 2

typedef enum {
  GS_OK = 0,
  GS_ERR_INVALID_ARG = -1,
  GS_ERR_CUDA = -2,
  GS_ERR_UNSUPPORTED = -3
} gs_status;

typedef enum { GS_F32 = 0, GS_BF16 = 1, GS_F64 = 2, GS_I8ROW = 3 } gs_dtype;   /* GS_F64: gs_sgd_fit's X only */

/* GS_I8ROW - an int8 feature table with one fp32 scale per row (graphsage_b200.Int8Features; numpy restatement in
 * oracle/int8_rows.py).  Each row is a byte array of `pitch` bytes, the scale stored inside it, so routines that copy rows
 * by bytes (gs_host_fetch, bulk row copies) move int8 rows unchanged:
 *   bytes [0, F)           q_c   int8
 *   bytes [F, P4)          zero                      P4 = round_up(F, 4)
 *   bytes [P4, P4 + 4)     s     fp32, little-endian
 *   bytes [P4 + 4, pitch)  zero                      pitch = gs_i8row_pitch(F) = round_up(P4 + 4, 16)
 * Quantise (gs_quantize_rows_i8): a = max_c |x_c|, s = fl(a / 127); if s == 0 every q_c = 0 (an all-zero row - the dummy
 * row N - has s = 0 and zero bytes), else q_c = clamp(rint_half_even(fl(x_c / s)), -127, 127).  Non-finite input is the
 * caller's to refuse.  Dequantise: deq_c = fl(float(q_c) * s), one fp32 rounding.  Every kernel that reads GS_I8ROW rows
 * (gs_gather_mean, gs_gather_rows_f32, gs_sage_layer_small_i8) sees exactly deq and from there computes what its fp32
 * form computes on the table deq: the same bits.  Where such a call takes a `pitch`, it counts bytes. */
int64_t gs_i8row_pitch(int32_t F);
/* fp32 rows x [n, F] (row stride ldx floats) -> GS_I8ROW rows out [n, out_pitch_bytes] (out_pitch_bytes % 16 == 0 and
 * >= gs_i8row_pitch(F); bytes past the row are zeroed).  One warp per row. */
int32_t gs_quantize_rows_i8(const float* x, int64_t n, int32_t F, int64_t ldx, void* out, int64_t out_pitch_bytes,
                            void* stream);
typedef enum { GS_ACT_NONE = 0, GS_ACT_RELU = 1 } gs_act;
/* how the neighbour part and the self part are combined */
typedef enum {
  GS_COMBINE_ADD = 0,    /* tf.add_n([from_self, from_neighs])      aggregators.py:55-56 */
  GS_COMBINE_CONCAT = 1  /* tf.concat([from_self, from_neighs], 1)  aggregators.py:57-58 */
} gs_combine;
/* arithmetic of the dense contraction */
typedef enum {
  GS_MATH_FP32_SIMT = 0,  /* fp32 FFMA on CUDA cores (bring-up / cross-check path)          */
  GS_MATH_TF32X3 = 1,     /* wgmma tf32, 3-term hi/lo split, fp32 accumulate                 */
  GS_MATH_TF32 = 2,       /* wgmma tf32 single pass                                          */
  GS_MATH_BF16 = 3        /* wgmma bf16 operands, fp32 accumulate                            */
} gs_math;

int32_t gs_version(void);
const char* gs_last_error_string(void);
/* Tuning knobs for experiments; returns the previous value.  Keys (default):
 *   gather_variant (2)      gs_gather_mean / gs_gather_rows: 2 grouped double-buffered TMA, 1 whole-node TMA, 0 LDG
 *   gather_ctas_per_sm (8)  grid cap of the LDG / simple gather kernels
 *   halo_fetch_ctas_per_sm (2)  grid of gs_halo_fetch
 *   k4_operands (1)         gs_maxpool/meanpool_mlp_fused: 1 = gathered rows are the wgmma A operand, 0 = the weight slice is
 *                           A and the gathered rows are B
 *   k4_tile (128)           rows per K4 tile: 128 (fanout <= 128) or 256 (fanout <= 256)
 *   k4_mma_depth (1)        wgmma groups in flight in the K4 K loop (1 or 2)
 *   k4_producer (0)         K4 row gather: 0 = cp.async 16-byte pieces, 1 = register-staged 128-bit loads
 *   k4_cluster (0)          launch a tile's hidden slices as a thread-block cluster of this size (-1 = all slices; clamped to
 *                           a divisor of hidden / 128 that is <= 8; 0 = no clusters)
 * Every K4 configuration the tests name is parity-tested (tests/test_gpu_parity.py: K4_VARIANTS).
 * The Python host also reads them from the environment: GS_TUNING="key=value,key=value". */
int32_t gs_set_tuning(const char* key, int32_t value);

/* ---------------------------------------------------------------------------------------------
 * UniformNeighborSampler._call           reference graphsage/neigh_samplers.py:24-29
 *   out[i, j] = adj[ids[i], pi[j]], j < k, ONE column permutation pi per call.
 *   pi = col_perm (device int32[>=k]) if non-null, else the on-device Philox4x32-10 forward
 *   Fisher-Yates prefix of (seed, counter + (counter_dev ? *counter_dev : 0)) - bit-identical to
 *   oracle/sampler.py:perm_prefix.  ids outside [0, n_rows) read the dummy row n_rows-1.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_sample_padded(const int32_t* adj, int64_t n_rows, int32_t max_deg,
                         const int32_t* ids, int64_t n, int32_t k,
                         const int32_t* col_perm, uint64_t seed, uint64_t counter,
                         const uint64_t* counter_dev, int32_t* out, void* stream);

/* SampleAndAggregate.sample - the whole frontier expansion (reference graphsage/models.py:254-275) in
 * ONE launch: hop t (t = 1..n_hops) is sample_padded(samples[t-1], fanout[t-1]) with RNG counter
 * counter + t - 1 (fanout[] is in HOP order, i.e. reversed layer order: {10, 25} for samples_1=25,
 * samples_2=10).  out[t-1] receives the B*fanout[0]*...*fanout[t-1] ids of hop t (row-major nested).
 * Bit-identical to n_hops successive gs_sample_padded calls.  n_hops <= GS_MAX_HOPS. */
#define GS_MAX_HOPS 4
int32_t gs_sample_padded_khop(const int32_t* adj, int64_t n_rows, int32_t max_deg,
                              const int32_t* seeds, int64_t n_seeds, const int32_t* fanout_host,
                              int32_t n_hops, uint64_t seed, uint64_t counter,
                              const uint64_t* counter_dev, int32_t* const* out_host, void* stream);

/* WeightedNeighborSampler - fixed-fanout draws with replacement in proportion to a per-entry weight, from per-row
 * alias tables (contract: oracle/alias_sampling.py, bit for bit).
 * gs_csr_alias_build - the table: one 16-byte record (thr, id, alias, 0) per CSR entry, int32 table[n_entries * 4]
 *   aligned with indices (row v's d buckets at indptr[v] ..).  weights: fp32, one per entry; finite w > 0 is eligible,
 *   a row with +inf entries draws uniformly among them, a row with none eligible draws the dummy n_nodes.  Integer
 *   masses summing to d 2^32 per row (every eligible entry >= 1) and an integer Vose sweep, both in a fixed order.
 *   Rows of 2^31 entries or more: GS_ERR_UNSUPPORTED.  Set-up work; deterministic, no atomics, no allocation on the
 *   device.
 * gs_sample_alias - out[t * k + j] (k <= GS_MAX_ALIAS_FANOUT) = draw j of ids[t]: Philox4x32-10 block
 *   (c_lo, c_hi, t, 0x90000000 + (j >> 1)) with c = counter + (counter_dev ? *counter_dev : 0), words (0, 1) for even j,
 *   (2, 3) for odd j: bucket = mulhi32(a, d), id if b < thr else alias.  ids outside [0, n_nodes) and empty rows give
 *   n_nodes.
 * gs_sample_alias_khop - every hop of SampleAndAggregate.sample in one launch (n_hops <= GS_MAX_HOPS, fanout <= 64),
 *   byte-identical to n_hops gs_sample_alias calls with counters counter, counter + 1, ... */
#define GS_MAX_ALIAS_FANOUT 1024
int32_t gs_csr_alias_build(const int64_t* indptr, const int32_t* indices, const float* weights, int64_t n_nodes,
                           int64_t n_entries, int32_t* table, void* stream);
int32_t gs_sample_alias(const int64_t* indptr, const int32_t* table, int64_t n_nodes, const int32_t* ids, int64_t n,
                        int32_t k, uint64_t seed, uint64_t counter, const uint64_t* counter_dev, int32_t* out,
                        void* stream);
int32_t gs_sample_alias_khop(const int64_t* indptr, const int32_t* table, int64_t n_nodes, const int32_t* seeds,
                             int64_t n_seeds, const int32_t* fanout_host, int32_t n_hops, uint64_t seed,
                             uint64_t counter, const uint64_t* counter_dev, int32_t* const* out_host, void* stream);

/* Per-node draws from a CSR adjacency (north_star's warp-per-node mode; no reference
 * counterpart).  Semantics: oracle/sampler.py:sample_csr.  k <= 32. */
int32_t gs_sample_csr(const int64_t* indptr, const int32_t* indices, int64_t n_nodes,
                      const int32_t* ids, int64_t n, int32_t k, int32_t replace_if_short,
                      uint64_t seed, uint64_t counter, const uint64_t* counter_dev,
                      int32_t pad_id, int32_t* out, void* stream);

/* tf.nn.fixed_unigram_candidate_sampler(unique=False)   reference graphsage/models.py:336-343
 *   num_sampled ids drawn with replacement with probability proportional to the weights behind `cdf`
 *   (cdf[i] = sum_{j<=i} deg[j]^0.75, float64, non-decreasing, length n).  Draw j uses word j&3 of
 *   Philox4x32-10 block (counter, c2 = 0, GS unigram stream tag + j>>2): u = (draw + 0.5) / 2^32 * cdf[n-1],
 *   out[j] = first index with cdf[index] > u (oracle/sampler.py:sample_unigram; TF's own stream is unobtainable). */
int32_t gs_sample_unigram(const double* cdf, int64_t n, int32_t num_sampled, uint64_t seed, uint64_t counter,
                          const uint64_t* counter_dev, int32_t* out, void* stream);

/* tf.nn.fixed_unigram_candidate_sampler(unique=True)   reference graphsage/models.py:450-457 (Node2VecModel)
 *   num_sampled DISTINCT ids: the first num_sampled distinct ids of the draw sequence, in draw order - TF draws in sequence
 *   and rejects ids it already holds.  Draw j (j = 0, 1, ...) maps to an id by the rule of gs_sample_unigram, with word j&3
 *   of Philox4x32-10 block (counter + (counter_dev ? *counter_dev : 0), c2 = 0, GS unique-unigram stream tag + j>>2)
 *   (oracle/node2vec.py:sample_unigram_unique).  The true classes do not change which ids are drawn.
 *   Limits: num_sampled <= GS_MAX_UNIQUE_SAMPLED and <= n.  The caller must not ask for more ids than have positive weight
 *   (the Python host refuses it); the kernel stops after GS_UNIQUE_DRAW_BUDGET draws in any case: positions it could not
 *   fill are -1 and *status (device int32, may be NULL; never cleared by the kernel) is set to 1.  One warp, no host sync. */
#define GS_MAX_UNIQUE_SAMPLED 1024
#define GS_UNIQUE_DRAW_BUDGET (1 << 20)
int32_t gs_sample_unigram_unique(const double* cdf, int64_t n, int32_t num_sampled, uint64_t seed, uint64_t counter,
                                 const uint64_t* counter_dev, int32_t* out, int32_t* status, void* stream);

/* Device-side construction of the padded adjacency table from CSR (the sampler's input contract, reference
 * graphsage/minibatch.py:227-259; SURVEY section 8f row 3).  adj is [n_nodes + 1, max_deg] int32:
 *   row n_nodes (dummy) and rows of skipped nodes (skip[u] != 0: val/test nodes, minibatch.py:232-233) or of
 *   nodes without neighbours = n_nodes;  deg == max_deg: the neighbours in CSR order;
 *   deg <  max_deg: max_deg draws WITH replacement (minibatch.py:242-243);
 *   deg >  max_deg: max_deg distinct neighbours (Floyd's algorithm; minibatch.py:240-241).
 * Draw j of node u is word j&3 of Philox block (counter, c2 = u, build tag + j>>2)  (oracle/adjacency.py:
 * build_padded_adj; the reference's numpy RandomState stream is reproduced by the HOST builder
 * graphsage_b200/minibatch.py instead).  max_deg <= 1024.  deg (float32 [n_nodes], may be NULL) receives the
 * neighbour counts (minibatch.py:237). */
int32_t gs_build_padded_adj(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int32_t max_deg,
                            const uint8_t* skip, uint64_t seed, uint64_t counter, int32_t* adj, float* deg,
                            void* stream);

/* host helper: the first k entries of pi for (seed, counter) - what the kernel computes */
int32_t gs_perm_prefix_host(uint64_t seed, uint64_t counter, int32_t max_deg, int32_t k,
                            int32_t* out_host);

/* ---------------------------------------------------------------------------------------------
 * tf.nn.embedding_lookup(features, ids)   reference graphsage/models.py:299
 *   out[i, 0:F] = feats[ids[i], 0:F].  When row bytes are 16-B multiples and pointers 16-B
 *   aligned the copy is staged global->shared->global by the TMA bulk-copy engine.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_gather_rows(const void* feats, int32_t dtype, int64_t n_rows, int32_t F,
                       int64_t pitch, const int32_t* ids, int64_t n, void* out,
                       int64_t out_pitch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused K-hop gather + fixed-fanout segmented mean:
 *   tf.nn.embedding_lookup (models.py:299) + tf.reduce_mean(neigh_vecs, axis=1)
 *   (aggregators.py:48), or the GCN form mean(concat([neigh, self]))  (aggregators.py:106-107),
 *   without materialising the [n*k, F] neighbour tensor.
 * A call processes up to GS_MAX_SEGMENTS segments (one per hop) in one launch.  For segment s,
 * output row r = out_row0 + i (i < n):
 *   neigh row j of i = src[neigh_ids ? neigh_ids[i*k + j] : neigh_row0 + i*k + j]
 *   self  row   of i = src[self_ids  ? self_ids[i]        : self_row0 + i]
 *   out_mean[r] = (sum_j neigh_j (+ self if include_self)) / (k (+1 if include_self))
 *   out_self[r] = self row (only if out_self != NULL)
 * src is [n_src_rows, F] with `pitch`; F columns are produced, columns F..out_pitch-1 are zeroed.
 * dtype GS_F32, or GS_BF16: a bfloat16 table (rows 16-byte multiples: pitch % 8 == 0, out_pitch % 8 == 0) summed in fp32 -
 * the outputs stay fp32 and equal the fp32 kernel's on the bf16-rounded table (half the gathered bytes); or GS_I8ROW
 * (pitch in bytes, % 16 == 0, >= gs_i8row_pitch(F); out_pitch % 8 == 0 and <= 1536): whole rows by bulk copy, dequantised
 * in registers - the fp32 kernel's outputs on the dequantised table (a quarter of the fp32 bytes).
 * --------------------------------------------------------------------------------------------- */
#define GS_MAX_SEGMENTS 4
typedef struct {
  const int32_t* self_ids;   /* device, may be NULL */
  const int32_t* neigh_ids;  /* device, may be NULL */
  int64_t self_row0;
  int64_t neigh_row0;
  int64_t n;
  int32_t k;
  int32_t _pad;
  int64_t out_row0;
} gs_segment;

int32_t gs_gather_mean(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                       const gs_segment* segments_host, int32_t n_segments, int32_t include_self,
                       void* out_self, void* out_mean, int64_t out_pitch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Node-partitioned feature table (multi-GPU, SURVEY 8e; no reference counterpart - the reference is
 * single-device).  Shard r owns the global ids [row_start[r], row_start[r+1]) (contiguous ranges - align them
 * with communities); every rank maps all shards into its address space (CUDA IPC over NVLink/NVSwitch), so the
 * gather kernel resolves
 *   row(id) = base[owner(id)] + (id - row_start[owner(id)]) * pitch
 * and pulls remote rows itself - one cp.async.bulk per row over NVLink into shared memory (or 128-bit loads with
 * gather_variant=0): the halo exchange is fused into the gather, no staging buffer, no collective on the data path.
 * A rank may also hold REPLICAS of the remote rows it reads most: remap (device int32 [n_global_rows], may be NULL)
 * gives, for every id, the row index inside this rank's OWN buffer (own rows, zero row, replicas) or -1 when the
 * row has to come from its owner.  Ids outside [0, n_global_rows-1) - including the dummy id N - read the caller's
 * local zero row (index zero_row of its own buffer).
 * gs_gather_mean_sharded has the semantics of gs_gather_mean with `src` replaced by the table.
 * --------------------------------------------------------------------------------------------- */
#define GS_MAX_SHARDS 16
typedef struct {
  const void* base[GS_MAX_SHARDS];       /* device pointers; shard r holds its own rows first */
  int64_t row_start[GS_MAX_SHARDS + 1];  /* row_start[0] = 0 ... row_start[n_shards] = N */
  int32_t n_shards;
  int32_t my_shard;
  int64_t n_global_rows;                 /* N + 1 (the dummy row is virtual: every shard carries its own zero row) */
  int64_t zero_row;                      /* index of the all-zero row inside base[my_shard] */
  const int32_t* remap;                  /* device, [n_global_rows] or NULL (see above) */
} gs_sharded_table;

/* ids_are_locators: 0 = global ids; 1 = gs_translate_ids locators; 2 = gs_halo_translate locators (negative values index
 * `staging`, this step's halo rows fetched by gs_halo_fetch; staging has the table's pitch) */
int32_t gs_gather_mean_sharded(const gs_sharded_table* table_host, int32_t dtype, int32_t F, int64_t pitch,
                               const gs_segment* segments_host, int32_t n_segments, int32_t include_self,
                               int32_t ids_are_locators, const void* staging, void* out_self, void* out_mean,
                               int64_t out_pitch, void* stream);
/* Halo staging - every remote row a step needs crosses NVLink ONCE (a frontier repeats remote nodes; peer reads bypass the
 * local L2).  Per step:  gs_halo_begin (claim[] = -1, *count = 0)  ->  gs_halo_claim for every id list (first sighting of a
 * remote id takes the next staging slot; stage_ids[slot] = id)  ->  gs_halo_fetch (rows of stage_ids[0 .. *count) from their
 * owners into staging[slot])  ->  gs_halo_translate for every id list (out = row of this GPU's own buffer when the row is
 * held locally, else -(slot) - 1)  ->  gs_gather_mean_sharded(..., ids_are_locators = 2, staging).
 * claim: int32 [n_global_rows]; count: int32 [1]; stage_ids: int32 [capacity]; staging: float [capacity, staging_pitch];
 * capacity >= the number of ids claimed (the sum of the lists' lengths always suffices). */
int32_t gs_halo_begin(int32_t* claim, int64_t n_global_rows, int32_t* count, void* stream);
int32_t gs_halo_claim(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, int32_t* claim, int32_t* count,
                      int32_t* stage_ids, int64_t capacity, void* stream);
int32_t gs_halo_fetch(const gs_sharded_table* table_host, int32_t F, int64_t pitch, const int32_t* stage_ids,
                      const int32_t* count, int64_t capacity, float* staging, int64_t staging_pitch, void* stream);
int32_t gs_halo_translate(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, const int32_t* claim,
                          int32_t* out, void* stream);
/* ids -> locators for a table with replicas (remap != NULL): out[i] = remap[ids[i]] (a row index inside this GPU's own
 * buffer) when the row is held locally - own rows, replicas, the zero row for ids outside [0, N) -, else -(ids[i]) - 1.
 * One cheap, fully parallel pass per id list; the gather kernel then needs no table lookup on its copy-issue path. */
int32_t gs_translate_ids(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, int32_t* out, void* stream);
int32_t gs_gather_rows_sharded(const gs_sharded_table* table_host, int32_t dtype, int32_t F, int64_t pitch,
                               const int32_t* ids, int64_t n, void* out, int64_t out_pitch, void* stream);

/* Shard buffers are allocated by the library with cudaMalloc so that they can be exported through
 * CUDA IPC (the only allocation the library ever makes; freed by gs_shard_free). */
int32_t gs_shard_alloc(int64_t bytes, void** dev_ptr_out);
int32_t gs_shard_free(void* dev_ptr);
int32_t gs_ipc_export(const void* dev_ptr, uint8_t* handle64_out_host);
int32_t gs_ipc_import(const uint8_t* handle64_host, void** dev_ptr_out);
int32_t gs_ipc_close(void* dev_ptr);

/* ---------------------------------------------------------------------------------------------
 * Feature table in host memory (graphsage_b200.HostFeatures).  The [N+1, pitch] rows stay in page-locked host memory
 * that the device addresses directly; per step the rows the batch reads are staged into a device "working set"
 *   [C cached rows | 1 zero row | S staging rows]     (one contiguous table, the host table's pitch and dtype)
 * and layer 0 runs on it with translated ids.  The hit test is the halo one with a single shard: describe the working
 * set as a gs_sharded_table with n_shards = 1, row_start = {0, N}, base[0] = the working set, zero_row = C and
 * remap = cache_slot (device int32 [N+1]: the working-set row of a cached id, -1 otherwise).  Per step:
 *   gs_halo_begin  ->  gs_halo_claim per id list (every distinct uncached id in [0, N) takes the next staging slot)
 *   ->  gs_host_fetch (rows stage_ids[0 .. *count) from the host table into the staging rows)
 *   ->  gs_host_translate per id list.
 * No step reads *count on the host: every launch size follows from the batch shape, so the sequence is capturable. */
/* Page-lock host_ptr[0 .. bytes) once, mapped into the device address space; *dev_alias_out is the address the kernels
 * read it through.  gs_host_unregister undoes it (the memory itself stays the caller's). */
int32_t gs_host_register(void* host_ptr, int64_t bytes, void** dev_alias_out);
int32_t gs_host_unregister(void* host_ptr);
/* staging[i] = host_alias[stage_ids[i]] for i in [0, min(*count, capacity)): whole rows of row_bytes (a multiple of 16)
 * over the host link with 16-byte loads, several rows in flight per warp.  The grid does not depend on *count. */
int32_t gs_host_fetch(const void* host_alias, int64_t row_bytes, const int32_t* stage_ids, const int32_t* count,
                      int64_t capacity, void* staging, void* stream);
/* gs_halo_translate with non-negative rows: out[i] = the working-set row of ids[i] - remap[id] for a cached id, zero_row
 * for an id outside [0, N), stage_row0 + claim[id] for a staged one. */
int32_t gs_host_translate(const gs_sharded_table* table_host, const int32_t* ids, int64_t n, const int32_t* claim,
                          int64_t stage_row0, int32_t* out, void* stream);
/* The sampled blocks' layer-0 load (no working set, no claim): out[i, 0:F) = the row of ids[i] widened to fp32, columns
 * F..out_pitch-1 zeroed, for i < n.  The row is cache[cache_slot[id]] when cache_slot[id] >= 0 (the working set's cached
 * rows), the zero row for an id outside [0, n_nodes) - the dummy id N included; no host read is made for it - and else
 * host_alias[id] over the host link (gs_host_register).  dtype GS_F32 / GS_BF16 (pitch in elements; bf16 widened
 * exactly) or GS_I8ROW (pitch in bytes; deq_c = fl(float(q_c) * s), the scale read from the row), the same pitch for
 * host and cache rows: 16-byte multiples at 16-byte aligned addresses.  out: 16-byte aligned, out_pitch % 4 == 0 and
 * >= F (and <= gs_i8row_pitch(F) for GS_I8ROW).  Duplicate ids are allowed; no atomics, no allocation, no host
 * synchronisation; a capped grid keeps several rows' loads in flight per warp, as gs_host_fetch does.  int8 rows with
 * F <= 4092 are read as whole-row copies read them, one warp per row, the scale taken from the row's own unit. */
int32_t gs_host_gather_rows_f32(const void* host_alias, const void* cache, const int32_t* cache_slot, int32_t dtype,
                                int64_t n_nodes, int32_t F, int64_t pitch, const int32_t* ids, int64_t n, float* out,
                                int64_t out_pitch, void* stream);

/* embedding_lookup (models.py:299) with the result widened to fp32: out[i, 0:F] = (float)feats[ids ? ids[i] : row0 + i, 0:F],
 * columns F..out_pitch-1 zeroed.  feats is GS_BF16, GS_F32 or GS_I8ROW (pitch in bytes; the dequantised values).  The bf16
 * max-pool path uses it for the SELF rows, which meet the fp32 self_weights contraction (aggregators.py:185); over an int8
 * table the pooling aggregators read their neighbour and self rows through it. */
int32_t gs_gather_rows_f32(const void* feats, int32_t dtype, int64_t n_rows, int32_t F, int64_t pitch,
                           const int32_t* ids, int64_t row0, int64_t n, float* out, int64_t out_pitch,
                           void* stream);
/* fp32 [n, F] (row stride ldx) -> bf16 [n, out_pitch], round-to-nearest-even, pad columns zeroed: the next layer's
 * bf16 source table of the max-pool path (the hidden[hop] list of models.py:321-329 kept in the K4 operand type). */
int32_t gs_cast_rows_bf16(const float* x, int64_t n, int32_t F, int64_t ldx, void* out_bf16, int64_t out_pitch,
                          void* stream);

/* ---------------------------------------------------------------------------------------------
 * R-MAT graph written directly as CSR on the device (BASELINE.json configs[4]: scale 27 trimmed to 10^8 nodes, about 20
 * entries per node, a, b, c, d = 0.57, 0.19, 0.19, 0.05).  No reference counterpart - the reference reads graphs from
 * disk (graphsage/utils.py:19-75); this is the synthetic stand-in at that size.  Contract: oracle/rmat.py, csrc/rmat.cu.
 *   1. gs_rmat_degrees -> deg[n_nodes] (int32);  2. caller: indptr = exclusive prefix sum (int64 [n_nodes + 1]);
 *   3. gs_rmat_fill -> indices[indptr[n_nodes]] (int32 neighbour ids, unsorted, duplicates possible, no self loops).
 * Node ids are scrambled by y = (x * mul + add) mod n_nodes, which must be a bijection: (mul * mul_inv) mod n_nodes == 1.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_rmat_degrees(int32_t scale, int64_t n_nodes, double edge_factor, double a, double b, double c, double d,
                        uint64_t seed, uint64_t mul, uint64_t mul_inv, uint64_t add, int32_t* deg_out, void* stream);
/* long_rows (device int64 [n_long], may be NULL with n_long = 0): the rows with more than long_threshold entries - R-MAT's
 * hubs (1.2 M entries in one row at scale 27); they are filled by a whole grid each instead of one warp.  n_long <= 65535. */
int32_t gs_rmat_fill(int32_t scale, int64_t n_nodes, double a, double b, double c, double d, uint64_t seed, uint64_t mul,
                     uint64_t mul_inv, uint64_t add, const int64_t* indptr, int32_t* indices, const int64_t* long_rows,
                     int64_t n_long, int64_t long_threshold, void* stream);

/* segmented max over fixed fanout: out[i, c] = max_j x[i*k + j, c]   (aggregators.py:182) */
int32_t gs_segment_max(const float* x, int64_t n, int32_t k, int32_t C, int64_t ldx,
                       float* out, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The dense contraction of an aggregator (aggregators.py:51-64, 110-116, 184-195; Dense
 * layers.py:104-116):
 *   part p (p < n_parts <= 2):  P_p = A_p[M, K_p] @ B_p[K_p, N_p]      (B row-major, ldb)
 *   combine ADD   : out[:, 0:N]            = act(P_0 + P_1 + bias)      (N_0 == N_1)
 *   combine CONCAT: out[:, 0:N_0]          = act(P_0 + bias[0:N_0]),
 *                   out[:, N_0:N_0+N_1]    = act(P_1 + bias[N_0:])
 *   bias may be NULL.  fp32 in/out.  `math` selects the arithmetic (gs_math).
 *   workspace: device scratch of gs_sage_gemm_workspace_bytes(...) bytes (may be NULL if 0).
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  const float* A; int64_t lda; int32_t K;
  const float* B; int64_t ldb; int32_t N;
} gs_gemm_part;

int64_t gs_sage_gemm_workspace_bytes(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts,
                                     int32_t math);
int32_t gs_sage_gemm(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine,
                     const float* bias, int32_t act, int32_t math, float* out, int64_t ldo,
                     void* workspace, void* stream);

/* Weight packing for the tensor-core modes can be hoisted out of the step when the weights do not
 * change (inference): gs_sage_gemm_pack fills `workspace` (gs_sage_gemm_workspace_bytes) from the parts'
 * B matrices; gs_sage_gemm_prepacked then runs only the GEMM.  gs_sage_gemm == pack + prepacked. */
int32_t gs_sage_gemm_pack(const gs_gemm_part* parts_host, int32_t n_parts, int32_t math, void* workspace,
                          void* stream);
int32_t gs_sage_gemm_prepacked(int64_t M, const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine,
                               const float* bias, int32_t act, int32_t math, float* out, int64_t ldo,
                               const void* workspace, void* stream);

/* gs_sage_gemm_prepacked with the A rows of a part read BY ID from a row table, so rows that only feed the GEMM need no
 * gathered copy (the mean layer-0 self rows: their ids index the feature table).  row_ids_host[p] (p < n_parts; the array
 * or an entry may be NULL, and an entry with n_ranges == 0 means the same) turns parts[p].A into a table of
 * n_table_rows rows (row stride lda):
 *   operand row r of part p = parts[p].A[ranges[s].ids[r - ranges[s].row0] * lda + 0:K]  for the first range s with
 *   row0 <= r < row0 + n;  ids outside [0, n_table_rows) read row n_table_rows - 1 (the zero dummy row: the rule of
 *   gs_gather_mean);  rows no range covers are zero.
 * The loaded values, the operand split and the MMA order are those of the dense form, so the result is bit-identical to
 * gs_sage_gemm_prepacked on the gathered rows, in every math (workspace as for gs_sage_gemm_prepacked; none for
 * GS_MATH_FP32_SIMT).  Limits: n_ranges <= GS_MAX_SEGMENTS, 1 <= n_table_rows < 2^31. */
typedef struct {
  const int32_t* ids;   /* device, n ids */
  int64_t row0;         /* first operand row they feed */
  int64_t n;
} gs_row_range;
typedef struct {
  int64_t n_table_rows;
  int32_t n_ranges;
  int32_t _pad;
  gs_row_range ranges[GS_MAX_SEGMENTS];
} gs_gemm_row_ids;
int32_t gs_sage_gemm_rows(int64_t M, const gs_gemm_part* parts_host, const gs_gemm_row_ids* row_ids_host, int32_t n_parts,
                          int32_t combine, const float* bias, int32_t act, int32_t math, float* out, int64_t ldo,
                          const void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------------
 * One whole aggregator layer for a SMALL number of output rows (the last layers of the recursion:
 * 512 rows at batch 512) in one launch, exact fp32 FFMA:
 *   mean over the fanout (gs_gather_mean semantics, one segment) -> two (or one) matmuls ->
 *   add | concat -> + bias -> act -> optional row l2_normalize (reference aggregators.py:43-64 /
 *   101-116, models.py:368).  parts: part 0 multiplies the SELF rows, part 1 the MEAN rows; with
 *   n_parts == 1 the single part multiplies the mean rows (GCN form, include_self = 1).
 *   parts[i].A is ignored (the operands are produced in shared memory).
 *   If counter_dev != NULL, *counter_dev += counter_inc after the layer (advances the samplers'
 *   device-side call counter for the next CUDA-graph replay).
 * Limits: K_p <= 2048, total output width <= 1024.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_sage_layer_small(const float* src, int64_t n_src_rows, int32_t F, int64_t pitch,
                            const gs_segment* segment_host, int32_t include_self,
                            const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine,
                            const float* bias, int32_t act, int32_t l2_normalize,
                            float* out, int64_t ldo, uint64_t* counter_dev, uint64_t counter_inc,
                            void* stream);
/* gs_sage_layer_small over a GS_I8ROW table (pitch in bytes, % 16 == 0, >= gs_i8row_pitch(F); 16-byte aligned): the bits
 * gs_sage_layer_small gives on the dequantised table held with a 16-byte-aligned pitch that is a multiple of 4 floats (the
 * layout SampleAndAggregate keeps fp32 tables in).  The one-layer model of <= 2,048 rows runs layer 0 here. */
int32_t gs_sage_layer_small_i8(const void* src, int64_t n_src_rows, int32_t F, int64_t pitch,
                               const gs_segment* segment_host, int32_t include_self,
                               const gs_gemm_part* parts_host, int32_t n_parts, int32_t combine,
                               const float* bias, int32_t act, int32_t l2_normalize,
                               float* out, int64_t ldo, uint64_t* counter_dev, uint64_t counter_inc,
                               void* stream);

/* ---------------------------------------------------------------------------------------------
 * K4 - the max-pool aggregator's neighbour branch fused end to end on the tensor cores (wgmma, bf16 operands, fp32
 * accumulate):   out[g, h] = max_{j<k} relu( table[row(g,j), 0:K] . Wm[0:K, h] + bm[h] )
 *   reference graphsage/aggregators.py:176-182 (reshape -> Dense(relu,bias) -> reshape -> reduce_max),
 *   graphsage/layers.py:104-116, with the gather of graphsage/models.py:299 fused in front.
 *   row(g, j) = row_ids ? row_ids[g*k + j] : row0 + g*k + j;  table is bf16 [n_rows, pitch] (pitch % 8 == 0).
 *   packed_weights: gs_maxpool_mlp_pack(Wm fp32 [K, hidden] row-major) into gs_maxpool_mlp_workspace_bytes
 *   bytes (do it once per weight update).  Limits: K <= 640, k <= 128, hidden % 128 == 0 (else
 *   GS_ERR_UNSUPPORTED: use gs_gather_rows + gs_sage_gemm + gs_segment_max).
 * --------------------------------------------------------------------------------------------- */
int64_t gs_maxpool_mlp_workspace_bytes(int32_t K, int32_t hidden);
int32_t gs_maxpool_mlp_pack(const float* Wm, int64_t ldw, int32_t K, int32_t hidden, void* workspace,
                            void* stream);
int32_t gs_maxpool_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch,
                             const int32_t* row_ids, int64_t row0, int64_t n_groups, int32_t k,
                             const void* packed_weights, const float* bias, int32_t hidden,
                             float* out, int64_t ldo, void* stream);
/* MeanPoolingAggregator's neighbour branch (reference graphsage/aggregators.py:246-273): same kernel, the
 * epilogue averages relu(x + b) over the fanout instead of taking the max. */
int32_t gs_meanpool_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch,
                              const int32_t* row_ids, int64_t row0, int64_t n_groups, int32_t k,
                              const void* packed_weights, const float* bias, int32_t hidden,
                              float* out, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K5 - the two-layer max-pool aggregator's neighbour branch fused end to end (wgmma, bf16 operands, fp32 accumulate):
 *   h1 = bf16_rne(relu(table[row(g,j), 0:K] . W1 + b1));  out[g, u] = max_{j<k} relu(h1 . W2[:, u] + b2[u])
 *   reference graphsage/aggregators.py:276-361 (TwoMaxLayerPoolingAggregator: reshape -> Dense -> Dense -> reshape ->
 *   reduce_max) with the gather of graphsage/models.py:299 fused in front; the gathered rows and h1 stay on chip.
 *   Rows are addressed as in gs_maxpool_mlp_fused.  packed_w1 / packed_w2: gs_maxpool_mlp_pack of W1 fp32 [K, h1] and
 *   of W2 fp32 [h1, h2].  b1 / b2 may be NULL (zero).  Limits: k <= 128, K <= 640, h1 % 128 == 0, h2 % 256 == 0 (else
 *   GS_ERR_UNSUPPORTED: use gs_gather_rows + gs_sage_gemm twice + gs_segment_max).  No atomics, no allocation.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_maxpool2_mlp_fused(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch,
                              const int32_t* row_ids, int64_t row0, int64_t n_groups, int32_t k,
                              const void* packed_w1, const float* b1, int32_t h1, const void* packed_w2,
                              const float* b2, int32_t h2, float* out, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Backward of the pooling branch through K4 (bf16 operands, fp32 accumulate; no atomics, deterministic).
 * One hop: X = the n_groups*k gathered rows (addressed as in gs_maxpool_mlp_fused), pre = X Wm, b = bias,
 * dhp [n_groups, hidden] = gradient of the pooled output.  Same limits as K4: k <= 128, K <= 640, hidden % 128 == 0
 * (else GS_ERR_UNSUPPORTED).
 *
 * B1 gs_pool_mlp_backward_dp: recomputes pre with K4's main loop (128-row tiles of G = 128 / k groups), then
 *   max:  hp = relu(max_j pre_j + b); if hp > 0, dpre_j = [fl(pre_j + b) == hp] * (dhp / count), count = number of
 *         such j (ties split evenly: TensorFlow's reduce_max gradient times the ReLU mask); else dpre_j = 0
 *   mean: dpre_j = (dhp / k) * [fl(pre_j + b) > 0]
 *   and writes into dp (gs_pool_mlp_dp_bytes): dP = bf16(dpre) as tile images of dP^T, then the fp32 per-(tile,
 *   column) sums of dpre (per parity of the group index: group sums in j order added in g order; then even + odd).
 *   pre here is bit for bit the fp32 pre-activation the default K4 forward (gs_maxpool_mlp_fused /
 *   gs_meanpool_mlp_fused without tuning keys) accumulates for the same row: the same main loop, tiles and row slots,
 *   so dhp reaches exactly the rows whose values the forward returned (oracle/pool_backward.py).
 *   packed_weights: gs_maxpool_mlp_pack.
 * B2 gs_pool_mlp_backward_dw: dWm += X^T dP (dWm [K, hidden] fp32, ldw == hidden) and dbm += the column sums of dpre,
 *   X re-gathered from the table; both combined in a fixed order (workspace: gs_pool_mlp_dw_workspace_bytes).
 * B3 gs_pool_mlp_backward_dx: dx[r, :Kd] = (dP Wm^T)[r, :Kd] for the n_groups*k gathered rows (fp32, overwritten);
 *   packed: gs_pool_mlp_dx_pack(Wm) into gs_pool_mlp_dx_pack_bytes(Kd, hidden) bytes.
 * --------------------------------------------------------------------------------------------- */
int64_t gs_pool_mlp_dp_bytes(int64_t n_groups, int32_t k, int32_t hidden);
int32_t gs_pool_mlp_backward_dp(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch,
                                const int32_t* row_ids, int64_t row0, int64_t n_groups, int32_t k,
                                const void* packed_weights, const float* bias, int32_t hidden, const float* dhp,
                                int64_t lddhp, int32_t pool_mean, void* dp, void* stream);
int64_t gs_pool_mlp_dw_workspace_bytes(int64_t n_groups, int32_t k, int32_t K, int32_t hidden);
int32_t gs_pool_mlp_backward_dw(const void* table_bf16, int64_t n_rows, int32_t K, int64_t pitch,
                                const int32_t* row_ids, int64_t row0, int64_t n_groups, int32_t k, int32_t hidden,
                                const void* dp, void* workspace, int64_t workspace_bytes, float* dWm, int64_t ldw,
                                float* dbm, void* stream);
int64_t gs_pool_mlp_dx_pack_bytes(int32_t Kd, int32_t hidden);
int32_t gs_pool_mlp_dx_pack(const float* Wm, int64_t ldw, int32_t Kd, int32_t hidden, void* packed, void* stream);
int32_t gs_pool_mlp_backward_dx(int64_t n_groups, int32_t k, int32_t hidden, const void* dp, const void* packed,
                                int32_t Kd, float* dx, int64_t ldx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * One pipelined step from HOST buffers in a single call (no per-kernel host work), on three streams:
 *   h2d_stream     : wait ev_done (this slot's previous step no longer reads ids_dev), copy ids host->device,
 *                    record ev_ids
 *   compute_stream : wait ev_ids and ev_drained (this slot's previous result has left the device), launch the
 *                    captured CUDA graph(s) of the step, record ev_done
 *   copy_stream    : wait ev_done, copy the result device->host, record ev_drained
 * so the id upload of step i+1 and the result download of step i-1 both overlap the kernels of step i.
 * All handles are the caller's CUDA objects (cudaGraphExec_t, cudaStream_t, cudaEvent_t as void*); events must
 * have been recorded at least once; host buffers should be pinned.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_pipeline_step(const void* ids_host, void* ids_dev, int64_t ids_bytes, void* const* graph_execs_host,
                         int32_t n_graphs, const void* out_dev, void* out_host, int64_t out_bytes,
                         void* h2d_stream, void* compute_stream, void* copy_stream, void* ev_ids, void* ev_done,
                         void* ev_drained);

/* *counter_dev += inc, on the stream: advances the samplers' device-side call counter once per step (the counter a
 * CUDA-graph replay reads, see gs_sample_padded) when the step's last kernel is not gs_sage_layer_small. */
int32_t gs_bump_counter(uint64_t* counter_dev, uint64_t inc, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Gradient of the trainable node-embedding table (identity_dim > 0): the IndexedSlices gradient of
 * tf.nn.embedding_lookup(embeds, ids) at reference graphsage/models.py:299, densified - TF 1.8's clip_by_value
 * (supervised_models.py:95-99, models.py:379-383) converts it to a dense tensor with duplicate ids summed.
 *   out[r, 0:d] = sum over lists l, contributions i < l.n with l.ids[i] == r of  l.scale * l.grad[(i / l.group) * l.ldg + 0:d]
 * for every r in [0, n_rows); rows nobody addresses are zero (the whole [n_rows, d] block at row stride ldo is written, also
 * when there are no contributions).  ids outside [0, n_rows) contribute nothing.  The layer-0 backward passes, per hop
 * segment: mean - (self ids, dxs, 1, 1) and (neighbour ids, dxm, k, 1/k); gcn - (self ids, dxm, 1, 1/(k+1)) and
 * (neighbour ids, dxm, k, 1/(k+1)); max-/mean-pool - (self ids, dxs, 1, 1) and (neighbour ids, dxn, 1, 1).
 * Deterministic (bit-identical on every call, no atomics).  Summation order for a row r:
 *   number the contributions of all lists in call order (list 0 first, i ascending) and sort them by (r, number); cut
 *   that sorted sequence into fixed chunks of 32.  Within a chunk the products scale * grad are added left to right
 *   in fp32.  A row whose contributions span several chunks gets one such partial sum per chunk (pieces q = 0, 1, ...
 *   in sorted order); piece q goes to accumulator (q / 8) % 4 of lane q % 8, each accumulator adds its pieces in
 *   ascending q from +0, a lane adds its accumulators 0..3 in order, and the row is lane 0 + lane 1 + ... + lane 7, in order.
 *   So a long run of one id (the padding id, a hub) is split into chunks that are summed in parallel.  Every product
 *   scale * grad is rounded to fp32 before it is added (no fused multiply-add), each piece starts from +0, and every
 *   addition is one fp32 rounding: the result is oracle/sparse_grad.py's embedding_grad_reference bit for bit.
 * workspace: device scratch of gs_embedding_grad_workspace_bytes(...) bytes (0 when there are no contributions); it
 * depends on the lists' lengths, n_rows and d only.  Limits: n_lists <= GS_MAX_EMBED_LISTS, fewer than 2^31 contributions,
 * n_rows < 2^31 - 1, ldg >= d, group >= 1.
 * --------------------------------------------------------------------------------------------- */
#define GS_MAX_EMBED_LISTS 8
typedef struct {
  const int32_t* ids;   /* device, n ids */
  const float* grad;    /* device gradient rows, row stride ldg (elements); contribution i reads row i / group */
  int64_t ldg;
  int64_t n;            /* contributions */
  int32_t group;
  float scale;
} gs_embed_grad_list;

int64_t gs_embedding_grad_workspace_bytes(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows,
                                          int32_t d);
int32_t gs_embedding_grad(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows, int32_t d, float* out,
                          int64_t ldo, void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dropout for training (tf.nn.dropout at reference aggregators.py:46-47 / 104-105, layers.py:107).  TF's mask stream
 * cannot be reproduced, so masks follow a counter-based contract (oracle/dropout.py), regenerated in the backward pass
 * instead of being stored.  A SITE is one dropout application over a logical [rows, F] tensor:
 *   element (pos, c) is kept iff word c % 4 of philox4x32_10(ctr = (c / 4, pos & 0xffffffff, pos >> 32, call),
 *   key = (seed & 0xffffffff, seed >> 32)) is >= T = floor(rate * 2^32) (computed in float64 from the fp32 rate);
 *   a kept element becomes x / keep, keep = fp32(1 - rate) (IEEE division), a dropped element 0.  0 <= rate < 1.
 * Columns are logical (0 .. F-1, independent of any pitch).  Positions: neighbour j of output row i of a segment:
 * pos = i * k + j (the row-major [n, k, F] flattening); self row of i: pos = i; any other [rows, F] tensor: pos = row.
 * The call number a kernel uses is (uint32_t)(call + (call_dev ? *call_dev : 0)), read on the stream when the kernel runs -
 * the convention of the samplers' counter_dev.  A CUDA graph bakes `call` into its launches; with call_dev pointing at a
 * device word that is set (or advanced with gs_bump_counter) before each replay, every replay draws fresh masks.  With
 * call_dev == NULL the site is exactly the host-numbered site.
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  uint64_t seed;
  uint32_t call;
  float rate;
  const uint64_t* call_dev;   /* device, optional: added to call */
} gs_dropout_site;

/* gs_gather_mean (GS_F32 tables only) with dropout applied to the gathered rows in registers:
 *   out_self[r] = drop(self_sites[s], pos = i, self row)                                   (if out_self != NULL)
 *   out_mean[r] = (sum_j drop(neigh_sites[s], pos = i*k + j, neigh row j) (+ drop(self row))) / (k (+1 if include_self))
 * summed in j order, the self row last - the order of gs_gather_mean, which this equals bit for bit when every rate is 0.
 * neigh_sites_host / self_sites_host hold one site per segment. */
int32_t gs_gather_mean_dropout(const float* src, int64_t n_src_rows, int32_t F, int64_t pitch, const gs_segment* segments_host,
                               int32_t n_segments, const gs_dropout_site* neigh_sites_host,
                               const gs_dropout_site* self_sites_host, int32_t include_self, float* out_self,
                               float* out_mean, int64_t out_pitch, void* stream);

/* Masked scale, elementwise over a [rows, F] block:
 *   v = keep(site, pos, c) ? (x[(r / group) * ldx + c] * scale) / keep : 0,  pos = pos_ids ? pos_ids[r] : r
 *   out[r * ldo + c] = accumulate ? out[r * ldo + c] + v : v
 * group >= 1 repeats each x row for `group` consecutive output rows (the fanout mean's backward).  out may alias x when
 * group == 1 and ldo == ldx.  pos_ids (device int32 [rows], may be NULL) names each row's position by id: the
 * full-neighbourhood self rows and MLP inputs of a minibatch block, masked by their global node ids.  Each element is read
 * and written by one thread: bit-identical on every call. */
int32_t gs_dropout_apply(const float* x, int64_t ldx, int64_t rows, int32_t F, int32_t group, float scale,
                         gs_dropout_site site, int32_t accumulate, float* out, int64_t ldo, const int32_t* pos_ids,
                         void* stream);

/* gs_embedding_grad with a dropout site per list (sites_host[l]; NULL: no masks): contribution i of list l adds
 *   keep(site_l, pos = i, c) ? (l.scale * l.grad[(i / l.group) * l.ldg + c]) / keep : 0
 * to column c of its row - the gradient through drop(embedding_lookup(...)) with the masks regenerated, not stored.
 * Workspace, limits and the summation order are those of gs_embedding_grad (the query above gives the size). */
int32_t gs_embedding_grad_dropout(const gs_embed_grad_list* lists_host, const gs_dropout_site* sites_host, int32_t n_lists,
                                  int64_t n_rows, int32_t d, float* out, int64_t ldo, void* workspace,
                                  int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Node2Vec / DeepWalk baseline (reference graphsage/models.py:408-501, Node2VecModel).
 *
 * gs_embedding_sgd - the sparse GradientDescentOptimizer update of embedding tables (tf.train.GradientDescentOptimizer on the
 *   IndexedSlices gradient of embedding_lookup: scatter_sub with duplicate ids summed):
 *     table[r, 0:d] += alpha * (sum over list entries i with ids[i] == r of l.scale * l.grad[(i / l.group) * l.ldg + 0:d])
 *   for every TOUCHED row r, in place (alpha = -learning rate).  Rows no id addresses are never read or written; ids outside
 *   [0, n_rows) contribute nothing.  The row sum is formed in the summation order documented for gs_embedding_grad (same
 *   sort, chunks and combine), then added once: table[r] = fmaf(alpha, sum, table[r]), one rounding.  Bit-identical on
 *   every call.
 *   Lists, workspace (gs_embedding_grad_workspace_bytes) and limits as for gs_embedding_grad; ldt >= d.  Pass every list
 *   that touches the table in ONE call so that an id appearing in several lists is summed before the update. */
int32_t gs_embedding_sgd(const gs_embed_grad_list* lists_host, int32_t n_lists, int64_t n_rows, int32_t d, float alpha,
                         float* table, int64_t ldt, void* workspace, int64_t workspace_bytes, void* stream);

/* gs_skipgram_grad - one skip-gram forward + backward over the two tables (Node2VecModel._loss / _accuracy,
 * models.py:478-501), reading the tables only.  target row r = target[r * ldt + 0:d]; context row r = context[r * ldc + 0:d]
 * with its bias in column d (context[r * ldc + d]; ldc >= d + 1).  With t_i = target[batch1[i]], c_i = context[batch2[i]],
 * b_i its bias, n_j = context[neg[j]], nb_j its bias (i < B, j < S); ids outside [0, n_rows) read a zero row and bias:
 *     aff[i]        = t_i . c_i                      (no bias: the MRR affinities, models.py:491)
 *     neg_aff[i, j] = t_i . n_j                      ([B, S] row-major, no bias, models.py:493)
 *     *loss         = (sum_i softplus(-(aff_i + b_i)) + sum_ij softplus(neg_aff_ij + nb_j)) / B     (models.py:479-486)
 *   and the gradient of *loss, per lookup (duplicate ids are summed later, by gs_embedding_sgd):
 *     g_i = (sigmoid(aff_i + b_i) - 1) / B,  h_ij = sigmoid(neg_aff_ij + nb_j) / B
 *     gt[i, 0:d]     = g_i c_i + sum_j h_ij n_j      (j ascending)
 *     gc_pos[i, 0:d] = g_i t_i,   gc_pos[i, d] = g_i                       (bias gradient in column d)
 *     gc_neg[j, 0:d] = sum_i h_ij t_i,   gc_neg[j, d] = sum_i h_ij         (ldgc >= d + 1)
 *   Dot products (aff, neg_aff): lane l (of 32) holds s = +0 and s = fmaf(t_q, c_q, s) for q = l, l + 32, ...; the lanes
 *   are combined by the xor butterfly v += shfl_xor(v, o), o = 16, 8, 4, 2, 1, in fp32.  gc_pos[i, 0:d] = fp32(g_i * t_i).
 *   gt: v = fp32(g_i * c_iq), then v = fmaf(h_ij, n_jq, v) for j ascending.  gc_neg: CTA k (grid = min(ceil(B / 8), 256))
 *   takes the pair groups k, k + grid, ... (8 pairs each) and chains acc = fmaf(h_ij, t_iq, acc) from +0 over their rows
 *   in ascending i; a second kernel adds the CTA partials in CTA order.  loss: each pair's softplus(-(aff_i + b_i)),
 *   then + softplus(neg_aff_ij + nb_j) in j order; lane l (of 32) adds pairs l, l + 32, ... from +0, the butterfly
 *   combines the lanes, then one division by fp32(B).  sigmoid(x) = 1 / (1 + expf(-x)), softplus(x) = fmaxf(x, 0) +
 *   log1pf(expf(-|x|)).  No atomics, bit-identical on every call.  The contract and its error bounds are
 *   oracle/sparse_grad.py's skipgram_reference.  workspace: gs_skipgram_workspace_bytes(B, S, d).
 *   Limits: 1 <= B < 2^31, 1 <= S <= GS_MAX_UNIQUE_SAMPLED, d >= 1, n_rows < 2^31. */
int64_t gs_skipgram_workspace_bytes(int64_t B, int32_t S, int32_t d);
int32_t gs_skipgram_grad(const float* target, int64_t ldt, const float* context, int64_t ldc, int64_t n_rows, int32_t d,
                         const int32_t* batch1, const int32_t* batch2, int64_t B, const int32_t* neg, int32_t S, float* loss,
                         float* aff, float* neg_aff, float* gt, int64_t ldgt, float* gc_pos, float* gc_neg, int64_t ldgc,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SeqAggregator (reference graphsage/aggregators.py:363-449): TF 1.8 BasicLSTMCell(H) under dynamic_rnn with
 * sequence_length, over the k sampled neighbours of each of n nodes.  Gate column order i, j, f, o; with z = x·W_x + h·W_h + b
 *     c' = c·σ(z_f + 1) + σ(z_i)·tanh(z_j),   h' = tanh(c')·σ(z_o),   h_0 = c_0 = 0
 * Sequence i is rows i·k .. i·k + k - 1 of every [n·k, .] operand.  All three kernels are fp32 on the CUDA cores, read their
 * loop bounds (the lengths) on the device, allocate nothing, use no atomics and only enqueue on `stream`: bit-identical on
 * every call and capturable in a CUDA graph.
 *
 * gs_seq_lengths - the reference's length rule (:411-414): used[i, j] = 1 iff row x[(i·k + j)·ldx + 0..K) has an element
 *   that is not zero (-0.0 is zero), len[i] = max(1, sum_j used[i, j]).  The LSTM runs over the FIRST len[i] positions,
 *   whatever they hold.
 * gs_lstm_forward - P [n·k, 4H] (ldp) = X·W_x + b from the input projection; Wh the [H, 4H] recurrent block W_h (the
 *   kernel's bottom H rows, ldw).  Writes h_last[i] = h after len[i] steps ([n, H], ldh).  Both kernels clamp len[i]
 *   to [0, k]: a length above k runs k steps; a length <= 0 runs none (h_last[i] = 0, every saved row and every dZ
 *   row of sequence i zero; its P rows and dh_last row are not read).  P rows t >= len[i] are never read either.
 *   Training outputs, all three or none (NULL): gates [n·k, 4H] = (σ(z_i), tanh(z_j), σ(z_f + 1), σ(z_o)), c [n·k, H] = c_t,
 *   h_prev [n·k, H] = h_{t-1} (zero at t = 0); rows t >= len[i] are zeros.  Limits: H in {128, 256}, k >= 1, n < 2^31.
 * gs_lstm_backward - backpropagation through time from dh_last [n, H] (the gradient of h_last) with the forward's saved
 *   gates and c: dZ [n·k, 4H], the gradient of the pre-activations z_t, zero for t >= len[i].  dh_{t-1} = dz_t·W_hᵀ is
 *   carried inside the kernel (columns summed in ascending order).  Wh must be 16-byte aligned with ldw % 4 == 0.
 *   The weight and input gradients are dW_x = Xᵀ·dZ, dW_h = h_prevᵀ·dZ, db = column sums of dZ, dX = dZ·W_xᵀ (the caller's).
 * --------------------------------------------------------------------------------------------- */
int32_t gs_seq_lengths(const float* x, int64_t ldx, int64_t n, int32_t k, int32_t K, int32_t* len, void* stream);
int32_t gs_lstm_forward(const float* P, int64_t ldp, const float* Wh, int64_t ldw, const int32_t* len, int64_t n, int32_t k,
                        int32_t H, float* h_last, int64_t ldh, float* gates, int64_t ldg, float* c, int64_t ldc,
                        float* h_prev, int64_t ldhp, void* stream);
int32_t gs_lstm_backward(const float* dh_last, int64_t lddh, const float* gates, int64_t ldg, const float* c, int64_t ldc,
                         const int32_t* len, const float* Wh, int64_t ldw, int64_t n, int32_t k, int32_t H, float* dZ,
                         int64_t ldz, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The logistic classifier of the reference's eval scripts (eval_scripts/{ppi,reddit,citation}_eval.py:
 * SGDClassifier(loss="log")): scikit-learn's plain SGD loop (_sgd_fast.pyx.tp, _plain_sgd) for the log loss, an L2
 * penalty alpha, an intercept, the "optimal" learning rate, no averaging and no class or sample weights, in fp64, over P
 * independent binary problems that share one X.  Contract: oracle/sgd.py.  Neither entry needs a workspace.
 *
 * gs_sgd_orders - the sample order of every epoch.  Problem p's permutation sigma is the Fisher-Yates shuffle of arange(n)
 *   with our_rand_r (xorshift32; a zero state becomes 1; draw = state % 2^31) from seeds[p] (device uint32 [P]):
 *   for i < n - 1: j = i + draw % (n - i); swap(ind[i], ind[j]).  scikit-learn passes the seed by value, so every epoch
 *   applies the same swaps to the previous epoch's order:  orders[p, 0, k] = sigma[k],
 *   orders[p, e, k] = sigma[orders[p, e - 1, k]].  orders is int32 [P, epochs, n].  sigma is one sequential chain per
 *   problem (one thread); the later epochs are a parallel gather.
 * gs_sgd_fit - problem p learns w (d fp64 weights, wscale = 1) and b = 0 from X [n, d] (row stride ldx, GS_F32 or GS_F64,
 *   every element widened exactly to fp64) with labels[p * ldy + row] (> 0: positive, else negative; y = 1 or 0) in
 *   the order orders[p] (all epochs, t = 1, 2, ... across epochs):
 *     pred   = fl(dot * wscale) + b                       dot: see below
 *     eta    = 1 / (alpha * ((optimal_init + t) - 1))
 *     g      = ((1 - y) - y e) / (1 + e), e = exp(-pred)   if pred > -37, else exp(pred) - y; clipped to +-1e12
 *     update = -eta * g
 *     wscale = wscale * max(0, 1 - eta * alpha);  wscale < 1e-9: w = wscale * w, wscale = 1
 *     update != 0:  w = w + x * (update / wscale),  b = b + update
 *   coef[p * ldc + j] = wscale * w[j] (fp64), intercept[p] = b.  Every product and sum is rounded separately (no FMA).
 *   Dot-product order: lane l (0..31) sums w[j] * x[j] for j = l, l + 32, l + 64, ... (< d) left to right from 0.0; the 32
 *   partial sums are then combined by the xor butterfly v += shuffle_xor(v, m) for m = 16, 8, 4, 2, 1.  exp is CUDA's
 *   double exp (not correctly rounded): results are close to, not bit-identical with, a correctly rounded restatement.
 *   One warp per problem with w in registers; the rows of upcoming steps are prefetched with cp.async into a shared ring.
 * Limits (else GS_ERR_UNSUPPORTED): d <= GS_SGD_MAX_D, P <= GS_SGD_MAX_PROBLEMS, epochs <= GS_SGD_MAX_EPOCHS, n < 2^31.
 * --------------------------------------------------------------------------------------------- */
#define GS_SGD_MAX_D 1024
#define GS_SGD_MAX_PROBLEMS 65535
#define GS_SGD_MAX_EPOCHS 1024
int32_t gs_sgd_orders(const uint32_t* seeds, int32_t P, int64_t n, int32_t epochs, int32_t* orders, void* stream);
int32_t gs_sgd_fit(const void* x, int32_t dtype, int64_t n, int32_t d, int64_t ldx, const int32_t* labels, int64_t ldy,
                   const int32_t* orders, int32_t P, int32_t epochs, double alpha, double optimal_init, double* coef,
                   int64_t ldc, double* intercept, void* stream);

/* ---------------------------------------------------------------------------------------------
 * run_random_walks         reference graphsage/utils.py:77-92 (the `<prefix>-walks.txt` co-occurrence pairs)
 *   For start position t < n (global position i = start_offset + t) and walk w < num_walks (W), with L = walk_len:
 *     node = starts[t];  curr = node;  for j = 0 .. L-1:
 *       if curr != node: emit (node, curr)
 *       if j < L-1: curr = indices[indptr[curr] + mulhi32(draw_j, deg(curr))]   (the reference's L-th choice is unused)
 *   draw_s is word s % 4 of philox4x32_10(ctr = (counter_lo, counter_hi, i, 0x50000000 + w * ceil((L-1)/4) + s / 4),
 *   key = (seed_lo, seed_hi)); mulhi32(a, b) = (a * b) >> 32.  A start outside [0, n_nodes) or without neighbours emits
 *   nothing.  A walk that reaches a node without neighbours, or a neighbour id outside [0, n_nodes), emits it and stops
 *   (the reference would raise; its undirected graphs never get there).  Pairs are ordered by t, then w, then j.
 *   Bit-identical to oracle/walks.py; the draws depend only on (i, w, s), so calls over consecutive chunks of starts with
 *   the matching start_offset give the pairs of one call.
 * gs_random_walks_workspace_bytes - workspace for (n, num_walks, walk_len); -1 (see gs_last_error_string) outside the
 *   limits: 1 <= num_walks <= GS_WALK_MAX_WALKS, 2 <= walk_len <= GS_WALK_MAX_LEN, n * num_walks < 2^31 - 1.
 * gs_random_walks - runs every walk (one thread each; the visited ids and per-walk counts go to the workspace), scans the
 *   counts (CUB, integer: deterministic) and writes the pair count P to the device word *n_pairs.  Also requires
 *   start_offset + n <= 2^32 and n_nodes < 2^31 - 1.
 * gs_random_walks_emit - with the same workspace after gs_random_walks on the same stream: out int32 [P, 2] =
 *   (starts[t], visited id) pairs.  The caller reads *n_pairs to size out (one device-to-host read per call), so the
 *   pair is not meant for CUDA-graph capture.  No atomics: every pair's position is its walk's scanned offset.
 * --------------------------------------------------------------------------------------------- */
#define GS_WALK_MAX_WALKS (1 << 20)
#define GS_WALK_MAX_LEN 33
int64_t gs_random_walks_workspace_bytes(int64_t n, int32_t num_walks, int32_t walk_len);
int32_t gs_random_walks(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, const int32_t* starts, int64_t n,
                        int32_t num_walks, int32_t walk_len, uint64_t seed, uint64_t counter, int64_t start_offset,
                        void* workspace, int64_t workspace_bytes, int64_t* n_pairs, void* stream);
int32_t gs_random_walks_emit(const int32_t* starts, int64_t n, int32_t num_walks, int32_t walk_len, const void* workspace,
                             int64_t workspace_bytes, int32_t* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * node2vec's second-order (p, q) walk (Grover & Leskovec, KDD'16) by rejection sampling.  Contract:
 * oracle/biased_walks.py.  Every rule of gs_random_walks above holds - start excluded, L positions, the L-th move unused,
 * a start of degree 0 emits nothing, a sink or out-of-range id ends the walk, pair order, start_offset - and the same
 * workspace (gs_random_walks_workspace_bytes) and gs_random_walks_emit follow it.  Only the next node changes: from
 * current node v, reached from t, every CSR entry x of v's row (duplicates once each) is a candidate of class
 *     return  x == t                                    a = 1/p
 *     in      x != t, x an entry of t's row (t -> x)    a = 1
 *     out     otherwise                                 a = 1/q
 *   with float64 thr_c = 2^32 if a_c == max(a) else floor(a_c / max(a) * 2^32): the chain moves to entry x with
 *   probability thr_x / sum over v's entries of thr.  GS_WALK_PQ_MIN <= p, q <= GS_WALK_PQ_MAX (finite), so thr_c >= 1.
 *   Move 0 (no t) takes entry mulhi32(word 0 of call 0, deg): uniform and always accepted.
 *   Move s >= 1: attempts a = 0 .. GS_WALK_BIASED_ATTEMPTS - 1: candidate entry mulhi32(cand_a, deg) of v's row in its
 *   given order, accepted iff (uint64)acc_a < thr_class(x).  If all reject: u = w0 | w1 << 32, target =
 *   floor(u * S / 2^64) (S = sum of thr over the row), and the first entry whose inclusive prefix sum of thr exceeds it.
 *   Words: philox4x32_10(ctr = (counter_lo, counter_hi, i, 0x60000000 + ((w * 32 + s) << 3) + call), key = seed); calls
 *   0..6 carry attempts 2 call and 2 call + 1 as (cand, acc, cand, acc); call 7's words 0, 1 are u.  w < 2^20 and s < 32,
 *   so the stream is exactly [0x60000000, 0x70000000): no other kStream* base lies in it, and the uniform walk's words
 *   end below 0x50800000.
 *   p == q == 1 runs gs_random_walks (sorted_indices unused, may be NULL): the uniform walk's pairs, byte for byte.
 * gs_csr_sort_rows - sorted_indices int32 [nnz] = indices sorted ascending (signed) within each row
 *   [indptr[i], indptr[i+1]); entries outside every row are copied unchanged.  The membership test "x in t's row" is a
 *   binary search in t's sorted row; the candidates still come from `indices`' own order.  Start-up work: a device copy
 *   and a CUB segmented sort, no host synchronisation.  Rows must lie in [0, nnz); n_nodes, nnz < 2^31 - 1.
 *   workspace: gs_csr_sort_rows_workspace_bytes(...) bytes (0 when nnz or n_nodes is 0); -1 outside the limits.
 * gs_random_walks_biased - one thread per walk, no atomics and no host synchronisation; writes P to *n_pairs as
 *   gs_random_walks does.  sorted_indices: gs_csr_sort_rows of (indptr, indices).
 * --------------------------------------------------------------------------------------------- */
#define GS_WALK_PQ_MIN 1e-4
#define GS_WALK_PQ_MAX 1e4
#define GS_WALK_BIASED_ATTEMPTS 14
int64_t gs_csr_sort_rows_workspace_bytes(int64_t n_nodes, int64_t nnz);
int32_t gs_csr_sort_rows(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                         int32_t* sorted_indices, void* workspace, int64_t workspace_bytes, void* stream);
int32_t gs_random_walks_biased(const int64_t* indptr, const int32_t* indices, const int32_t* sorted_indices,
                               int64_t n_nodes, const int32_t* starts, int64_t n, int32_t num_walks, int32_t walk_len,
                               double p, double q, uint64_t seed, uint64_t counter, int64_t start_offset, void* workspace,
                               int64_t workspace_bytes, int64_t* n_pairs, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Full-neighbourhood reduction over CSR rows (layer-wise inference, SampleAndAggregate.full_neighbor_embeddings): the
 * fixed-fanout reductions of gs_gather_mean / gs_segment_max (aggregators.py:48, 106-107, 182) with k made per row.
 * Contract: oracle/full_neighbor.py.  Output row i is for node v = rows ? rows[i] : i; its entries are
 * indices[indptr[v] .. indptr[v+1]) in CSR order.  An entry outside [0, n_src_rows) reads row n_src_rows - 1 (the clamp
 * of gs_gather_mean); a node with no entries, or v outside [0, n_nodes), reduces over that row alone (the dummy).
 *   GS_CSR_MEAN      acc = +0; acc += x_j in order; out = acc / (float)count
 *   GS_CSR_MEAN_SELF the same, then acc += src[v] (v clamped like an entry); out = acc / (float)(count + 1)   (GCN)
 *   GS_CSR_MAX       m = x_0; m = fmaxf(m, x_j) in order                                       (gs_segment_max)
 *   GS_CSR_SUM       see the backward below (fp32 only)
 * A CSR whose rows are a fixed-fanout sample gives the bits of gs_gather_mean / gs_segment_max.  dtype GS_F32, or GS_BF16
 * widened to fp32 (pitch % 8 == 0, out_pitch % 8 == 0, 16-byte-aligned src and out).  Output fp32 [n, out_pitch]; columns
 * F..out_pitch-1 are zeroed.  No allocation, no atomics, no host synchronisation: each output element is one sequential
 * chain, so two calls give the same bits.  Rows with more than 256 entries are spread over CTAs by 32-column slices.
 * --------------------------------------------------------------------------------------------- */
typedef enum { GS_CSR_MEAN = 0, GS_CSR_MEAN_SELF = 1, GS_CSR_MAX = 2, GS_CSR_SUM = 3 } gs_csr_op;
int32_t gs_csr_aggregate(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                         const int64_t* indptr, const int32_t* indices, int64_t n_nodes,
                         const int32_t* rows /* may be NULL */, int64_t n, int32_t op,
                         float* out, int64_t out_pitch, void* stream);

/* gs_csr_aggregate with full-neighbourhood training dropout (contract: oracle/full_neighbor_dropout.py), op GS_CSR_MEAN,
 * GS_CSR_MEAN_SELF or GS_CSR_SUM.  Every element a chain reads is masked first - drop(x) = keep ? x / keep : 0 with the
 * sites' Philox rule (gs_dropout_site), bf16 sources after widening - and the chain, its order and its divisor are
 * gs_csr_aggregate's.  Positions come from the map (pos_indptr int64, pos_ids int32 or NULL, pos_nnz): local row r is
 * global node g(r) = pos_ids ? pos_ids[r] : r (r clamped to the dummy row n_nodes first; pos_ids then has n_nodes + 1
 * entries, n_nodes for GS_CSR_SUM, whose rows are the source rows), and
 *   GS_CSR_MEAN / _MEAN_SELF  entry j of node v = rows ? rows[i] : i: neigh_site at pos_indptr[g(v)] + j; the implicit
 *                             dummy entry of an empty row (or of a v outside [0, n_nodes)): neigh_site at pos_nnz + g(v);
 *                             the GCN self row: self_site at g(v);
 *   GS_CSR_SUM (fp32)         over gs_csr_transpose's graph with its t_slot: the entry from forward row i at slot s is
 *                             masked as that forward entry was - neigh_site at pos_indptr[g(i)] + s (s >= 0) or
 *                             pos_nnz + g(i) (s = -1), self_site at g(i) (s = -2).
 * The whole graph passes (indptr, NULL, len(indices)); a minibatch block (gs_csr_blocks_fill) passes (the global indptr,
 * the block's src_ids, the global nnz), so a block masks every element as the whole-graph pass does.  Both rates 0: the
 * plain gs_csr_aggregate kernel runs.  No allocation, no atomics, no host synchronisation: two calls give the same bits. */
int32_t gs_csr_aggregate_dropout(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                 const int64_t* indptr, const int32_t* indices, const int32_t* t_slot /* GS_CSR_SUM */,
                                 int64_t n_nodes, const int32_t* rows /* may be NULL */, int64_t n, int32_t op,
                                 gs_dropout_site neigh_site, gs_dropout_site self_site, const int64_t* pos_indptr,
                                 const int32_t* pos_ids /* may be NULL */, int64_t pos_nnz, float* out, int64_t out_pitch,
                                 void* stream);

/* gs_csr_aggregate_dropout over a sampled block (gs_csr_sampled_blocks_fill_offsets; contract:
 * oracle/sampled_blocks_dropout.py), op GS_CSR_MEAN or GS_CSR_MEAN_SELF: entry j of a row of node v is masked at
 * pos_indptr[g(v)] + pos_off[indptr[v] + j] - its offset in g(v)'s raw CSR row - instead of + j, so a sampled entry is
 * masked as the same global entry is in the whole-graph pass.  pos_off: int32, one per entry of `indices`; not read for
 * an empty row, whose implicit dummy entry stays at pos_nnz + g(v).  Everything else, and both rates 0, as above.  The
 * backward sum over a sampled block runs through gs_csr_aggregate_dropout's GS_CSR_SUM with t_slot mapped through the
 * offsets (t_slot' = pos_off[indptr[i] + t_slot] where t_slot >= 0). */
int32_t gs_csr_aggregate_dropout_offsets(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                         const int64_t* indptr, const int32_t* indices, int64_t n_nodes,
                                         const int32_t* rows /* may be NULL */, int64_t n, int32_t op,
                                         gs_dropout_site neigh_site, gs_dropout_site self_site, const int64_t* pos_indptr,
                                         const int32_t* pos_ids /* may be NULL */, int64_t pos_nnz,
                                         const int32_t* pos_off, float* out, int64_t out_pitch, void* stream);

/* gs_csr_aggregate over weighted edges (contract: oracle/weighted.py), every op: weight is fp32, one value per entry of
 * `indices` (data, no gradient; any finite value).  Entry j's term is fl(weight[indptr[v] + j] * x_j) - the product rounded
 * to fp32 before it joins the chain, never contracted into it - and the chain, its order and its divisor (count, not the
 * weights' sum) are gs_csr_aggregate's: mean (Σ fl(w x)) / count, GCN the same sum plus the node's own row (weight 1)
 * over count + 1, max max fl(w x).  The implicit dummy entry of an empty row, or of a v outside [0, n_nodes), weighs 1, so
 * all-one weights give gs_csr_aggregate's bits.  GS_CSR_SUM (fp32) reads weights aligned with its own (transposed)
 * indices: the backward of the weighted means is the sum of fl(w * g / count) over the transposed rows, each transposed
 * entry carrying its forward entry's weight (1 for slots -1 and -2).  No allocation, no atomics, no host
 * synchronisation. */
int32_t gs_csr_aggregate_weighted(const void* src, int32_t dtype, int64_t n_src_rows, int32_t F, int64_t pitch,
                                  const int64_t* indptr, const int32_t* indices, const float* weight, int64_t n_nodes,
                                  const int32_t* rows /* may be NULL */, int64_t n, int32_t op, float* out,
                                  int64_t out_pitch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Backward of the full-neighbourhood reductions (SupervisedGraphsage.full_neighbor_train_step).  Contract:
 * oracle/full_neighbor_grad.py.  Nodes 0 .. N-1 have CSR rows; the dummy node N closes every [N+1, .] table.
 *
 * GS_CSR_SUM (op of gs_csr_aggregate above, GS_F32 only): acc = +0; acc += x_j in CSR order; out = acc.  A row with no
 *   entries, or v outside [0, n_nodes), is +0 - not the dummy row.  With the transposed CSR below it is the backward of the
 *   means: dsrc[j] = sum over the rows i that read j of g[i] / count_i, in ascending i.
 *
 * The EFFECTIVE CSR of the forward (N + 1 rows): row i < N holds its entries in CSR order, an entry outside [0, N] replaced
 *   by N (the forward's clamp); an empty row (indptr[i+1] <= indptr[i]) holds {N}; the dummy row N holds {N}.  with_self
 *   appends the row's own id i to every row (GS_CSR_MEAN_SELF).
 * gs_csr_transpose - its transpose, on the device: t_indptr int64 [N + 2], t_indices int32 [capacity]; row j of the
 *   transpose holds the source rows i of every effective entry equal to j, in ascending i, entries of one row in CSR
 *   order (what a stable sort by destination gives: CUB's radix sort of (destination, source row) pairs in (i, position)
 *   order).  t_indptr[N + 1] is the effective entry count; t_indices past it are unspecified.  capacity = nnz +
 *   (N + 1) * (1 + with_self), nnz the length of `indices`, which every row's entries must lie in.  Integer work only, no
 *   host synchronisation: the count stays on the device.  workspace: gs_csr_transpose_workspace_bytes(...) bytes;
 *   -1 (see gs_last_error_string) outside the limits n_nodes < 2^31 - 2, capacity < 2^31.
 *   t_slot (int32 [capacity], may be NULL): for each transposed entry, where it sits in its forward row i = t_indices[.]:
 *   j for the row's CSR entry j, -1 for the implicit {N} entry (empty row, dummy row), -2 for the with_self entry - the
 *   positions gs_csr_aggregate_dropout's GS_CSR_SUM masks by.  It comes from the same sort (the slot is sorted as the
 *   value and both outputs are derived from it), so t_indptr and t_indices are the bytes of a call without it.
 * gs_csr_max_backward - the gradient of m = GS_CSR_MAX(z) (TensorFlow's reduce_max gradient: split evenly among ties),
 *   then the ReLU of the Dense layer that made z (z = relu(.) >= 0):
 *   (a) for every effective forward row i <= N and column c: cnt = #{entries e of row i : z[e][c] == m[i][c]}
 *       (duplicates counted), s[i][c] = dm[i][c] / (float)cnt;
 *   (b) for every node j <= N: acc = +0; for i in transposed row j, in order: if z[j][c] == m[i][c], acc += s[i][c];
 *       dz[j][c] = z[j][c] > 0 ? acc : +0.
 *   z, m, dm, s, dz: fp32 [N + 1, F] with their own row pitches (only columns 0..F-1 are read or written).  s is the
 *   caller's scratch, read by (b).  Each output element is
 *   one sequential chain; rows longer than 256 entries are spread over CTAs by 32-column slices (gs_csr_aggregate's hub
 *   split).  No allocation, no atomics, no host synchronisation: two calls give the same bits.
 * --------------------------------------------------------------------------------------------- */
int64_t gs_csr_transpose_workspace_bytes(int64_t n_nodes, int64_t nnz, int32_t with_self);
int32_t gs_csr_transpose(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz, int32_t with_self,
                         int64_t* t_indptr, int32_t* t_indices, int32_t* t_slot /* may be NULL */, void* workspace,
                         int64_t workspace_bytes, void* stream);
int32_t gs_csr_max_backward(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm, int64_t lddm,
                            int32_t F, const int64_t* indptr, const int32_t* indices, const int64_t* t_indptr,
                            const int32_t* t_indices, int64_t n_nodes, float* s, int64_t lds, float* dz, int64_t lddz,
                            void* stream);
/* gs_csr_max_backward of m = GS_CSR_MAX over weighted edges (gs_csr_aggregate_weighted; oracle/weighted.py): weight is
 * aligned with `indices` (the forward's; the dummy entry of an empty row and the dummy row weigh 1), t_weight with
 * t_indices (t_weight[k] = weight[indptr[t_indices[k]] + t_slot[k]] for t_slot >= 0, else 1).
 *   (a) cnt = #{entries e of row i : fl(w_e * z[e][c]) == m[i][c]}, s[i][c] = dm[i][c] / (float)cnt;
 *   (b) acc = +0; for i in transposed row j, in order, with that entry's weight w: if fl(w * z[j][c]) == m[i][c],
 *       acc += fl(w * s[i][c]); dz[j][c] = z[j][c] > 0 ? acc : +0. */
int32_t gs_csr_max_backward_weighted(const float* z, int64_t ldz, const float* m, int64_t ldm, const float* dm,
                                     int64_t lddm, int32_t F, const int64_t* indptr, const int32_t* indices,
                                     const float* weight, const int64_t* t_indptr, const int32_t* t_indices,
                                     const float* t_weight, int64_t n_nodes, float* s, int64_t lds, float* dz,
                                     int64_t lddz, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Receptive-field blocks of a minibatch over whole neighbourhoods (full_neighbor_minibatch_*).  Contract:
 * oracle/full_neighbor_blocks.py.  For a CSR over nodes 0 .. N-1 (N = n_nodes; the dummy node is N), seeds clamped to
 * [0, N] (an id outside [0, N) is N) and L = n_layers: V_L = the seeds; V_l (l = L-1 .. 0) = the sorted-unique union of
 * V_{l+1}, the clamped entries of V_{l+1}'s raw rows, and {N}.  Block l: src_ids int32 [|V_l|] = V_l; indptr int64
 * [|V_l|] - one row per local node but the last (the dummy), V_{l+1}'s members holding their raw rows relabelled to
 * positions in V_l, every other row empty; indices int32 [entries]; rows int32 = the positions in V_l of V_{l+1}
 * (l < L-1, ascending) or of the clamped seeds (l = L-1, in seed order).  gs_csr_aggregate over a block with its rows
 * gives the whole-graph layer's bits for those nodes.
 * gs_csr_blocks_plan - device only: builds every V_l and writes counts_dev int64 [2L] = (|V_l|, entries of block l) for
 *   l = 0 .. L-1.  No host synchronisation inside; the caller reads counts_dev once to size the outputs.
 * gs_csr_blocks_fill - with the same workspace, after gs_csr_blocks_plan on the same stream, and counts = a HOST copy of
 *   counts_dev: writes the blocks into the caller's arrays (one pointer per block; n_out = |V_{l+1}| or n_seeds rows).
 * Integer work only, no atomics: two calls give the same bytes.  workspace: gs_csr_blocks_workspace_bytes(...) bytes,
 *   (L + 1) id arrays and position maps of N + 2 int32, a flag array, an int64 degree array and CUB's temporary storage;
 *   -1 (see gs_last_error_string) outside n_nodes < 2^31 - 3, n_seeds < 2^31, 1 <= n_layers <= GS_MAX_BLOCK_LAYERS.
 * --------------------------------------------------------------------------------------------- */
#define GS_MAX_BLOCK_LAYERS 8
int64_t gs_csr_blocks_workspace_bytes(int64_t n_nodes, int64_t nnz, int64_t n_seeds, int32_t n_layers);
int32_t gs_csr_blocks_plan(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, void* workspace,
                           int64_t workspace_bytes, int64_t* counts_dev, void* stream);
int32_t gs_csr_blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers, void* workspace,
                           int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                           int64_t* const* indptr_out, int32_t* const* indices_out, int32_t* const* rows_out,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sampled receptive-field blocks (sampled_minibatch_*): the blocks above built over S_l, a per-layer sample of each row.
 * Contract: oracle/sampled_blocks.py.  S_l(v) for node v < N with d = the raw row length and k = fanouts[l] (1 <= k <=
 * GS_MAX_FANOUT): every entry in CSR order when d <= k; else the k entry positions of Floyd's algorithm - for i = 0 .. k-1:
 * j = d - k + i, t = (u_i * (j + 1)) >> 32, take t unless already taken, else j - sorted ascending.  Positions, not ids:
 * a repeated id is drawn as separate entries.  u_i = word 0 of Philox4x32-10(counter = (i, v, call mod 2^32,
 * 0x70000000 | l), key = seed).  The draw of t is biased by at most j / 2^32.
 * gs_csr_sampled_blocks_plan / _fill - gs_csr_blocks_plan / _fill with V_l = sorted-unique(V_{l+1}, the clamped entries
 *   of S_l over V_{l+1}'s nodes, N) and block l's member rows holding S_l(v); the same workspace
 *   (gs_csr_blocks_workspace_bytes), layout and rules.  The plan and the fill draw the same words again (nothing is
 *   stored between them).  fanouts: HOST int32 [n_layers], block l uses fanouts[l]; nnz < 2^31.  Block entries:
 *   sum over V_{l+1} of min(d, k_l).  Integer work only, no atomics: two calls with the same (seed, call) give the same
 *   bytes.
 * gs_csr_sample_rows - S_layer over every node as a CSR: out_indptr int64 [N + 1] (exclusive scan of min(d, k)), and, when
 *   out_indices is not NULL, out_indices int32 [out_indptr[N]] = the sampled entries as stored in `indices` (not
 *   clamped).  Call it with out_indices NULL, read out_indptr[N], then again with the array.  workspace:
 *   gs_csr_sample_rows_workspace_bytes(...) bytes; 0 <= layer < GS_MAX_BLOCK_LAYERS.
 * --------------------------------------------------------------------------------------------- */
#define GS_MAX_FANOUT 256
int32_t gs_csr_sampled_blocks_plan(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                   const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts,
                                   uint64_t seed, uint64_t call, void* workspace, int64_t workspace_bytes,
                                   int64_t* counts_dev, void* stream);
int32_t gs_csr_sampled_blocks_fill(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                   const int32_t* seeds, int64_t n_seeds, int32_t n_layers, const int32_t* fanouts,
                                   uint64_t seed, uint64_t call, void* workspace, int64_t workspace_bytes,
                                   const int64_t* counts, int32_t* const* src_ids, int64_t* const* indptr_out,
                                   int32_t* const* indices_out, int32_t* const* rows_out, void* stream);
/* gs_csr_sampled_blocks_fill that also writes, per block, offsets_out[l] int32 [entries of block l] aligned with
 * indices_out[l]: each entry's offset q in its node's raw CSR row - the sorted Floyd position when d > k_l, the entry's
 * own index j when d <= k_l - which gs_csr_aggregate_dropout_offsets masks by.  The same kernels; the other four arrays
 * are the bytes of gs_csr_sampled_blocks_fill. */
int32_t gs_csr_sampled_blocks_fill_offsets(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz,
                                           const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                           const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                           int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                                           int64_t* const* indptr_out, int32_t* const* indices_out,
                                           int32_t* const* rows_out, int32_t* const* offsets_out, void* stream);
int64_t gs_csr_sample_rows_workspace_bytes(int64_t n_nodes, int64_t nnz);
int32_t gs_csr_sample_rows(const int64_t* indptr, const int32_t* indices, int64_t n_nodes, int64_t nnz, int32_t k,
                           uint64_t seed, uint64_t call, int32_t layer, void* workspace, int64_t workspace_bytes,
                           int64_t* out_indptr, int32_t* out_indices /* may be NULL */, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Weighted sampled blocks: the sampled blocks above with S_l^w(v), neighbours drawn in proportion to sample_weight
 * (fp32, one per CSR entry, aligned with indices; NULL only when nnz = 0).  Contract: oracle/weighted_sampling.py.
 * Eligible entries have w > 0 (NaN, zero and negative weights are never drawn), d+ of them: every eligible entry in CSR
 * order when d+ <= k; else the k eligible entries with the smallest (key_j, j), key_j = E_j / w_j in fp64 (+inf weights
 * give 0), E_j = -ln U_j by the oracle's fixed sequence of fp64 operations, U_j = (2m + 1) 2^-53 from words (0, 1) (j
 * even) or (2, 3) (j odd) of Philox4x32-10(counter = (j >> 1, v, call mod 2^32, 0x80000000 | l), key = seed) - sorted
 * ascending by position.  The order of the smallest keys is successive sampling in proportion to w.
 * gs_csr_weighted_blocks_plan / _fill / _fill_offsets - gs_csr_sampled_blocks_plan / _fill / _fill_offsets over
 *   S_l^w: the same workspace (gs_csr_blocks_workspace_bytes), layout, offsets and one read of counts_dev; block
 *   entries: sum over V_{l+1} of min(d+, k_l).  The plan and the fill recompute the selection (nothing is stored between
 *   them); a selection reads every weight of its row, a row of 4096 or more entries spread over a CTA.  No atomics: two
 *   calls with the same (seed, call) give the same bytes.
 * gs_csr_sample_rows_weighted - gs_csr_sample_rows over S_layer^w (out_indptr: exclusive scan of min(d+, k)); the same
 *   workspace (gs_csr_sample_rows_workspace_bytes) and two-call protocol.
 * --------------------------------------------------------------------------------------------- */
int32_t gs_csr_weighted_blocks_plan(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                    const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                    int64_t workspace_bytes, int64_t* counts_dev, void* stream);
int32_t gs_csr_weighted_blocks_fill(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds, int32_t n_layers,
                                    const int32_t* fanouts, uint64_t seed, uint64_t call, void* workspace,
                                    int64_t workspace_bytes, const int64_t* counts, int32_t* const* src_ids,
                                    int64_t* const* indptr_out, int32_t* const* indices_out, int32_t* const* rows_out,
                                    void* stream);
int32_t gs_csr_weighted_blocks_fill_offsets(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                            int64_t n_nodes, int64_t nnz, const int32_t* seeds, int64_t n_seeds,
                                            int32_t n_layers, const int32_t* fanouts, uint64_t seed, uint64_t call,
                                            void* workspace, int64_t workspace_bytes, const int64_t* counts,
                                            int32_t* const* src_ids, int64_t* const* indptr_out,
                                            int32_t* const* indices_out, int32_t* const* rows_out,
                                            int32_t* const* offsets_out, void* stream);
int32_t gs_csr_sample_rows_weighted(const int64_t* indptr, const int32_t* indices, const float* sample_weight,
                                    int64_t n_nodes, int64_t nnz, int32_t k, uint64_t seed, uint64_t call, int32_t layer,
                                    void* workspace, int64_t workspace_bytes, int64_t* out_indptr,
                                    int32_t* out_indices /* may be NULL */, void* stream);

/* tf.nn.l2_normalize(x, 1)   reference graphsage/models.py:368-370, supervised_models.py:85 */
int32_t gs_l2_normalize_rows(float* x, int64_t n, int32_t C, int64_t ldx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GRAPHSAGE_B200_H_ */
