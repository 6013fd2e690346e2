/*
 * b200flow.h — C ABI of libb200flow.so: the H100 (sm_90a) hot path of the
 * flow-classification pipeline that biagiom/spark-network-traffic-classifier
 * drives through pyspark.ml.
 *
 * The reference has no FFI of its own: its operator API is the pyspark.ml
 * Estimator/Transformer contract exercised at
 *   code/network_traffic_classifier_kdd99.py:34-37,45-46,64,79,82,86-91
 *   code/network_traffic_classifier_cicids17.py:41-46,68,83,86,90-95
 * Each entry point below names the MLlib operator (SURVEY.md §8a row) whose
 * arithmetic it replaces.  The Python shim in
 * spark-network-traffic-classifier_b200/pyspark binds these through ctypes
 * (see INTEGRATION.md for the stub a maintainer would add).
 *
 * Conventions
 *  - every data pointer is a DEVICE pointer owned by the caller unless the
 *    parameter name ends in _host; the library allocates no persistent memory;
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*);
 *    nothing synchronises the host;
 *  - return value: 0 = ok, negative = error (b200flow_last_error() has text);
 *  - rows are `int64_t`; everything else that indexes columns/bins/classes is int32;
 *  - RNG: Philox4x32-10, keyed by (seed, purpose) and counted by GLOBAL row /
 *    (tree,node) so results do not depend on how rows are sharded over GPUs
 *    (spec in DESIGN.md §RNG).
 */
#ifndef B200FLOW_H
#define B200FLOW_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200FLOW_OK            0
#define B200FLOW_ERR_ARG      -1
#define B200FLOW_ERR_CUDA     -2
#define B200FLOW_ERR_LIMIT    -3

/* element types of dense matrices handed to / produced by the library */
#define B200FLOW_F32 0
#define B200FLOW_F64 1

/* ---- encode plan: one descriptor per OUTPUT slot of the assembled vector ---- */
#define B200FLOW_SRC_F32    0  /* numeric field stored as float   */
#define B200FLOW_SRC_F64    1  /* numeric field stored as double  */
#define B200FLOW_SRC_I32    2  /* numeric field stored as int32   */
#define B200FLOW_SRC_INDEX  3  /* int32 dictionary code -> StringIndexer rank, emitted as a number */
#define B200FLOW_SRC_ONEHOT 4  /* int32 dictionary code -> rank; emits (rank == hot) ? 1 : 0       */

typedef struct b200flow_slot {
    int32_t kind;      /* B200FLOW_SRC_*                                             */
    int32_t src_off;   /* byte offset of the source field inside one raw record      */
    int32_t lut_off;   /* INDEX/ONEHOT: first entry of this column's code->rank LUT  */
    int32_t lut_len;   /* INDEX/ONEHOT: dictionary size; code outside [0,len) or rank<0 = invalid */
    int32_t hot;       /* ONEHOT: the rank this slot lights up for                   */
    int32_t reserved;
    double  mean;      /* StandardScaler withMean: subtracted first (0.0 = off)      */
    double  scale;     /* StandardScaler withStd: 1/sigma, or 0 when sigma==0 (1.0 = off) */
} b200flow_slot;       /* 40 bytes */

const char* b200flow_last_error(void);
int  b200flow_version(void);

/* ------------------------------------------------------------------ encode ---
 * R1  StringIndexer.fit  (kdd99.py:34-37, cicids17.py:45): per-code counts of one
 * int32 dictionary-code field of the raw records.  counts[K] (int64) is ADDED to
 * (caller zeroes; multi-GPU: allreduce the K counts).  Codes outside [0,K) are ignored. */
int b200flow_category_counts(const void* records, int64_t n_rows, int32_t row_bytes,
                             int32_t src_off, int32_t K, int64_t* counts, void* stream);

/* the same for up to 8 code fields in ONE pass over the records (a Pipeline of StringIndexers, kdd99.py:34-37): counts is the
 * concatenation [K_0 | K_1 | ...] (int64, zero-initialised by the caller); src_offs / Ks are HOST arrays of n_cols entries;
 * sum(K) <= 8192. */
int b200flow_category_counts_multi(const void* records, int64_t n_rows, int32_t row_bytes, int32_t n_cols,
                                   const int32_t* src_offs_host, const int32_t* Ks_host, int64_t* counts, void* stream);

/* R2+R3+R3b+R3c  StringIndexerModel.transform + OneHotEncoder + StandardScaler +
 * VectorAssembler.transform fused (kdd99.py:37,46; cicids17.py:42,46): raw AoS
 * records -> dense row-major [n_rows, n_out] matrix (out_dtype F32/F64), computed
 * in fp64: out = (value - mean) * scale.
 *   plan        device array of n_out b200flow_slot
 *   lut         device int32 LUT pool (rank per code, -1 = unseen), may be NULL
 *   label_*     optional label column: int32 code field -> rank (int32) in label_out
 *               (label_off < 0: no label); an unseen label marks the row invalid
 *   valid_out   optional uint8[n_rows]: 0 when the row has an unseen code, or
 *               (check_nan != 0) a NaN numeric field  (handleInvalid="skip"/"error")
 * Full tiles move global->shared->global with TMA bulk copies; records and the
 * output must be 16-byte aligned. */
int b200flow_encode(const void* records, int64_t n_rows, int32_t row_bytes,
                    const b200flow_slot* plan, int32_t n_out,
                    const int32_t* lut, int32_t lut_total,
                    int32_t label_off, int32_t label_lut_off, int32_t label_lut_len,
                    int32_t check_nan,
                    void* out, int32_t out_dtype, int32_t* label_out, uint8_t* valid_out,
                    void* stream);

/* R2+R3 feeding R4/R5 without the dense matrix (SURVEY.md 8d "Encode -> bins"; the vector VectorAssembler builds at
 * kdd99.py:45-46 / cicids17.py:41-46 is consumed by RandomForest.run at kdd99.py:79 / cicids17.py:83 only through
 * findSplits and TreePoint.convertToTreeRDD):
 * sample_records = b200flow_sample_rows on raw records: the Bernoulli row sample of findSplits, every sampled row
 * evaluated through the encode plan (F slots) in fp64; round_f32 != 0 rounds each value to float first (the value an
 * f32 feature matrix would have held).  sample is COLUMN-major [F][cap] fp64 as for sample_rows. */
int b200flow_sample_records(const void* records, int64_t n_rows, int32_t row_bytes,
                            const b200flow_slot* plan, int32_t F, const int32_t* lut, int32_t round_f32,
                            uint64_t seed, uint64_t keep_threshold, int64_t row_offset,
                            double* sample, int64_t cap, int32_t* n_sampled, void* stream);

/* encode_bins = b200flow_encode + b200flow_bin_rows in one pass: raw records -> uint8 TreePoint records
 * tp[n_rows][tp_stride] (bin per plan slot, the label's StringIndexer rank at byte F, zero padding), 16-byte words out.
 * bad (int32[2], caller zeroes): bad[0] += categorical cells outside [0, arity) / non-integral (binned to a value no
 * left-set contains), bad[1] += NaN numeric cells (when check_nan) + unseen dictionary codes.  label_out optional. */
int b200flow_encode_bins(const void* records, int64_t n_rows, int32_t row_bytes,
                         const b200flow_slot* plan, int32_t F, const int32_t* lut, int32_t lut_total,
                         int32_t label_off, int32_t label_lut_off, int32_t label_lut_len,
                         int32_t check_nan, int32_t round_f32,
                         int32_t thr_f32 /* != 0: every continuous slot's value is exactly a float (f32 field with mean 0 / scale 1, or
                                            round_f32): the search then runs on thresholds rounded DOWN to float — the same bins */,
                         const double* thresholds, const int32_t* n_thr, const int32_t* arity, int32_t max_bins,
                         uint8_t* tp, int32_t tp_stride, int32_t* label_out, int32_t* bad, void* stream);

/* R3c  StandardScaler.fit (ml/feature/StandardScaler.scala [MLlib]; north_star encode, not called by kdd99.py/cicids17.py): per-column shifted power sums of a dense [n, D] matrix
 * (leading dimension ld elements): sum[d] += Σ(x-shift[d]), sumsq[d] += Σ(x-shift[d])².
 * shift may be NULL (=0).  Two calls (shift = 0, then shift = mean) give the
 * corrected two-pass variance; multi-GPU: allreduce the 2·D doubles between them. */
int b200flow_column_moments(const void* x, int32_t dtype, int64_t n_rows, int32_t D, int64_t ld,
                            const double* shift, double* sum, double* sumsq, void* stream);

/* --------------------------------------------------------------- tree prep ---
 * R4  RandomForest.findSplits (inside fit: kdd99.py:79, cicids17.py:83), sampling half: Bernoulli(keep_threshold / 2^32) row
 * sample keyed by (seed, global row); gathers the sampled rows of the dense feature
 * matrix into a COLUMN-major fp64 buffer sample[F][cap]; *n_sampled is advanced
 * atomically (caller zeroes; rows beyond cap are counted but not stored). */
int b200flow_sample_rows(const void* x, int32_t dtype, int64_t n_rows, int32_t F, int64_t ld,
                         uint64_t seed, uint64_t keep_threshold, int64_t row_offset,
                         double* sample, int64_t cap, int32_t* n_sampled, void* stream);

/* R4  findSplitsForContinuousFeature: for every continuous feature (arity[f]==0)
 * sort its n_s samples (in place, sample[f*cap .. +n_s)), run-length the distinct
 * values and walk MLlib's stride rule -> thresholds[f*(max_bins-1) ..], n_thr[f].
 * Categorical features (arity>0) get n_thr = 0.  scratch: F * pow2ceil(n_s) doubles. */
int b200flow_find_splits(double* sample, int64_t cap, int32_t n_s, int32_t F,
                         const int32_t* arity, int32_t max_bins,
                         double* thresholds, int32_t* n_thr,
                         const int32_t* n_s_dev /* NULL, or the device-side sample count (then n_s is a host upper bound) */,
                         void* stream);

/* R5  TreePoint.convertToTreeRDD/findBin: dense features (+ int32 labels, may be NULL)
 * -> binned TreePoint records tp[n][tp_stride] (uint8): bytes [0,F) = bin per feature
 * (continuous: lower_bound over thresholds; categorical: (int)x), byte F = label.
 * bad_rows (int32, caller zeroes) counts rows with a categorical value outside
 * [0,arity) or non-integral (MLlib raises). */
int b200flow_bin_rows(const void* x, int32_t dtype, int64_t n_rows, int32_t F, int64_t ld,
                      const double* thresholds, const int32_t* n_thr, const int32_t* arity,
                      int32_t max_bins, const int32_t* labels,
                      uint8_t* tp, int32_t tp_stride, int32_t* bad_rows, void* stream);

/* helper of R5-R7 inside RandomForestClassifier.fit (kdd99.py:79, cicids17.py:83) and of R9 (kdd99.py:82); no MLlib counterpart — exact because the histograms are integer sums.  Row de-duplication (flow records repeat massively: KDD99 has 4.9 M rows but ~1.07 M distinct ones).  Rows whose TreePoint
 * records (first key_bytes bytes: bins + label) are identical are interchangeable for the trees: uid[row] = index of the
 * row's unique record (numbered in order of each group's first row), tp_unique[U][tp_stride] = the unique records,
 * *n_unique = U (device scalar).  Scratch (caller-owned): table/minrow int32[table_cap] (power of two >= 2*n_rows),
 * slot_of/rep/flag int32[n_rows], pos int64[n_rows+1]. */
int b200flow_dedup_rows(const uint8_t* tp, int64_t n_rows, int32_t tp_stride, int32_t key_bytes,
                        int32_t* table, int32_t* minrow, int64_t table_cap, int32_t* slot_of, int32_t* rep,
                        int32_t* flag, int64_t* pos, int64_t* n_unique, int32_t* uid, uint8_t* tp_unique, void* stream);

/* R6  BaggedPoint.convertToBaggedRDD (inside fit: kdd99.py:79, cicids17.py:83): W[tree][uid[row]] += Poisson weight of (tree, global row).  poisson_cdf: 32 increasing
 * uint32 thresholds, weight = #{k: cdf[k] != 2^32-1 && r >= cdf[k]} with r = word tree%4 of Philox(seed,'BAGG', row, tree/4);
 * NULL = no bagging (weight 1 per row, numTrees==1); poisson_cdf_host = the same 32 values in host memory (the first
 * thresholds travel as kernel arguments).  uid NULL = identity.  perm (optional) = the rows grouped by unique id
 * (b200flow_group_rows); uid is then given in that order (uperm): a duplicate group is a run of adjacent lanes and costs one
 * RED per warp and tree.  W uint32[T][n_unique], caller zeroes. */
int b200flow_bag_weights(uint64_t seed, int32_t T, int64_t row_offset, int64_t n_rows,
                         const uint32_t* poisson_cdf, const uint32_t* poisson_cdf_host,
                         const int32_t* uid, const int32_t* perm, int64_t n_unique, uint32_t* W, void* stream);

/* R6 helper (BaggedPoint.convertToBaggedRDD, inside fit: kdd99.py:79, cicids17.py:83): counting sort of the rows by unique id: perm[p] = row, uperm[p] = uid[perm[p]] (non-decreasing).  Scratch: gsize/cursor
 * int32[n_unique], goff int64[n_unique+1]. */
int b200flow_group_rows(const int32_t* uid, int64_t n_rows, int64_t n_unique, int32_t* gsize, int64_t* goff,
                        int32_t* cursor, int32_t* perm, int32_t* uperm, void* stream);

/* R6 (BaggedPoint.convertToBaggedRDD, inside fit: kdd99.py:79, cicids17.py:83): entries of every tree = its non-zero (unique record, summed weight) pairs in unique-id order.  Pass 1: non-zeros per
 * (tree, block of 1024 uniques) -> blk_cnt[T][n_blocks]. */
int b200flow_bag_count(const uint32_t* W, int32_t T, int64_t n_unique, int32_t* blk_cnt, void* stream);

/* R6 (inside fit: kdd99.py:79), pass 2: given blk_off = exclusive scan of blk_cnt (int64, tree-major) write the entries; one entry = 8 bytes
 * {uint32 unique record index, uint32 weight}. */
int b200flow_bag_fill(const uint32_t* W, int32_t T, int64_t n_unique, const int64_t* blk_off, void* ent, void* stream);

/* (no MLlib counterpart; inside fit: kdd99.py:79, cicids17.py:83) exclusive prefix sum utilities used by the trainer (single launch, any n) */
int b200flow_exclusive_scan_i32_to_i64(const int32_t* in, int64_t n, int64_t* out,
                                       int64_t* total, void* stream);

/* ------------------------------------------------------------ tree growing ---
 * One LEVEL of every tree is processed at once.  An active node is a "slot":
 *   slot_tree[s], slot_nid[s] (MLlib node id: root 1, children 2i/2i+1),
 *   slot_node[s]  index of the node in the forest node pool,
 *   seg_begin/seg_end[s]  its bagged entries inside ent (8-byte {record index, weight} pairs).  */

/* per-node feature subsets (RandomForest.selectNodesToSplit [MLlib]; inside fit: kdd99.py:79, cicids17.py:83): m of F features by a
 * partial Fisher-Yates keyed by (seed, tree, nid), sorted ascending -> subset[s*m..].
 * m == F gives the identity. */
int b200flow_feature_subsets(uint64_t seed, int32_t n_slots, const int32_t* slot_tree,
                             const uint32_t* slot_nid, int32_t F, int32_t m,
                             uint16_t* subset, void* stream);

/* R7  findBestSplits/binSeqOp (ml/tree/impl/RandomForest.scala [MLlib]; inside fit: kdd99.py:79, cicids17.py:83) — HOT LOOP A.  hist[s][j][bin][class] += w for every entry
 * of slot s and every j < m (feature subset[s*m+j]).  hist (uint32) must be zeroed by
 * the caller; layout stride = m * n_bins * C.  chunk_off = exclusive scan over slots of
 * ceil(len/chunk_rows) (int64[n_slots+1]); the grid is one CTA per chunk. */
int b200flow_hist_level(const uint8_t* tp, int32_t tp_stride, int32_t F,
                        const void* ent,
                        int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end,
                        const int64_t* chunk_off, int64_t n_chunks, int32_t chunk_rows,
                        const uint16_t* subset, int32_t m, int32_t n_bins, int32_t C,
                        uint32_t* hist, void* stream);

/* split record written by score_level, one per slot */
typedef struct b200flow_split {
    int32_t  feat;        /* feature index, -1 = no valid split (leaf)                   */
    int32_t  kind;        /* 0 continuous (left iff bin <= bin_thr), 1 categorical (mask) */
    int32_t  bin_thr;     /* continuous: split index s (threshold = thresholds[f][s])     */
    int32_t  flags;       /* bit0 node is leaf, bit1 left child leaf, bit2 right child leaf */
    double   gain;
    double   impurity;    /* of this node                                                 */
    uint64_t mask[4];     /* categorical: bit c set = category c goes left                */
} b200flow_split;         /* 64 bytes */

/* R8  binsToBestSplit / calculateImpurityStats / Gini — HOT LOOP B.  Reads the (all-reduced)
 * histograms, writes split[s], the node's own class counts and both children's class counts
 * (uint32 [n_slots][C] each).  feat_bins[f] = number of bins of feature f; feat_kind[f]:
 * 0 continuous, 1 ordered categorical, 2 unordered categorical (bins = categories).
 * level/max_depth/min_instances/min_info_gain as in MLlib's Strategy. */
int b200flow_score_level(const uint32_t* hist, int32_t n_slots, const uint16_t* subset,
                         int32_t m, int32_t n_bins, int32_t C,
                         const int32_t* feat_bins, const int32_t* feat_kind,
                         int32_t level, int32_t max_depth, int32_t min_instances,
                         double min_info_gain,
                         b200flow_split* split, uint32_t* node_counts,
                         uint32_t* left_counts, uint32_t* right_counts, void* stream);

/* forest node pool (SoA, all trees in one pool; roots are nodes 0..T-1) */
typedef struct b200flow_node {
    int32_t feat;      /* -1 = leaf                                      */
    int32_t kind_bin;  /* kind<<16 | bin_thr                             */
    int32_t left;      /* pool index of left child; right = left + 1     */
    uint32_t nid;      /* MLlib node id                                  */
} b200flow_node;       /* 16 bytes */

/* R8 driver side (LearningNode growth in RandomForest.findBestSplits, ml/tree/impl/RandomForest.scala [MLlib]; inside fit:
 * kdd99.py:79, cicids17.py:83).  Grows the pool by one level: for each slot writes its node record (+ mask, counts), creates
 * two children per split (counts from left/right_counts), and emits the next level's slots for
 * the non-leaf children (next_* arrays, capacity 2*n_slots; next_parent = parent slot*2+side;
 * child_slot[2*s+side] = index of that child among the next slots, -1 when it is a leaf; may be NULL).
 * counters: int64[8] header {node pool size (in/out), number of next slots (out), overflow flag (out: 1 =
 * pool_capacity too small, nothing written), pool size before the call, 4 entries free for the caller}
 * followed by 2*ceil(n_slots/256) int32 of scratch. */
int b200flow_grow_level(int32_t n_slots, const int32_t* slot_tree, const uint32_t* slot_nid,
                        const int32_t* slot_node, const b200flow_split* split,
                        const uint32_t* node_counts, const uint32_t* left_counts,
                        const uint32_t* right_counts, int32_t C,
                        b200flow_node* nodes, uint64_t* node_mask, uint32_t* pool_counts,
                        int32_t* node_tree, int64_t pool_capacity,
                        int32_t* next_tree, uint32_t* next_nid, int32_t* next_node,
                        int32_t* next_parent, int32_t* child_slot, int64_t* counters, void* stream);

/* R7 unfused fallback (the row -> node relation MLlib recomputes with predictImpl in findBestSplits; inside fit: kdd99.py:79, cicids17.py:83): routes every entry of every split slot to its child: left entries grow up from seg_begin,
 * right entries grow down from seg_end inside the same range of the destination buffers;
 * cursors[s*2+{0,1}] (int32, caller zeroes) end as (#left, #right).  Entries of children
 * that are leaves are dropped. */
int b200flow_partition_level(const uint8_t* tp, int32_t tp_stride,
                             const void* ent, void* ent_out,
                             int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end,
                             const int64_t* chunk_off, int64_t n_chunks, int32_t chunk_rows,
                             const b200flow_split* split, int32_t* cursors, void* stream);

/* R7 (inside fit: kdd99.py:79, cicids17.py:83) fused with the row routing: partition_level(L) + hist_level(L+1) in ONE pass — every entry's TreePoint
 * record is gathered once, routed by its parent's split and accumulated into its CHILD's histogram
 * (hist_next[child_slot][j][bin][class], child feature subsets in subset_next, caller zeroes hist_next and
 * cursors).  The kernel is persistent (132 x k CTAs); each warp gathers the records of its entries with
 * asynchronous copies into a private shared-memory tile and there is no CTA barrier except when the parent slot
 * changes.
 * b200flow_route_hist_config() picks the launch shape for a level shape (host-only, no device needed): it returns
 * 1 and writes chunk_rows (entries per routing chunk = warps x entries per warp step; pass it to plan_route and to
 * route_hist_level) and m_pass (subset features whose two child histograms share shared memory; m_pass < m means
 * ceil(m / m_pass) feature passes over the entries, only the first of which routes — DecisionTree nodes, whose
 * histograms cover every feature), or returns 0 when even one feature's pair of child histograms does not fit
 * (then use partition_level followed by hist_level).
 * flags bit 0: route — write the kept entries to ent_out and count them in cursors (8-byte aligned: a slot's pair is
 * advanced by one 64-bit atomic); without it only the child
 * histograms are built (ent_out / cursors may be NULL): the level-0 pass, whose segments do not change, and the
 * pass that builds the deepest scored level, whose entries are never read again. */
int b200flow_route_hist_config(int32_t F, int32_t m, int32_t n_bins, int32_t C,
                               int32_t rec_bytes /* packed record size, 0: byte records */, int32_t* chunk_rows, int32_t* m_pass);
int b200flow_route_hist_level(const uint8_t* tp, int32_t tp_stride, int32_t F,
                              const int32_t* field_desc /* device, F + 1 descriptors: tp holds packed records of tp_stride
                                                           bytes (b200flow_pack_records); NULL: byte records */,
                              const void* ent, void* ent_out,
                              int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end,
                              const int64_t* chunk_off, const int64_t* n_chunks_dev /* = chunk_off[n_slots], on the device */,
                              int64_t n_chunks_max /* host upper bound: sizes the scratch and the table launch */,
                              int32_t chunk_rows,
                              const b200flow_split* split, const int32_t* child_slot, int32_t* cursors,
                              void* chunk_scratch /* 16 bytes per chunk (n_chunks_max), 16-byte aligned */,
                              const uint16_t* subset_next, int32_t m, int32_t n_bins, int32_t C,
                              uint32_t* hist_next, int32_t flags, void* stream);

/* Bit-packed TreePoint records for the level kernel (host-only, no device needed).  Field f < F holds a bin of feature f
 * (feat_bins[f] values), field F the label (C values); each takes max(1, bits(values - 1)) bits, fields are placed
 * first-fit-decreasing into 32-bit words and none crosses a word.  desc[f] (host, F + 1) = word | shift << 8 | mask << 16.
 * *rec_bytes = the words rounded up to 16 bytes when that is at most 64 bytes and at least one 16-byte granule below the
 * staged byte record, else 0 (keep the byte records; always for F > 255, which the level kernel does not take).  The layout
 * depends only on (feat_bins, C). */
int b200flow_packed_layout(int32_t F, const int32_t* feat_bins, int32_t C, int32_t* desc, int32_t* rec_bytes);
/* byte records tp[n_rows][tp_stride] -> packed[n_rows][rec_bytes] (desc on the device, as b200flow_packed_layout wrote it) */
int b200flow_pack_records(const uint8_t* tp, int32_t tp_stride, int64_t n_rows, int32_t F, const int32_t* desc,
                          int32_t rec_bytes, uint32_t* packed, void* stream);

/* routing plan of a scored level: n_chunks[s] = ceil(len(s) / chunk_rows) for a split parent with at least one non-leaf
 * child, else 0 (its exclusive scan is route_hist_level's chunk_off); also scatters split[s].gain into node_gain[slot_node[s]]
 * when node_gain != NULL (TreeEnsembleModel.featureImportances needs the gains; MLlib keeps them in the Node objects). */
int b200flow_plan_route(int32_t n_slots, const b200flow_split* split, const int64_t* seg_begin, const int64_t* seg_end,
                        int32_t chunk_rows, const int32_t* slot_node, double* node_gain, int32_t* n_chunks,
                        int32_t* cursors /* NULL, or int32[2 * n_slots] zeroed here for the routing pass */, void* stream);

/* R7/R8 bookkeeping (inside fit: kdd99.py:79, cicids17.py:83): segment table of the next level from the parents' ranges and the partition cursors */
int b200flow_next_segments(int32_t n_next /* or an upper bound */, const int64_t* n_next_dev /* NULL or the device-side count */,
                           const int32_t* next_parent,
                           const int64_t* seg_begin, const int64_t* seg_end,
                           const int32_t* cursors, int64_t* next_begin, int64_t* next_end,
                           void* stream);

/* R9 preparation (LeafNode / ImpurityCalculator.prob in ml/tree/Node.scala [MLlib]; fit at kdd99.py:79): leaf payloads: prob[node][k] = counts[k] / Σcounts (fp64 true division), 0 if Σ == 0 */
int b200flow_finalize_forest(int64_t n_nodes, const uint32_t* pool_counts, int32_t C,
                             double* leaf_prob, void* stream);

/* ----------------------------------------------------------------- predict ---
 * per-tree compact layout for b200flow_predict_forest, built once per model in two calls.  Tree t (t < T; pool nodes of
 * other trees are ignored) owns the 8-byte words [tree_off[t], tree_off[t+1]) of `layout`: its nodes in pool order (8-byte
 * records, child and payload offsets local to the tree), the C fp64 votes of its leaves (leaf_prob, or pool_counts as fp64
 * when dt_mode != 0) and the left-set masks of its categorical splits.
 * b200flow_forest_layout_size fills tree_off[T+1] (tree_off[T] = the words `layout` must hold) and the int32 scratch
 * [2*n_nodes + 4*T]; b200flow_build_forest_layout then writes `layout` (16-byte aligned) from the same scratch. */
int b200flow_forest_layout_size(const b200flow_node* nodes, const int32_t* node_tree, int64_t n_nodes, int32_t T, int32_t C,
                                int32_t* scratch, int64_t* tree_off, void* stream);
int b200flow_build_forest_layout(const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                 const uint32_t* pool_counts, const int32_t* node_tree, int64_t n_nodes, int32_t T, int32_t C,
                                 int32_t dt_mode, const int32_t* scratch, const int64_t* tree_off, uint64_t* layout, void* stream);

/* R9  RandomForestClassificationModel.transform (kdd99.py:82, cicids17.py:86) — HOT LOOP C.  Walks all T trees of the
 * compact layout for every binned row; raw[n][C] = Σ_t leaf votes (tree order, fp64, from 0.0), prob = raw/Σraw,
 * pred = first argmax.  The votes are leaf_prob, or the leaf class counts when the layout was built with dt_mode != 0
 * (DecisionTreeClassifier).  raw/prob may be NULL.  Each tree is staged whole in shared memory (the first words of a tree
 * larger than the buffer; the rest read from global).  F = features (bins tp[row][0..F-1]). */
int b200flow_predict_forest(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const uint64_t* layout,
                            const int64_t* tree_off, int32_t T, int32_t C, double* raw, double* prob, double* pred, void* stream);

/* R9 helper (model.transform, kdd99.py:82, cicids17.py:86): out[i] = src[idx[i]] for rows of row_bytes (multiple of 4): spreads the predictions computed once per UNIQUE test record
 * (b200flow_dedup_rows) back to the rows. */
int b200flow_gather_rows(const void* src, int32_t row_bytes, const int32_t* idx, int64_t n_rows, void* out, void* stream);

/* R10 MulticlassMetrics (evaluator.evaluate: kdd99.py:86-91, cicids17.py:90-95): confusion matrix cm[label*C + pred] += 1 (int64, caller zeroes).
 * pred / label are fp64 columns (as in the prediction DataFrame). */
int b200flow_confusion(const double* pred, const double* label, int64_t n_rows, int32_t C,
                       int64_t* cm, void* stream);

/* shared-memory table for b200flow_predict_grid_confusion / _scores: top[tree][nid] (16-byte b200flow_node,
 * [T][2^top_levels], entry 0 unused) = the tree's node with MLlib node id nid < 2^top_levels.  Built once per model; the
 * walk of the first top_levels levels then reads shared memory instead of issuing one L1 request per lane and level. */
int b200flow_build_top_nodes(const b200flow_node* nodes, const int32_t* node_tree, int64_t n_nodes, int32_t T,
                             int32_t top_levels, void* top, void* stream);

/* Model selection (CrossValidator / TrainValidationSplit over numTrees x maxDepth, DESIGN.md §5a): confusion matrices of
 * every truncated forest (first T_i trees, cut at depth d_j) on the validation records, from ONE walk of each tree.
 * tp[n_rows][tp_stride] = UNIQUE binned records with the label at byte F; mult[n_rows] = rows per unique record.
 * tree_cuts_host: 1 <= T_1 < ... < T_I <= T (I <= 256); depth_cuts_host: 0 <= d_1 < ... < d_J <= 30.
 * cm int64 [I][J][cm_side][cm_side] (cm_side >= C, caller zeroes): cm[i][j][label][pred] += mult, where pred is what
 * b200flow_predict_forest gives for the truncated forest; labels >= cm_side are not counted.  max_depth_cuts_per_launch: 0 = as many
 * as shared memory holds (the result does not depend on it).
 * top_nodes: NULL or the table of b200flow_build_top_nodes with top_levels levels. */
int b200flow_predict_grid_confusion(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const int32_t* mult,
                                    const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                    const uint32_t* pool_counts, int32_t T, int32_t C, int32_t dt_mode,
                                    const void* top_nodes, int32_t top_levels, const int32_t* tree_cuts_host,
                                    int32_t n_tree_cuts, const int32_t* depth_cuts_host, int32_t n_depth_cuts,
                                    int32_t cm_side, int32_t max_depth_cuts_per_launch, int64_t* cm, void* stream);
/* The same walk, for BinaryClassificationEvaluator: scores double [I][J][n_rows] (device) gets votes[1] of every truncated
 * forest for every record — rawPrediction[1] of that (tree_cuts[i], depth_cuts[j]) forest fitted on its own, bit for bit.
 * C >= 2; the records' label byte and multiplicities are not read. */
int b200flow_predict_grid_scores(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows,
                                 const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                 const uint32_t* pool_counts, int32_t T, int32_t C, int32_t dt_mode,
                                 const void* top_nodes, int32_t top_levels, const int32_t* tree_cuts_host,
                                 int32_t n_tree_cuts, const int32_t* depth_cuts_host, int32_t n_depth_cuts,
                                 int32_t max_depth_cuts_per_launch, double* scores, void* stream);

/* BinaryClassificationMetrics (BinaryClassificationEvaluator areaUnderROC / areaUnderPR, DESIGN.md §5b).
 * b200flow_binary_counts: S segments (1 <= S <= 65536, S * n < 2^32) of n fp64 scores, segment s at scores + s * score_stride;
 * int32 positive / negative counts per item at pos / neg + s * count_stride + i (count_stride 0: every segment shares them).
 * Items with pos + neg == 0 are ignored; a NaN score with a non-zero count is counted into *n_nan (device int64) and ignored.
 * Writes the distinct scores of every segment in DESCENDING order (-0.0 == +0.0) with their summed counts:
 * d_score / d_pos / d_neg [S][cap] (cap >= n, entries past n_distinct[s] untouched) and n_distinct int64 [S] (device).
 * scratch: device, 256-byte aligned, b200flow_binary_counts_scratch(S, n) bytes (host-only query, no device needed).
 * Integer counts throughout: the result does not depend on the order of the items. */
int b200flow_binary_counts_scratch(int32_t S, int64_t n, int64_t* scratch_bytes);
int b200flow_binary_counts(const double* scores, int64_t score_stride, const int32_t* pos, const int32_t* neg,
                           int64_t count_stride, int32_t S, int64_t n, void* scratch, int64_t scratch_bytes,
                           double* d_score, int64_t* d_pos, int64_t* d_neg, int64_t cap, int64_t* n_distinct,
                           int64_t* n_nan, void* stream);
/* b200flow_binary_curve: distinct triples (as binary_counts writes them) -> auc[S][2] = {areaUnderROC, areaUnderPR} and the
 * curve points c_score / c_tp / c_fp [S][cap] (score, cumulative positives, cumulative negatives), c_n[S] of them.  num_bins
 * >= 0 down-samples as Spark does (g = n_distinct / num_bins; g >= 2 keeps ranks g-1, 2g-1, ... and the last).  Each area
 * is summed sequentially from 0.0 in curve order.  work: 2 * S * cap doubles of device scratch.  A segment with no
 * distinct score gets NaN areas. */
int b200flow_binary_curve(const double* d_score, const int64_t* d_pos, const int64_t* d_neg, int64_t cap,
                          const int64_t* n_distinct, int32_t S, int32_t num_bins, double* auc, double* c_score,
                          int64_t* c_tp, int64_t* c_fp, int64_t* c_n, double* work, void* stream);

/* ---------------------------------------------------------------- clustering ---
 * KMeans (k-means|| init + Lloyd) and ClusteringEvaluator (silhouette), DESIGN.md §5c.  Features are dense row-major f64
 * x[n_rows][ld], 1 <= D <= 256.
 * b200flow_kmeans_assign: centers [k][D] -> cluster[i] = first argmin center, dist[i] = its squared distance, summed in
 * feature order from 0.0 as acc = acc + t*t, t = x_j - c_j (no FMA, no norm trick). */
int b200flow_kmeans_assign(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* centers, int32_t k,
                           int32_t* cluster, double* dist, void* stream);
/* Grouped sums.  Global rows are cut into chunks of 4096 (chunk b = global rows [4096 b, 4096 (b + 1))).  Rows
 * [0, n_rows) of values [n_rows][ld] are global rows row_offset + i; they touch b200flow_group_sums_chunks(row_offset, n_rows)
 * chunks (host-only query), starting with chunk row_offset / 4096.  partials [n_chunks][G][W] (device): the sequential sum, in
 * row order from +0.0, of column w of the rows of that chunk with ids[i] == g (ids NULL: G == 1, every row); +0.0 where a
 * chunk has no member.  counts int64 [G] (optional, caller zeroes) += the member rows; ids outside [0, G) are skipped.
 * G <= 4096.  b200flow_group_sums_chain: totals [G][W] (device, in: the running totals, e.g. +0.0) += partials of chunk 0,
 * then chunk 1, ... sequentially, in place. */
int b200flow_group_sums_chunks(int64_t row_offset, int64_t n_rows, int64_t* n_chunks);
int b200flow_group_sums(const double* values, int64_t ld, const int32_t* ids, int64_t n_rows, int32_t W, int32_t G,
                        int64_t row_offset, double* partials, int64_t* counts, void* stream);
int b200flow_group_sums_chain(const double* partials, int64_t n_chunks, int32_t G, int32_t W, double* totals, void* stream);
/* keys[i] = (w0 << 32 | w1) ^ 2^63 as int64 (signed order = unsigned key order), (w0, w1) = the first two words of
 * Philox(seed, 'KMNS', (row_lo, row_hi, 0, 0)) of global row row_offset + i: the first-center / random-init key. */
int b200flow_kmeans_row_keys(uint64_t seed, int64_t row_offset, int64_t n_rows, int64_t* keys, void* stream);
/* k-means|| round `step` >= 1: flag[i] = u < ((2.0 * cost[i]) * k) / sum_cost, u = ((w0 << 21) | (w1 >> 11)) * 2^-53 from
 * Philox(seed, 'KMNS', (row_lo, row_hi, step, 0)). */
int b200flow_kmeans_select(uint64_t seed, int64_t row_offset, int64_t n_rows, int32_t step, const double* cost, int32_t k,
                           double sum_cost, uint8_t* flag, void* stream);
/* silhouette coefficient per row from the cluster statistics Y [G][D] (feature sums), psi [G] (sums of squared norms),
 * N int64 [G] (sizes; 0 = absent): d(g) = (norms[i] + psi[g] / N[g]) - (2 * (x . Y[g])) / N[g], dot sequential in j;
 * a = d(own) * N / (N - 1), b = min over the other present clusters; out = 1 - a/b (a < b), b/a - 1 (a > b), else 0, and 0
 * when the row's cluster has one member. */
int b200flow_silhouette_rows(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* norms, const int32_t* cluster,
                             const double* Y, const double* psi, const int64_t* N, int32_t G, double* out, void* stream);
/* BisectingKMeans, DESIGN.md §5t.  Distances as b200flow_kmeans_assign's; no cross-row reduction, so each row's outputs
 * depend on that row and the centers alone.
 * b200flow_bkm_assign: rows carry a dense node number node[i]; slot_of_node [num_nodes] gives the dividing slot s of a node
 * (-1: not dividing).  centers [2m][D] are the children of the m slots (slot s: 2s left, 2s+1 right), present uint8 [2m].
 * child[i] = 2s or 2s+1, the present child with the smaller squared distance (strict <: a tie goes left), or -1 when the
 * row's node is not dividing or neither child is present.  prev (optional, int32 [n_rows], -1 or a child index of the row's
 * slot): dist_prev[i] = the squared distance to centers[prev[i]] (0.0 where prev[i] or the row's slot is -1), the cost of
 * the previous assignment against the centers recomputed from it. */
int b200flow_bkm_assign(const double* x, int64_t n_rows, int32_t D, int64_t ld, const int32_t* node, int32_t num_nodes,
                        const int32_t* slot_of_node, const double* centers, int32_t m, const uint8_t* present, const int32_t* prev,
                        int32_t* child, double* dist_prev, void* stream);
/* b200flow_bkm_predict: the cluster tree as node arrays left, right [num_nodes] (-1: absent), leaf [num_nodes] (the leaf
 * ordinal, -1 for an internal node) and centers [num_nodes][D], num_nodes <= 4095, depth <= 63.  From root, each internal
 * node sends the row to the existing child with the smaller squared distance (a tie goes to the first, left, child).
 * out_leaf[i] = the leaf ordinal reached, out_dist[i] = the squared distance to that leaf's center (a root that is a leaf
 * works). */
int b200flow_bkm_predict(const double* x, int64_t n_rows, int32_t D, int64_t ld, const int32_t* left, const int32_t* right,
                         const int32_t* leaf, const double* centers, int32_t num_nodes, int32_t root, int32_t* out_leaf,
                         double* out_dist, void* stream);

/* ---------------------------------------------------------- neural network ---
 * MultilayerPerceptronClassifier, DESIGN.md §5d.  layers (host int32 [n_layers]) = [D, h_1, ..., h_k, K]: affine +
 * sigmoid per hidden layer, affine on top (softmax in the loss).  weights (device f64 [P]) in Spark's layout: per layer W
 * (out x in, column-major: (o, i) at o + i*out) then b (out), P = sum (in*out + out).  Features x [n_rows][ld] are f32
 * (x_dtype B200FLOW_F32) or f64 (B200FLOW_F64), converted to f64 before any arithmetic: equal values give equal bits.
 * Limits: at most 8 affine layers; sum over layers of ceil(out/8) * ceil((in+1)/8) <= 256 (the gradient's 8x8 tiles,
 * held in registers); 8 * (sum of padded W blocks + 32 * sum of padded activation widths) <= 226 KiB of shared memory
 * (b200flow_mlp_config reports both; [78,100,50,15] and [119,64,32,5] fit).
 * b200flow_mlp_config (host-only): *n_params = P, *smem_bytes = the kernels' dynamic shared memory; error beyond limits. */
int b200flow_mlp_config(const int32_t* layers, int32_t n_layers, int64_t* n_params, int64_t* smem_bytes);
/* partials [n_chunks][P + 1] (device; n_chunks = b200flow_group_sums_chunks(row_offset, n_rows)): for each 4096-row
 * global chunk the rows [0, n_rows) (global rows row_offset + i) touch, slot 0 = the sum over its rows of
 * logsumexp(z) - z[y] (z = the top affine output, labels int32 in [0, K)), slots 1..P = the sum of the gradient of that
 * loss in the weights' layout.  A chunk's partial depends only on which of its rows are present. */
int b200flow_mlp_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, const int32_t* labels,
                           const int32_t* layers, int32_t n_layers, const double* weights, int64_t row_offset,
                           double* partials, void* stream);
/* raw [n_rows][K] f64: the top affine output (Spark 3's predictRaw) of every row. */
int b200flow_mlp_forward(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, const int32_t* layers, int32_t n_layers,
                         const double* weights, double* raw, void* stream);

/* ------------------------------------------------------------ linear SVM ---
 * LinearSVC and OneVsRest(LinearSVC), DESIGN.md §5j.  Features x [n_rows][ld] are f32 (x_dtype B200FLOW_F32) or f64
 * (B200FLOW_F64), converted to f64 before any arithmetic; 1 <= D <= 255, K >= 1 class columns.  Column k's weights
 * weights[k] = [beta_k (D), b_k] (device f64 [K][D + 1]) act on [xs, 1].  Classes are cut into blocks of at most 256
 * columns whose gradient tiles fit in registers (8 * ceil(kb / 8) * ceil((D + 1) / 8) <= 256 * 8); a column's results do
 * not depend on K, on the other columns or on its block.
 * b200flow_svc_config (host-only): *block_classes = columns per block, *class_blocks = blocks, *smem_bytes = the kernels'
 * dynamic shared memory; error beyond the limits. */
int b200flow_svc_config(int32_t D, int64_t K, int32_t* block_classes, int32_t* class_blocks, int64_t* smem_bytes);
/* partials [n_chunks][K][D + 2] (device; n_chunks = b200flow_group_sums_chunks(row_offset, n_rows)): for each 4096-row
 * global chunk the rows [0, n_rows) (global rows row_offset + i) touch, and each column k, with xs_j = x_j * inv_std[j]
 * (one rounding), y' = +1 if labels[i] == positives[k] (int32 [K], device) else -1 and m = [xs, 1] . weights[k] (fp64
 * tensor cores, features in ascending order): slot 0 = the sum over the chunk's rows in row order from +0.0 of
 * 1 - y' m where that is > 0, slots 1..D+1 = the sum of -y' [xs, 1] over the same rows (fp64 tensor cores over the rows
 * in row order).  A chunk's partial depends only on which of its rows are present. */
int b200flow_svc_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const int32_t* labels,
                           const int32_t* positives, int64_t K, const double* inv_std, const double* weights,
                           int64_t row_offset, double* partials, void* stream);
/* raw [n_rows][K] f64: raw[i][k] = [x_i, 1] . weights[k] (unscaled), with b200flow_svc_loss_grad's margin arithmetic. */
int b200flow_svc_margins(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int64_t K,
                         const double* weights, double* raw, void* stream);

/* ------------------------------------------------------------ linear regression ---
 * LinearRegression, DESIGN.md §5n.  Features x [n_rows][ld] f32 or f64 (converted to f64 first), 1 <= D <= 255; labels y
 * [n_rows] f64; shift [D] (NULL: no centring) and inv [D] f64; w [D] f64; b_sigma = [b, sigma] f64 (read in huber mode
 * only), all device.  xs_j = (x_j - shift[j]) * inv[j] (no shift: x_j * inv[j]); m = sum_j xs_j w_j over j ascending.
 * partials [n_chunks][D + 3] (device; n_chunks = b200flow_group_sums_chunks(row_offset, n_rows)): for each 4096-row global
 * chunk the rows touch, sums over the chunk's present rows in row order from +0.0 of
 *   slot 0: the row's loss term, slots 1..D: a xs, slot D + 1: a, slot D + 2: the sigma derivative, where
 *   B200FLOW_LINREG_SQUARED: d = m - (y - y_shift) y_scale, loss d^2, a = d, sigma derivative 0;
 *   B200FLOW_LINREG_HUBER: z = (y - m - b) / sigma; |z| <= epsilon: loss sigma + z^2 sigma, a = -2z, derivative 1 - z^2;
 *     otherwise loss sigma + (2 epsilon |z| - epsilon^2) sigma, a = -2 epsilon sign(z), derivative 1 - epsilon^2.
 * A chunk's partial depends only on which of its rows are present and on the inputs. */
#define B200FLOW_LINREG_SQUARED 0
#define B200FLOW_LINREG_HUBER 1
int b200flow_linreg_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* y,
                              const double* shift, const double* inv, double y_shift, double y_scale, const double* w,
                              const double* b_sigma, double epsilon, int32_t mode, int64_t row_offset, double* partials,
                              void* stream);
/* AFTSurvivalRegression (Weibull), DESIGN.md §5q: b200flow_linreg_loss_grad's staging, margin and partials layout with
 * y = log_t [n_rows] f64 (the log of the survival time), censor [n_rows] int32 (1 when the event was observed, 0 when the
 * row is censored) and b_sigma = [b, sigma, log sigma] f64, all device.  z = (log t - m - b) / sigma and delta = censor:
 * loss delta log sigma - delta z + e^z, a = (delta - e^z) / sigma, sigma derivative (with respect to log sigma)
 * delta + (delta - e^z) z. */
int b200flow_aft_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* log_t,
                           const int32_t* censor, const double* shift, const double* inv, const double* w,
                           const double* b_sigma, int64_t row_offset, double* partials, void* stream);

/* ------------------------------------------------------------ generalized linear regression ---
 * GeneralizedLinearRegression, DESIGN.md §5o.  Features x [n_rows][ld] f32 or f64 (converted to f64 first), 1 <= D <= 255;
 * labels y, prior weights `weight` and offsets `offset` [n_rows] f64 (weight NULL: 1.0, offset NULL: 0.0); coef [D] f64; all
 * device.  family / link are the codes below; variance_power is tweedie's V(mu) = mu^p, link_power the power link's
 * (0: log).  Rows [0, n_rows) are global rows row_offset + i.  With m = x . coef (eight lane sums over j = s mod 8 in
 * ascending j, combined ((p0 + p4) + (p2 + p6)) + ((p1 + p5) + (p3 + p7))), eta = (m + intercept) + offset and
 * mu = project(unlink(eta)):
 *   B200FLOW_GLM_INIT: z = link(initialize(y, weight)) - offset, w = weight; rows_out [n_rows][2] = (z, w);
 *   B200FLOW_GLM_REWEIGHT: z = (eta - offset) + (y - mu) g'(mu), w = weight / (g'(mu)^2 V(mu)); rows_out = (z, w);
 *     partials [n_chunks][D + 2] of both: sum w, sum w x_j (j < D), sum w z;
 *   B200FLOW_GLM_SUMMARY (coef NULL: mu = mu_const, eta = link(mu) for every row): rows_out NULL or [n_rows][4] = the
 *     deviance, pearson, working and response residuals; partials [n_chunks][8] = sum weight, sum weight y, the deviance,
 *     the squared pearson residuals, the AIC log-likelihood terms, and for gamma sum weight log y, sum weight y / mu and
 *     sum weight log mu (0 otherwise);
 *   B200FLOW_GLM_PREDICT: rows_out [n_rows][2] = (mu, eta); y, weight and partials are not read.
 * n_chunks = b200flow_group_sums_chunks(row_offset, n_rows); each partial sums the chunk's present rows in row order from
 * +0.0, so it depends only on which of its rows are present and on the inputs. */
#define B200FLOW_GLM_GAUSSIAN 0
#define B200FLOW_GLM_BINOMIAL 1
#define B200FLOW_GLM_POISSON 2
#define B200FLOW_GLM_GAMMA 3
#define B200FLOW_GLM_TWEEDIE 4
#define B200FLOW_GLM_IDENTITY 0
#define B200FLOW_GLM_LOG 1
#define B200FLOW_GLM_INVERSE 2
#define B200FLOW_GLM_LOGIT 3
#define B200FLOW_GLM_PROBIT 4
#define B200FLOW_GLM_CLOGLOG 5
#define B200FLOW_GLM_SQRT 6
#define B200FLOW_GLM_POWER 7
#define B200FLOW_GLM_INIT 0
#define B200FLOW_GLM_REWEIGHT 1
#define B200FLOW_GLM_SUMMARY 2
#define B200FLOW_GLM_PREDICT 3
int b200flow_glm_rows(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* y,
                      const double* weight, const double* offset, const double* coef, double intercept, double mu_const,
                      int32_t family, int32_t link, double variance_power, double link_power, int32_t mode,
                      int64_t row_offset, double* rows_out, double* partials, void* stream);

/* ------------------------------------------------------------ isotonic regression ---
 * IsotonicRegression, DESIGN.md §5p.  Row i (0 <= i < n < 2^32) is (label[i * label_stride], feature[i * feature_stride],
 * weight[i * weight_stride]) with the feature f32 (B200FLOW_F32) or f64 (B200FLOW_F64) and label / weight f64 (weight
 * NULL: 1.0), all device.  checks int64 [2] (device) = the rows with a non-finite label, feature or weight, and the rows
 * with a negative weight; the fit is only meaningful when both are 0.  Rows with weight 0 are dropped.  isotonic == 0 fits
 * an antitonic model (labels negated, then the predictions).  Writes the model, *n_out (device int64) increasing
 * boundaries and their predictions, into boundaries / predictions [n] (device f64); an empty input gives *n_out = 0.
 * The model is Spark's one-partition result (makeUnique, PAV, compress, PAV again) with PAV run as a chunked merge tree:
 * chunk 0 takes the library's chunk size, any other value (<= 2^30) forces that one.  The bits depend only on the rows, in
 * order, and on the chunk size.
 * scratch: device, 256-byte aligned, b200flow_isotonic_scratch(n) bytes (host-only query, no device needed).
 * b200flow_isotonic_predict: out[i] = the model's prediction at x[i * stride] (f32 or f64): java.util.Arrays.binarySearch
 * over the K >= 1 boundaries, the first or last prediction outside them, the hit's on a hit, else
 * y1 + (y2 - y1) * (x - x1) / (x2 - x1).  A NaN x predicts the last prediction. */
int b200flow_isotonic_scratch(int64_t n, int64_t* scratch_bytes);
int b200flow_isotonic_fit(const void* feature, int32_t feature_dtype, int64_t feature_stride, const double* label,
                          int64_t label_stride, const double* weight, int64_t weight_stride, int64_t n, int32_t isotonic,
                          int64_t chunk, void* scratch, int64_t scratch_bytes, double* boundaries, double* predictions,
                          int64_t* n_out, int64_t* checks, void* stream);
int b200flow_isotonic_predict(const void* x, int32_t x_dtype, int64_t stride, int64_t n, const double* boundaries,
                              const double* predictions, int64_t K, double* out, void* stream);

/* ------------------------------------------------------------ column statistics, quantiles, transforms ---
 * Imputer, RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer and Bucketizer, DESIGN.md §5s.  Every call reads
 * D >= 1 columns of n rows: value (r, c) is at base + r * row_bytes + cols[2c] with dtype cols[2c + 1] (B200FLOW_F32,
 * B200FLOW_F64 or B200FLOW_I32), cols int32 [2 D] on the device; row_bytes and the offsets are multiples of 4 (an f64
 * field needs only 4-byte alignment, as in a raw record).  Values are widened to f64.  A value is missing when it is NaN or,
 * with has_missing, == missing.
 * b200flow_column_stats: stats int64 [6][D] (device) = per column the count of non-missing values, of +inf and of -inf;
 * the smallest and largest ordered key (Java's Double.compare order, -0.0 < 0.0, stored as key ^ 2^63 so that int64 order
 * is key order; INT64_MAX / INT64_MIN without values); the bits of the largest finite |x| (0 without one).  Sum the first
 * three rows, min the fourth and max the last two over ranks.
 * b200flow_column_sums: limbs int64 [D][4] (device, caller zeroes) += the 32-bit limbs (top one signed) of
 * rint(x 2^shift[c]) over column c's finite non-missing values, shift int32 [D] on the device; n < 2^31.
 * b200flow_quantile_hist / b200flow_quantile_step: exact rank select over T targets, ordered by column then rank.  state
 * int64 [6 T + 2 D + 1] (device): ranks [T] (1-based, among the column's non-missing values in Double.compare order),
 * then T words the library owns, then the values [T] (f64, written by the last step), then the columns [T], then T + 2 D + 1
 * words the library owns.  The caller fills ranks and columns, calls step(select = 0), then for pass = 0 .. 7: hist (which
 * zeroes hist int64 [group_bound][256] and counts the pass's digits of every group; group_bound >= the groups of the pass,
 * at most min(T, active columns 256^pass); at most 48 groups count in shared memory, more in global memory), sums hist over
 * ranks, and step(select = 1).
 * b200flow_bucketize: out [n][D] f64 = Spark's Bucketizer.binarySearchForBuckets of value (r, c) over column c's splits
 * splits[split_off[c] .. split_off[c + 1]) (device, strictly increasing, K >= 3 each): NaN -> K - 1 and flags[r] = 0
 * (flags uint8 [n], else 1); x == the last split -> the last bucket, K - 2; else
 * java.util.Arrays.binarySearch's hit or insertion point - 1.  checks int64 [2] (device) = NaN values, values outside the
 * splits (their output is meaningless and the caller must raise).
 * b200flow_impute_fill: column c is copied to outs[c] (a device pointer to n contiguous values of the column's own dtype,
 * outs uint64 [D] on the device) with every missing value replaced by the bits fill_bits[c] (device uint64 [D]; the low 32
 * bits for f32 / i32 columns).
 * b200flow_min_max: out [n][D] f64 = (x - emin[c]) * scale[c] + lo when scale[c] != 0, else constant, and NaN for NaN
 * (emin, scale f64 [D] device), no FMA.
 * b200flow_mode_keys: keys [n] (device) = the ordered keys of the non-missing values of one column col = {offset, dtype}
 * (host int32 [2]), -0.0 counted as 0.0, in any order; *count (device int64) = their number.
 * b200flow_mode: out f64 [2] (device) = the most frequent value among keys [M] (device, M >= 1, overwritten; the padding
 * key 0xFFFFFFFFFFFFFFFF is ignored) with the smallest one on ties, and its count; NaN and 0 when every key is padding.
 * scratch: device, 256-byte aligned, b200flow_mode_scratch(M) bytes (host-only query). */
#define B200FLOW_I32 2
int b200flow_column_stats(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols, int32_t has_missing,
                          double missing, int64_t* stats, void* stream);
int b200flow_column_sums(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols, int32_t has_missing,
                         double missing, const int32_t* shift, int64_t* limbs, void* stream);
int b200flow_quantile_hist(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                           int32_t has_missing, double missing, int64_t T, int64_t* state, int32_t pass, int64_t group_bound,
                           int64_t* hist, void* stream);
int b200flow_quantile_step(int64_t T, int32_t D, int64_t* state, const int64_t* hist, int32_t select, void* stream);
int b200flow_bucketize(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols, const double* splits,
                       const int32_t* split_off, double* out, uint8_t* flags, int64_t* checks, void* stream);
int b200flow_impute_fill(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols, int32_t has_missing,
                         double missing, const uint64_t* fill_bits, const uint64_t* outs, void* stream);
int b200flow_min_max(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols, const double* emin,
                     const double* scale, double lo, double constant, double* out, void* stream);
int b200flow_mode_keys(const void* base, int64_t row_bytes, int64_t n, const int32_t* col, int32_t has_missing, double missing,
                       uint64_t* keys, int64_t* count, void* stream);
int b200flow_mode_scratch(int64_t M, int64_t* scratch_bytes);
int b200flow_mode(uint64_t* keys, int64_t M, void* scratch, int64_t scratch_bytes, double* out, void* stream);

/* ------------------------------------------------------------ factorization machines ---
 * FMClassifier and OneVsRest(FMClassifier), DESIGN.md §5k.  Features x [n_rows][ld] are f32 (x_dtype B200FLOW_F32) or
 * f64 (B200FLOW_F64), converted to f64 before any arithmetic; 1 <= D <= 255, factor_size F >= 1, K >= 1 class columns.
 * Column k's weights weights[k] = [V_k (D x F, row-major), w_k (D), b_k] (device f64 [K][D (F + 1) + 1]).  With
 * s_f = sum_i v_if x_i and q_f = sum_i x_i^2 v_if^2 (fp64 tensor cores, features in ascending order), the raw value is
 * r = (b + x . w) + 1/2 (s_0^2 - q_0) + 1/2 (s_1^2 - q_1) + ...  Classes are cut into blocks whose gradient tiles fit in
 * registers and whose products fit in shared memory; a column's results do not depend on K, on the other columns or on
 * its block.  Every D <= 255 with F <= 32 fits.
 * b200flow_fm_config (host-only): *block_classes = classes per block, *class_blocks = blocks, *smem_bytes = the kernels'
 * dynamic shared memory; error beyond the limits. */
int b200flow_fm_config(int32_t D, int32_t factor_size, int64_t K, int32_t* block_classes, int32_t* class_blocks,
                       int64_t* smem_bytes);
/* partials [n_chunks][K][D (F + 1) + D + 3] (device; n_chunks = b200flow_group_sums_chunks(row_offset, n_rows)): for each
 * 4096-row global chunk the rows [0, n_rows) (global rows row_offset + i) touch, and each column k, over the chunk's rows
 * in the mini-batch (all rows when mini_batch_fraction == 1, else those whose Philox draw, purpose FMMB, key seed
 * batch_seed, counter (global row lo, hi, 0, 0), word 0, is < floor(fraction 2^32)), with y = 1 if labels[i] ==
 * positives[k] (int32 [K], device) else 0 and g = 1 / (1 + exp(-r)) - y: slot 0 = the loss sum in row order from +0.0
 * (log1pExp(-r) if y = 1, else log1pExp(r)), slot 1 = the row count, then sum g x_i s_f at 2 + i F + f, sum g x_i at
 * 2 + D F + i, sum g at 2 + D F + D, and sum g x_i^2 at 3 + D F + D + i (fp64 tensor cores over the rows in row order).
 * The factor gradient is the first block minus v_if times the last.  A chunk's partial depends only on which of its rows
 * are present. */
int b200flow_fm_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int32_t factor_size,
                          const int32_t* labels, const int32_t* positives, int64_t K, const double* weights,
                          double mini_batch_fraction, uint64_t batch_seed, int64_t row_offset, double* partials, void* stream);
/* raw [n_rows][K] f64: raw[i][k] = r of row i under weights[k], with b200flow_fm_loss_grad's arithmetic. */
int b200flow_fm_raw(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int32_t factor_size, int64_t K,
                    const double* weights, double* raw, void* stream);
/* FMRegressor, DESIGN.md §5r: b200flow_fm_loss_grad's partials for one column (K = 1) under the squared error, with labels
 * y [n_rows] f64 (device, used as they are): g = 2 (r - y), loss (r - y)^2.  The layout, the mini-batch draw and the
 * summation order are b200flow_fm_loss_grad's. */
int b200flow_fm_regression_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D,
                                     int32_t factor_size, const double* labels, const double* weights,
                                     double mini_batch_fraction, uint64_t batch_seed, int64_t row_offset, double* partials,
                                     void* stream);

/* ------------------------------------------------------------ mixture models ---
 * GaussianMixture (full covariance), DESIGN.md §5g.  Features x [n_rows][ld] f64, rows [0, n_rows) are global rows
 * row_offset + i; 1 <= D <= 256, 1 <= k <= 64.  A partial row of chunk b (b counted from the first 4096-row chunk the rows
 * touch, as for b200flow_group_sums) is [LL, then per component i: W_i, S_i [D], Q_i [D(D+1)/2]], width
 * 1 + k (1 + D + D(D+1)/2); Q_i is packed upper, (a, b) with a <= b at a + b(b+1)/2.
 * b200flow_gmm_estep: means [k][D], roots [k][D][D], log_consts [k] = log w_i + u_i.  Per row: q_i = sum over j in order of
 * y_j^2, y = roots_i (x - means_i); s_i = log_consts_i - 0.5 q_i; t_i = logaddexp(log 2^-52, s_i); resp [n_rows][k] =
 * exp(t_i - logsumexp(t)); pred [n_rows] = first argmax of resp; partials[b][0] = the sum of logsumexp(t) over the chunk's
 * rows in row order from +0.0.  resp, pred and partials may each be NULL. */
int b200flow_gmm_estep(const double* x, int64_t n_rows, int32_t D, int64_t ld, int32_t k, const double* means,
                       const double* roots, const double* log_consts, int64_t row_offset, double* resp, int32_t* pred,
                       double* partials, void* stream);
/* b200flow_gmm_moments: the rest of each partial row from resp [n_rows][k]: W_i = sum r_i, S_i = sum r_i x,
 * Q_i = sum r_i x x^T over the chunk's rows (fp64 tensor-core contractions in a fixed order; slot 0 is left alone). */
int b200flow_gmm_moments(const double* x, int64_t n_rows, int32_t D, int64_t ld, int32_t k, const double* resp,
                         int64_t row_offset, double* partials, void* stream);

/* ------------------------------------------------------ dimensionality reduction ---
 * PCA and Pearson correlation, DESIGN.md §5h.  Features x [n_rows][ld] f64, 1 <= D <= 256.
 * b200flow_centered_gram: rows [0, n_rows) are global rows row_offset + i.  partials [n_chunks][D(D+1)/2] (n_chunks =
 * b200flow_group_sums_chunks(row_offset, n_rows)): for each 4096-row global chunk the rows touch, the packed upper triangle
 * of (X - shift)^T (X - shift) over the chunk's present rows, (a, b) with a <= b at a + b(b+1)/2; shift [D] (NULL: zeros) is
 * subtracted as the rows are staged.  fp64 tensor-core contractions over the rows in row order; a chunk's partial depends
 * only on which of its rows are present. */
int b200flow_centered_gram(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* shift, int64_t row_offset,
                           double* partials, void* stream);
/* b200flow_weighted_centered_gram: as b200flow_centered_gram with a row weight w [n_rows] f64: the packed upper triangle
 * of (X - shift)^T W (X - shift), each staged (x_b - shift_b) multiplied by its row's weight as the contraction loads it
 * (GeneralizedLinearRegression's IRLS, DESIGN.md §5o). */
int b200flow_weighted_centered_gram(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* shift,
                                    const double* w, int64_t row_offset, double* partials, void* stream);
/* b200flow_pca_project: out [n_rows][k] = x pc, pc [D][k] row-major, 1 <= k <= 256; out[i][j] accumulates x[i][a] pc[a][j]
 * over a in ascending order (fp64 tensor cores), so a row's output depends on that row and pc alone, not on its position. */
int b200flow_pca_project(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* pc, int32_t k, double* out,
                         void* stream);

/* ------------------------------------------------------------ feature selection ---
 * Chi-square, ANOVA and F-value tests and the selectors built on them, DESIGN.md §5i.  Values x [n_rows][ld] f64, finite
 * (the caller checks), 1 <= W <= 256.
 * b200flow_distinct_values: per column w, the set of value keys in an open-addressed table tables[w][32768] (device, the
 * caller fills every slot with 0xFFFFFFFFFFFFFFFF, a NaN pattern that is never a key).  A key is the value's bits with -0.0
 * mapped to +0.0.  counts int32 [W] (caller zeroes) += the keys this call inserted; overflow int32 [W] (caller zeroes) is set
 * to 1 once counts[w] passes 10000, after which column w takes no more keys.  The table's contents are a set: which slot
 * holds a key depends on the launch. */
int b200flow_distinct_values(const double* x, int64_t n_rows, int32_t W, int64_t ld, uint64_t* tables, int32_t* counts,
                             int32_t* overflow, void* stream);
/* b200flow_dictionary_ids: ids[i] = the index of values[i * ld] in dict [L] (device, ascending, no duplicates, -0.0 equal to
 * +0.0 as in any f64 comparison), -1 when it is absent.  1 <= L <= 10000. */
int b200flow_dictionary_ids(const double* values, int64_t n_rows, int64_t ld, const double* dict, int32_t L, int32_t* ids,
                            void* stream);
/* b200flow_contingency_counts: counts int64 [n_values][L] (device, caller zeroes) += the rows with x[i][w] == dicts[v]
 * and label_ids[i] == l at row v = dict_off[w] + index of the value in dicts[dict_off[w] .. dict_off[w + 1]) (each range
 * ascending); dict_off int32 [W + 1] (device), n_values = dict_off[W] (host copy) <= 2^26 / L.  Rows whose value is absent
 * or whose label id is outside [0, L) are not counted.  1 <= L <= 256.  Integer counts: exact for any launch. */
int b200flow_contingency_counts(const double* x, int64_t n_rows, int32_t W, int64_t ld, const int32_t* label_ids, int32_t L,
                                const double* dicts, const int32_t* dict_off, int64_t n_values, int64_t* counts, void* stream);
/* b200flow_group_centered_moments: rows [0, n_rows) are global rows row_offset + i.  For each 4096-row global chunk they
 * touch (n_chunks = b200flow_group_sums_chunks(row_offset, n_rows)), partials [n_chunks][G][W'] (device):
 *   y NULL:  W' = W, [c][g][w] = sum over the chunk's rows with ids[i] == g of (x[i][w] - centers[g][w])^2;
 *   y [n_rows] (then G == 1 and ids is ignored): W' = 2W + 1, [c][0][w] = sum (x[i][w] - centers[w])^2,
 *            [c][0][W + w] = sum (x[i][w] - centers[w]) (y[i] - y_center), [c][0][2W] = sum (y[i] - y_center)^2.
 * Each sum runs over the rows in row order from +0.0 without FMA, so a chunk's partial depends only on which of its rows
 * are present.  ids NULL: every row is in group 0 (G == 1).  centers [G][W] (device).  1 <= G <= 256. */
int b200flow_group_centered_moments(const double* x, int64_t n_rows, int32_t W, int64_t ld, const int32_t* ids, int32_t G,
                                    const double* centers, const double* y, double y_center, int64_t row_offset,
                                    double* partials, void* stream);

/* ---------------------------------------------------------------- naive Bayes ---
 * NaiveBayes (multinomial, complement, bernoulli, gaussian), DESIGN.md §5u.  Features x [n_rows][ld] are dense row-major,
 * f32 (x_dtype 0) or f64 (x_dtype 1), widened exactly to f64; 1 <= D <= 256 and 1 <= C <= 256 classes.
 * b200flow_nb_moments: rows [0, n_rows) are global rows row_offset + i with class labels[i] (rows whose label is outside
 * [0, C) are left out) and weight weights[i] (NULL: 1.0).  For each 4096-row global chunk they touch (n_chunks =
 * b200flow_group_sums_chunks(row_offset, n_rows)), partials (device):
 *   centers NULL:      [n_chunks][C][D + 1], [c][j] = sum w x_j and [c][D] = sum w over the chunk's rows of class c;
 *   centers [C + 1][D]: [n_chunks][C + 1][D], [c][j] = sum w (x_j - centers[c][j])^2 over the rows of class c and
 *                      [C][j] = sum w (x_j - centers[C][j])^2 over every row with a label in [0, C).
 * Each sum runs over the rows in row order from +0.0 without FMA, w (t t) for a centred term.  bad int64 [5] (optional,
 * caller zeroes; counted by the pass without centers only) += the number of values x that are {non-finite, negative, not 0
 * or 1}, of weights that are negative, NaN or infinite, and of labels outside [0, C). */
int b200flow_nb_moments(const void* x, int32_t x_dtype, int64_t n_rows, int32_t D, int64_t ld, const int32_t* labels,
                        const double* weights, int32_t C, const double* centers, int64_t row_offset, double* partials,
                        int64_t* bad, void* stream);
/* b200flow_nb_raw: raw [n_rows][C] (device f64); each value is one sum over j in feature order from 0.0, without FMA:
 *   model 0 (gaussian): raw[i][c] = c0[c] - (s + c1[c]) / 2, s = sum (d d) / b[c][j], d = x_j - a[c][j];
 *   model 1 (linear):   raw[i][c] = sum x_j a[c][j], then + c0[c];
 *   model 2:            model 1, then raw[i][c] -= m + log(sum over the present classes in class order of exp(raw[i][c] - m)),
 *                       m the row's largest present value.
 * a, b [C][D], c0, c1 [C] (device f64; b and c1 gaussian only); classes with present[c] == 0 get -inf.  bad int64 [1]
 * (optional, caller zeroes) += the number of values x that are not exactly 0 or 1. */
int b200flow_nb_raw(const void* x, int32_t x_dtype, int64_t n_rows, int32_t D, int64_t ld, int32_t model, const double* a,
                    const double* b, const double* c0, const double* c1, const uint8_t* present, int32_t C, double* raw,
                    int64_t* bad, void* stream);

/* ------------------------------------------------------- gradient-boosted trees ---
 * GBTClassifier (binary, LogLoss), DESIGN.md §5e.  The regression trees reuse the forest's level loop: feature_subsets,
 * partition_level, next_segments, grow_level (with C = 6: a node's int64 stats {Σw, Σw·q, Σw·q2} travel as six opaque
 * uint32 words in pool_counts) and predict (C = 1 over the payloads).  Residuals are on a fixed-point grid: rq int64
 * [n][2] = {q, q2}, q = rint(r 2^S), q2 = rint((q 2^-S)^2 2^S2), S = 60 - ceil(log2 max(n_global, 2)), S2 = S - 2, so every
 * histogram sum is an exact integer below 2^62.  rq must be 16-byte aligned.
 * b200flow_gbt_hist_level: hist int64 [n_slots][m][n_bins][3] (caller zeroes) += {w, w·q, w·q2} of every entry of the slot
 * at the bin of each subset feature; entries, segments and the chunk table as for b200flow_hist_level. */
int b200flow_gbt_hist_level(const uint8_t* tp, int32_t tp_stride, const void* ent, const int64_t* rq, int32_t n_slots,
                            const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off, int64_t n_chunks,
                            int32_t chunk_rows, const uint16_t* subset, int32_t m, int32_t n_bins, int64_t* hist, void* stream);
/* OneVsRest(GBTClassifier), DESIGN.md §5f: b200flow_gbt_hist_level over the slots of K classes' trees at once.  rq is
 * int64 [K][class_rows][2] and slot s reads {q, q2} of its records from block slot_class[s]; tp and the entries are shared. */
int b200flow_gbt_hist_level_classes(const uint8_t* tp, int32_t tp_stride, const void* ent, const int64_t* rq, int64_t class_rows,
                                    const int32_t* slot_class, int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end,
                                    const int64_t* chunk_off, int64_t n_chunks, int32_t chunk_rows, const uint16_t* subset,
                                    int32_t m, int32_t n_bins, int64_t* hist, void* stream);
/* Variance split scoring, one CTA per slot: split[s] as score_level writes it (categorical features are ordered by centroid
 * sum/count; a child is a leaf at level + 1 == max_depth or when its variance is below 2^-52), and the int64 stats [3] of
 * the node and of both children (zero when there is no split). */
int b200flow_gbt_score_level(const int64_t* hist, int32_t n_slots, const uint16_t* subset, int32_t m, int32_t n_bins,
                             const int32_t* feat_bins, const int32_t* feat_kind, int32_t S, int32_t S2, int32_t level,
                             int32_t max_depth, int32_t min_instances, double min_info_gain, b200flow_split* split,
                             int64_t* node_stats, int64_t* left_stats, int64_t* right_stats, void* stream);
/* payload[i] = tree_weight[node_tree[i]] * ((Σw·q 2^-S) / Σw) for the n_nodes pool nodes (stats int64 [n_nodes][3]) */
int b200flow_gbt_leaf_values(int64_t n_nodes, const int64_t* stats, const int32_t* node_tree, const double* tree_weight,
                             int32_t S, double* payload, void* stream);
/* per binned record (label at byte F, 0 or 1; y = 2 label - 1): tree < 0 sets margin = +0.0 and rq to y's grid values;
 * tree >= 0 walks that tree (root = pool node `tree`), margin += payload of its leaf, rq = grid of 4y / (1 + exp(2y margin))
 * (csrc/portable_exp.h; a NaN residual becomes 0). */
int b200flow_gbt_update(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const b200flow_node* nodes,
                        const uint64_t* node_mask, const double* payload, int32_t tree, int32_t S, int32_t S2, double* margin,
                        int64_t* rq, void* stream);
/* b200flow_gbt_update for n_classes relabelled problems at once (OneVsRest): margin f64 [K][n_rows], rq int64 [K][n_rows][2];
 * class k's label is (label byte == k) and its tree of iteration `tree` is rooted at pool node k n_iter + tree.  tree < 0
 * initialises every class. */
int b200flow_gbt_update_classes(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, int32_t n_classes,
                                const b200flow_node* nodes, const uint64_t* node_mask, const double* payload, int32_t tree,
                                int32_t n_iter, int32_t S, int32_t S2, double* margin, int64_t* rq, void* stream);
/* GBTClassificationModel output from the margins: raw [n][2] = {-F, F}, prob [n][2] = {1 / (1 + exp(2F)), 1 - that},
 * pred = F > 0; raw / prob / pred may be NULL. */
int b200flow_gbt_output(const double* margin, int64_t n_rows, double* raw, double* prob, double* pred, void* stream);

/* -------------------------------------------------- regression (csrc/regression.cu, DESIGN.md §5l) ---
 * Labels y' = y 2^-E on the grid of the variance-tree kernels above: q = rint(y' 2^S), q2 = rint((q 2^-S)^2 2^S2); the
 * level loop passes S - E and S2 - 2E to b200flow_gbt_score_level, so gains and leaf values come out in label units. */
/* out int64[2] (caller zeroes): [0] += labels that are NaN or ±inf, [1] = max |y| over the finite labels (as its bits);
 * tp != NULL: the 8 bytes of y[i] are written to bytes [offset, offset + 8) of record i (tp_stride bytes each) */
int b200flow_reg_labels(const double* y, int64_t n_rows, uint8_t* tp, int32_t tp_stride, int32_t offset, int64_t* out,
                        void* stream);
/* totals int64[n_trees] (caller zeroes) += Σ_u W[t][u] over the bag weights W int32 [n_trees][n_unique] */
int b200flow_reg_tree_weights(const int32_t* W, int32_t n_trees, int64_t n_unique, int64_t* totals, void* stream);
/* rq int64 [n_rows][2] (16-byte aligned) = {q, q2} of each record's label: read from its bytes [offset, offset + 8) when tp
 * != NULL, else y[u]; 0 < S, S2 <= 62 */
int b200flow_reg_grid(const uint8_t* tp, int32_t tp_stride, int32_t offset, const double* y, int64_t n_rows, int32_t E,
                      int32_t S, int32_t S2, int64_t* rq, void* stream);
/* table f64 [n_nodes][width]: [0] = (Σw·q 2^-S) / Σw of each node's stats int64 [n_nodes][3]; width 2 adds [1] = the
 * node's variance (Σw·q2 2^-S2 - (Σw·q 2^-S)^2 / Σw) / Σw, 0 for an empty node */
int b200flow_reg_leaf_table(int64_t n_nodes, const int64_t* stats, int32_t S, int32_t S2, double* table, int32_t width,
                            void* stream);
/* out[i] = in[i] / d for n_rows doubles, IEEE-rounded (in == out allowed): the forest's prediction, Σ over trees / T */
int b200flow_reg_divide(const double* in, int64_t n_rows, double d, double* out, void* stream);
/* GBTRegressor (DESIGN.md §5m).  payload[i] = weight * ((Σw·q 2^-S) / Σw) for the pool nodes i < n_nodes with
 * node_tree[i] == tree (stats int64 [n_nodes][3]); the other nodes' payloads are left as they are.  -1022 < S < 1022. */
int b200flow_gbr_leaf_values(int64_t n_nodes, const int64_t* stats, const int32_t* node_tree, int32_t tree, double weight,
                             int32_t S, double* payload, void* stream);
/* per unique record u (label y[u], or the 8 bytes at [offset, offset + 8) of its record when y == NULL): tree < 0 sets
 * margin = +0.0 and resid = y; tree >= 0 walks that tree (root = pool node `tree`), margin += its leaf's payload, and
 * resid = 2 (y - margin) (loss 0, squared) or (y - margin < 0 ? -1 : +1) (loss 1, absolute).  A NaN resid becomes 0.
 * max_out int64[1] (caller zeroes) = max |resid| over the records, as its bits. */
int b200flow_gbr_update(const uint8_t* tp, int32_t tp_stride, int32_t offset, const double* y, int64_t n_rows,
                        const b200flow_node* nodes, const uint64_t* node_mask, const double* payload, int32_t tree, int32_t loss,
                        double* margin, double* resid, int64_t* max_out, void* stream);
/* RegressionEvaluator terms of each row: mode 0 {y, y^2, (y - p)^2, |y - p|}, mode 1 {(y - mean)^2, (p - mean)^2}.
 * out int64[5] (caller zeroes): [0] += rows with a non-finite label, prediction or term, [1 + k] = max |term k| (bits). */
int b200flow_reg_eval_max(const double* label, const double* pred, int64_t n_rows, int32_t mode, double mean, int64_t* out,
                          void* stream);
/* limbs int64 [4][4] (caller zeroes): limbs[k][j] += Σ_rows limb j of rint(term k 2^sh_k) as a two's-complement 128-bit
 * integer (32-bit limbs, the top one signed); rows counted by b200flow_reg_eval_max are skipped.  n_rows < 2^31. */
int b200flow_reg_eval_sums(const double* label, const double* pred, int64_t n_rows, int32_t mode, double mean, int32_t sh0,
                           int32_t sh1, int32_t sh2, int32_t sh3, int64_t* limbs, void* stream);

/* -------------------------------------------------- either side of the path ---
 * DataFrame.randomSplit (kdd99.py:52, cicids17.py:56): split id per row from a uniform keyed
 * by (seed, global row): first k with u < cum_bounds[k] (n_splits <= 32).  out uint8[n]. */
int b200flow_random_split(uint64_t seed, int64_t row_offset, int64_t n_rows,
                          const double* cum_bounds_host, int32_t n_splits, uint8_t* split_id,
                          void* stream);

/* SURVEY 8f rank 1 (Dataset.randomSplit kdd99.py:52, where cicids17.py:30-35, handleInvalid=skip cicids17.py:41): stable row compaction (where / handleInvalid="skip" / one randomSplit part):
 * keeps rows with flag[i] == want; out_rows gets the kept rows' row_bytes-sized records in
 * order.  Counting per block and the scan happen inside; scratch: (n_blocks+1) int64 followed by
 * n_blocks int32, n_blocks = ceil(n/1024); *n_kept (device int64) receives the count. */
int b200flow_compact_rows(const void* rows, int64_t n_rows, int32_t row_bytes,
                          const uint8_t* flag, int32_t want, void* out_rows,
                          int64_t* scratch, int64_t* n_kept, void* stream);

/* -------------------------------------------------- CSV text -> flow records ---
 * SURVEY 8f rank 3: replaces `spark.read.csv(path, inferSchema=True, header=...)` at kdd99.py:25 and
 * cicids17.py:19-20.  The caller copies the file's bytes to the device (16-byte aligned) and owns every buffer.
 * Unquoted fields, ',' delimiter, LF or CRLF line ends, blank lines skipped (univocity's default).
 * Column classes follow Spark's inference order; parsing is exact (Java parseInt / parseDouble semantics, see
 * csrc/csv_number.h) or the field is counted in bad[] — never approximated. */
#define B200FLOW_CSV_NULL   0
#define B200FLOW_CSV_INT32  1
#define B200FLOW_CSV_INT64  2   /* inference only: such a column is read as DOUBLE (the record layout has no int64) */
#define B200FLOW_CSV_DOUBLE 3
#define B200FLOW_CSV_STRING 4   /* stored as an int32 dictionary code; -1 = null */
typedef struct b200flow_csv_col {
    int32_t type;       /* B200FLOW_CSV_INT32 / DOUBLE / STRING */
    int32_t rec_off;    /* byte offset of the field inside the output record (4-byte aligned) */
    int32_t str_index;  /* STRING: which dictionary table (0..n_string_columns-1) */
    int32_t reserved;
} b200flow_csv_col;
/* bad[8] (device, zero-initialised except [1] and [5] = ~0): [0] rows whose field count != n_cols, [1] first such row,
 * [2] rows longer than 4096 bytes, [3] fields that do not parse as their column's type, [4] numeric literals outside the
 * exact range (more than 19 digits that straddle a rounding boundary, |exponent| > 27), [5] first (row << 16 | col) of
 * [3]/[4], [6] dictionary table full, [7] dictionary lookups that failed (hash collision). */

/* line index, step 1: counts[b] = non-empty lines starting in text block b (4096 bytes each); flags[0] bit 0 = a '"' was seen */
int b200flow_csv_count_lines(const uint8_t* text, int64_t n_bytes, int32_t* counts, unsigned long long* flags, void* stream);
/* line index, step 2: bases = exclusive prefix sum of counts (int64); row_starts[i] = byte offset of non-empty line i */
int b200flow_csv_line_starts(const uint8_t* text, int64_t n_bytes, const int64_t* bases, int64_t* row_starts, void* stream);
/* inferSchema: col_class[c] = max over rows of the field's class (atomicMax into zeroed int32[n_cols]), col_null[c] = 1 if
 * any field of the column is empty.  flags: bit 0 ignoreLeadingWhiteSpace, bit 1 ignoreTrailingWhiteSpace. */
int b200flow_csv_infer(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols,
                       int32_t flags, int32_t* col_class, int32_t* col_null, unsigned long long* bad, void* stream);
/* string columns: keys [n_str][2^cap_log2] (zeroed) receive the 64-bit FNV-1a hash of every distinct value, pos_len
 * (filled with INT64_MAX) the smallest (byte offset << 16 | length) at which it occurs — order of first appearance */
int b200flow_csv_dictionary(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols,
                            int32_t flags, const b200flow_csv_col* cols, unsigned long long* keys, long long* pos_len,
                            int32_t cap_log2, unsigned long long* bad, void* stream);
/* fields -> records[n_rows][row_bytes]; slot_code[n_str][2^cap_log2] = dictionary code of each occupied slot (the host
 * assigns codes after reading the tables); a STRING field must byte-equal its slot's first occurrence or bad[7] counts it */
int b200flow_csv_parse(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols,
                       int32_t flags, const b200flow_csv_col* cols, const unsigned long long* keys, const long long* pos_len,
                       const int32_t* slot_code, int32_t cap_log2, void* records, int32_t row_bytes, unsigned long long* bad,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200FLOW_H */
