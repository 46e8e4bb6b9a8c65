/* pfz.h -- C ABI of libpfz.so: the H100 (sm_90a) pairwise string-similarity hot path that
 * drops in behind PolyFuzz's BaseMatcher plugins.
 *
 * The reference (MaartenGr/PolyFuzz @ v0.4.3) is pure Python and has no FFI of its own; its hot
 * path calls third-party native code through Python.  Each entry point below names the reference
 * call site / third-party routine it replaces (file:line into the reference tree, `sk:` =
 * scikit-learn 1.9.0).  INTEGRATION.md shows the ctypes stubs a maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; buffers are caller-allocated
 *     (PyTorch tensors in the shipped host code); the library never frees or retains them, except
 *     for workspaces it is handed explicitly;
 *   - every function returns 0 on success, non-zero on failure; pfz_last_error() then returns a
 *     thread-local human-readable message (CUDA error string included);
 *   - the last argument is the CUDA stream (cudaStream_t passed as void*); all work is enqueued on
 *     it and nothing synchronises unless stated;
 *   - strings travel as UTF-32 code points: `blob` (uint32) + `offsets` (int64, n+1 entries);
 *   - there is NO CPU fallback: on a machine without an sm_90 device the calls fail.
 */
#ifndef PFZ_H
#define PFZ_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PFZ_ABI_VERSION 1

/* flags for the n-gram analyser */
#define PFZ_FLAG_CLEAN         1   /* _clean_string: lower, keep [a-z0-9 ], collapse spaces, strip */
#define PFZ_FLAG_REMOVE_SPACE  2   /* drop n-grams that contain U+0020                            */

/* edit-distance metrics */
#define PFZ_METRIC_LEV       0     /* Levenshtein distance, unit costs                             */
#define PFZ_METRIC_INDEL     1     /* |a|+|b|-2*LCS                                                */
#define PFZ_METRIC_NORM_LEV  2     /* 1 - lev/max(|a|,|b|)                                         */
#define PFZ_METRIC_RATIO     3     /* rapidfuzz fuzz.ratio = (1 - indel/(|a|+|b|))*100             */
#define PFZ_METRIC_JARO      4     /* jellyfish jaro_similarity(from, to), in [0, 1]                */
#define PFZ_METRIC_JARO_WINKLER 5  /* jellyfish jaro_winkler_similarity(from, to), long_tolerance=False */
#define PFZ_METRIC_OSA       6     /* optimal string alignment distance (restricted Damerau-Levenshtein) */
#define PFZ_METRIC_NORM_OSA  7     /* 1 - osa/max(|a|,|b|)                                         */
#define PFZ_METRIC_DL        8     /* unrestricted Damerau-Levenshtein distance (pfz_dl_* only)    */
#define PFZ_METRIC_NORM_DL   9     /* 1 - dl/max(|a|,|b|)                   (pfz_dl_* only)        */

int         pfz_abi_version(void);
const char *pfz_last_error(void);
/* number of CUDA kernels this library has launched in this process (monotonic) */
int64_t     pfz_launch_count(void);
/* device properties the host code needs for launch sizing: sm_count, max dynamic smem per block */
int pfz_device_info(int32_t *sm_count, int32_t *smem_per_block_optin, int32_t *cc_major, int32_t *cc_minor);

/* integer-ALU throughput probe: 8 independent LOP3/IADD chains per thread, sm_count*8 blocks of 256 threads,
 * `iters` x 64 lane-ops per thread.  scratch: uint32[sm_count*8*256] on device.  *lane_ops_host receives the number of
 * 32-bit lane-operations the launch executes; the caller times the launch (CUDA events) -> measured INT32 issue peak,
 * the roofline denominator of K3 (bench.py).  Not on the product path.                                            */
int pfz_int_alu_probe(int32_t iters, uint32_t *scratch, int64_t *lane_ops_host, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K1  char-n-gram TF-IDF vectoriser.
 * Replaces: polyfuzz/models/_tfidf.py:142-146 (_clean_string), :120-139 (_create_ngrams),
 *           :102-118 (_extract_tf_idf) and sk:feature_extraction/text.py:1257-1320 (_count_vocab),
 *           :1204-1216 (_sort_features), :1651-1739 (TfidfTransformer fit/transform),
 *           sk:utils/sparsefuncs_fast.pyx:578-605 (row l2 normalise).
 *
 * An n-gram is represented by an order-preserving integer code: sum_i sym(c_i) * base^(nmax-1-i)
 * with sym >= 1 (0 = "no character"), so integer order == Python string order used for sklearn's
 * alphabetical vocabulary.  Clean mode: fixed alphabet ' '<'0'..'9'<'a'..'z' (base 38).  Raw mode:
 * sym_table[code point] (uint32[0x110000], 0xFFFFFFFF = not in the fitted alphabet), base = A+1.
 * ---------------------------------------------------------------------------------------------- */

/* raw mode alphabet: mark every code point that occurs (present: uint8[0x110000], pre-zeroed) */
int pfz_alphabet_mark(const uint32_t *blob, int64_t n_chars, uint8_t *present, void *stream);

/* Stage A: per string: (clean,) enumerate n-grams, sort, run-length encode.
 *   occ_ptr[r]   (int64[n+1], host-computed upper bound prefix: sum_n max(0, len_r-n+1))
 *   codes/tf     output at occ_ptr[r] .. occ_ptr[r]+row_cnt[r]  (codes ascending, distinct)
 *   long_rows    (int32[n_long], rows whose slot count exceeds PFZ_WARP_ROW_SLOTS; may be NULL)      */
#define PFZ_WARP_ROW_SLOTS 256
#define PFZ_MAX_ROW_SLOTS  8192
int pfz_ngram_rows(const uint32_t *blob, const int64_t *offsets, int32_t n_rows,
                   int32_t ngram_lo, int32_t ngram_hi, int32_t flags,
                   const uint32_t *sym_table, uint32_t base,
                   const int64_t *occ_ptr, const int32_t *long_rows, int32_t n_long,
                   uint64_t *codes, int32_t *tf, int32_t *row_cnt, void *stream);

/* Stage B (fit), small code space (base^nmax <= 2^24): document frequency by direct addressing.
 *   df_dense (int32[code_space], pre-zeroed) accumulates over one or more lists (call once per list) */
int pfz_df_dense(const uint64_t *codes, const int64_t *occ_ptr, const int32_t *row_cnt, int32_t n_rows,
                 int32_t *df_dense, void *stream);
/*   then compact: vocab_keys (ascending codes with df>0), df (int32[V]), rank_dense (int32[code_space],
 *   -1 = absent); *n_vocab_dev (int32 on device).  ws: >= pfz_scan_ws_bytes(code_space) bytes.         */
int pfz_vocab_compact_dense(const int32_t *df_dense, int64_t code_space, uint64_t *vocab_keys, int32_t *df,
                            int32_t *rank_dense, int32_t *n_vocab_dev, void *ws, void *stream);

/* Stage B (fit), large code space: gather all per-row distinct codes of the fit lists into
 * `keys` (uint64[cap_pow2], padded with ~0), sort (bitonic), unique+count.                           */
int pfz_gather_codes(const uint64_t *codes, const int64_t *occ_ptr, const int32_t *row_cnt, int32_t n_rows,
                     uint64_t *keys, int64_t *cursor_dev, void *stream);
int pfz_sort_u64(uint64_t *keys, int64_t n_pow2, void *stream);
int pfz_vocab_from_sorted(const uint64_t *sorted_keys, int64_t n_keys_cap, const int64_t *n_keys_dev,
                          uint64_t *vocab_keys, int32_t *df, int32_t *n_vocab_dev, void *ws, void *stream);

/* idf[v] = table[df[v]] for v < *n_vocab_dev: the host evaluates sklearn's np.log((n+1)/(df+1)) + 1 (sk:feature_extraction/text.py:
 * 1679-1694) once for every possible df = 0..n_docs with numpy (same bits as the reference) and the device only looks it up, so
 * neither df nor idf crosses PCIe during a fit.                                                                              */
int pfz_idf_lookup(const int32_t *df, const int32_t *n_vocab_dev, int64_t cap, const double *table, int64_t n_table, double *idf, void *stream);

/* Stage C: emit the l2-normalised TF-IDF CSR for one list with a FIXED vocabulary (transform).
 *   lookup: rank_dense (may be NULL) else binary search in vocab_keys[n_vocab]; OOV n-grams dropped
 *   idf: float64[n_vocab] (computed by the host with numpy exactly as sklearn does, text.py:1679-1694)
 *   indptr int32[n_rows+1]; indices int32[cap]; data float64[cap], cap >= occ_ptr[n_rows]
 *   ws: >= pfz_scan_ws_bytes(n_rows+1) + 4*(n_rows+1) bytes                                           */
int pfz_tfidf_emit(const uint64_t *codes, const int32_t *tf, const int64_t *occ_ptr, const int32_t *row_cnt,
                   int32_t n_rows, const int32_t *rank_dense, const uint64_t *vocab_keys, int32_t n_vocab,
                   const double *idf, int32_t *indptr, int32_t *indices, double *data, void *ws, void *stream);

int64_t pfz_scan_ws_bytes(int64_t n);

/* ------------------------------------------------------------------------------------------------
 * K2  sparse cosine with fused per-row top-k.
 * Replaces: sparse_dot_topn.awesome_cossim_topn (call site polyfuzz/models/_utils.py:82) plus
 *           polyfuzz/models/_utils.py:84-87 (diagonal removal), :128-136 (_top_n_idx_sparse),
 *           :139-146 (_top_n_similarities_sparse, without the 3-dp rounding which stays in the
 *           DataFrame assembly).
 * Canonical contract: fp64, per (from-row, to-row) products added in ascending term order, each
 * product rounded before the add; candidate iff score > min_similarity (strict) and not the
 * diagonal; ranking key (score desc, to-index asc); empty slots idx=-1, score=0.
 * ---------------------------------------------------------------------------------------------- */

/* Inverted index of the to-matrix: postings grouped by (term, to-tile of `tile` rows).
 *   seg      int32[n_vocab*(n_tiles)+1]  prefix offsets, entry t*n_tiles+tau = start of (term t, tile tau)
 *   post_idx uint16[nnz] to-row LOCAL to its tile (row - tau*tile);  post_val float64[nnz]
 *   (posting order inside a (term, tile) segment is unspecified -- every to-row occurs at most once
 *    per term, so the per-pair addition order, ascending term, does not depend on it)
 *   ws: >= pfz_scan_ws_bytes(n_vocab*n_tiles+1) + 4*(n_vocab*n_tiles+1) bytes                         */
#define PFZ_INDEX_BANK_ORDER   1 /* arrange each segment so that 16 consecutive postings hit distinct 8-byte smem banks (fp64 accumulators) */
#define PFZ_INDEX_BANK_ORDER32 2 /* ... 32 consecutive postings hit distinct 4-byte banks (fp32 accumulators: DENSE32 / BLOCK)          */
int pfz_index_build(const int32_t *indptr, const int32_t *indices, const double *data, int32_t n_rows,
                    int32_t n_vocab, int32_t tile, int32_t n_tiles, int32_t flags,
                    int32_t *seg, uint16_t *post_idx, double *post_val, float *post_val32 /* may be NULL */,
                    float *term_maxw /* float[n_vocab], max weight per term rounded up; may be NULL */,
                    void *ws, void *stream);

/* top-k of (from CSR) x (to inverted index).
 *   k <= 32.  n_splits > 1 splits the to-tiles over blockIdx.y and writes partial lists
 *   [n_splits][n_from][k] (then call pfz_topk_merge).  self_match: exclude global to-index ==
 *   from_index_base + i.  Output indices are GLOBAL: to_index_base + local row.
 *   excl_val/excl_idx (may be NULL): per-row exclusive lower key -- only candidates ranking strictly
 *   AFTER (excl_val[i], excl_idx[i]) are considered (used to page through top_n > 32).
 *   row_counter: int32[n_splits] on device, zeroed by the callee (dynamic row scheduling).
 *   variant: PFZ_K2_LIST  -- touched-list selection, work ~ postings (sparse inputs, e.g. uniform text)
 *            PFZ_K2_DENSE -- threshold-crossing flags + dense accumulator clear (rows that touch a
 *                            sizeable fraction of every tile, e.g. company names); same results.
 *            PFZ_K2_DENSE32 -- like DENSE with an fp32 FILTER: fp32 weights (post_val32) and fp32 shared-memory
 *                            sums decide which to-rows could rank before the k-th key (margin 3e-5); each of
 *                            those is re-scored exactly from the two CSR rows (b_* = the to-matrix CSR the index
 *                            was built from), so indices and scores are bit-identical to the other variants.
 *                            Requires l2-normalised rows with positive weights (TF-IDF).  With term_maxw the
 *                            kernel also skips whole posting lists whose summed upper bound cannot lift a
 *                            to-row over the k-th key (MaxScore-style; exactness is kept by the re-scoring). */
#define PFZ_K2_LIST  1
#define PFZ_K2_DENSE 2
#define PFZ_K2_DENSE32 3
int pfz_spcos_topk(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from,
                   const int32_t *seg, const uint16_t *post_idx, const double *post_val,
                   const float *post_val32, const int32_t *b_indptr, const int32_t *b_indices, const double *b_data,
                   const float *term_maxw,
                   int32_t n_vocab, int32_t tile, int32_t n_tiles, int32_t n_to,
                   int32_t k, double min_similarity, int32_t self_match,
                   int64_t from_index_base, int64_t to_index_base, int32_t n_splits,
                   const double *excl_val, const int32_t *excl_idx,
                   int32_t *top_idx, double *top_val, int32_t *row_counter, int32_t variant, void *stream);

/* PFZ_K2_BLOCK -- from-row-block variant of K2 (csrc/pfz_spcos_block.cu): the from-rows are clustered by their heaviest
 * terms and scored block_rows (4, 8 or 16) at a time by one CTA, so one load of a posting chunk serves every row of the block
 * that contains the term; fixed-point sums in shared memory (red.shared.add.u32) filter, the to-rows whose sum passes a row's
 * gate are listed in the workspace and re-scored exactly from the two CSR rows by a second kernel (as PFZ_K2_DENSE32): indices
 * and scores are bit-identical to the other variants.  Same reference call site (polyfuzz/models/_utils.py:82).
 *   post_pk: uint2[nnz] in segment order of an index built with PFZ_INDEX_BANK_ORDER32: acc_bits 32: {tile-local row,
 *            round(weight * 2^26)} (pfz_index_pack_q26); acc_bits 16: {accumulator word byte offset | half-word selector << 16,
 *            max(1, round(weight * 2^15))} (pfz_index_pack_q15 with the same tile).
 *   tile: multiple of 128 in 128..4096; k <= 32; from-rows <= 128 terms each (*err_flag_dev is set to 1 otherwise); n_from < 2^22.
 *   acc_bits: 16 (two fixed-point accumulators per word, unit 2^-15: twice the tile in the same shared memory, filter margin
 *            4 m + 2 units for a from-row of m terms; tile must be a multiple of 256) or 32 (one per word, unit 2^-26, margin 1e-5).
 *   nnz_cap_from: capacity of a_indices / a_data (>= nnz).  ws: >= pfz_spcos_block_ws_bytes(...) bytes (clustering keys, block
 *            tables, and 192 candidate slots per (split, from-row)).
 *   Output as pfz_spcos_topk: [n_splits][n_from][k] partial lists (pfz_topk_merge when n_splits > 1).
 * pfz_spcos_block_gcnt_offset: byte offset in ws of int32 gcnt[n_splits][n_from], the candidates each (split, from-row) left
 *   for exact re-scoring in the last call (a diagnostic: how much the filter let through).                                 */
int64_t pfz_spcos_block_ws_bytes(int32_t n_from, int64_t nnz_cap_from, int32_t n_vocab, int32_t n_splits);
int64_t pfz_spcos_block_gcnt_offset(int32_t n_from, int64_t nnz_cap_from, int32_t n_vocab, int32_t n_splits);
int pfz_index_pack_q26(const uint16_t *post_idx, const double *post_val, const int32_t *nnz_dev, void *post_pk, void *stream);
int pfz_index_pack_q15(const uint16_t *post_idx, const double *post_val, const int32_t *nnz_dev, int32_t tile, void *post_pk, void *stream);
int pfz_spcos_topk_block(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from, int64_t nnz_cap_from,
                         const int32_t *seg, const void *post_pk, const int32_t *b_indptr, const int32_t *b_indices, const double *b_data,
                         int32_t n_vocab, int32_t tile, int32_t n_tiles, int32_t n_to, int32_t k, double min_similarity, int32_t self_match,
                         int64_t from_index_base, int64_t to_index_base, int32_t n_splits, int32_t block_rows, int32_t acc_bits,
                         int32_t *top_idx, double *top_val, int32_t *err_flag_dev, void *ws, void *stream);

/* PFZ_K2_HASH -- sparse-regime variant of K2 (csrc/pfz_spcos_hash.cu): one CTA per from-row accumulates the postings the row
 * visits in a shared-memory hash table keyed by the to-row (atom.shared.cas + red.shared.add.u32, fixed point 2^-26), scans
 * the table once and re-scores the sums above the row's threshold exactly; work ~ postings, independent of n_tiles.  For
 * inputs where a from-row touches a small fraction of the to-rows (uniform text).  Same reference call site
 * (polyfuzz/models/_utils.py:82), bit-identical results.
 *   index: built with tile = 65536 (the largest the 16-bit local rows allow) + pfz_index_pack_q26; from-rows <= 256 terms.
 *   table_slots: 1024 | 2048 | 8192 | 16384; a row whose postings exceed half the table is scored in several tile-range passes;
 *   *err_flag_dev: 2 = table overflow (a single tile held more postings than the table), 3 = row longer than 256 terms.
 *   excl_val/excl_idx: as pfz_spcos_topk (paging).  Output [n_splits][n_from][k].                                        */
int pfz_spcos_topk_hash(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from, const int32_t *seg,
                        const void *post_pk, const int32_t *b_indptr, const int32_t *b_indices, const double *b_data, int32_t tile,
                        int32_t n_tiles, int32_t n_to, int32_t k, double min_similarity, int32_t self_match, int64_t from_index_base,
                        int64_t to_index_base, int32_t n_splits, int32_t table_slots, const double *excl_val, const int32_t *excl_idx,
                        int32_t *top_idx, double *top_val, int32_t *row_counter, int32_t *err_flag_dev, void *stream);

/* merge n_lists sorted top-k lists per row ([n_lists][n_from][k_in]) into [n_from][k_out];
 * same key.  Used for tile splits and for the per-shard lists after the NCCL all-gather.            */
int pfz_topk_merge(const int32_t *idx, const double *val, int32_t n_lists, int32_t n_from, int32_t k_in,
                   int32_t k_out, int32_t *out_idx, double *out_val, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K3  all-pairs edit distance with a fused per-row arg-best.
 * Replaces: rapidfuzz process.extractOne / scorer loops as called at polyfuzz/models/_rapidfuzz.py:99-113
 *           and polyfuzz/models/_distance.py:89-102 (np.argmax = first maximum).
 * Symbols are bytes: sym_table (uint8[0x110000]) maps the code points of the from-strings to 1..255
 * and everything else to 0 (the host batches from-strings whose joint alphabet exceeds 255).
 * ---------------------------------------------------------------------------------------------- */

/* to-list layout: `order` = to-rows sorted by length (ascending); sorted position p lives in group p/32,
 * lane p%32; group g occupies ceil(maxlen_g/4) x 32 uint32 words starting at grp_word_off[g]
 * (4 symbols per word, lane-interleaved).  slen[p] receives the length of sorted string p.          */
int pfz_lev_pack(const uint32_t *to_blob, const int64_t *to_offsets, const int32_t *order, int32_t n_to,
                 const uint8_t *sym_table, const int64_t *grp_word_off, uint32_t *packed, int32_t *slen, void *stream);

/* scores the from-strings listed in from_ids (all of one word class: n_words = 0 -> length <= 32 (one
 * 32-bit word), 1/2/4/8/16 -> length <= 64*n_words) against every to-string.
 *   metric: PFZ_METRIC_*; for NORM_LEV / JARO / JARO_WINKLER / NORM_OSA a candidate needs score >= score_cutoff; for RATIO
 *           rapidfuzz's two steps: ns = 1 - indel/(|a|+|b|) >= score_cutoff/100 (fuzz.ratio) and score = ns*100 >= score_cutoff
 *           (extractOne), which differ whenever (ns*100)/100 != ns -- e.g. ns = 17/25 is rejected at score_cutoff 68.0
 *   exclude_self: skip to-row == from-row + self_shift
 *   part_*: [n_splits][n_from] partial bests (merge with pfz_lev_merge); ties -> lowest to-index;
 *           part_dist holds the distance, or for JARO / JARO_WINKLER the number of matching characters
 *   matrix (may be NULL): int32 [n_from][matrix_ld] full distance matrix (Levenshtein, Indel, or OSA for OSA /
 *           NORM_OSA); must be NULL for JARO / JARO_WINKLER
 * OSA / NORM_OSA: optimal string alignment (restricted Damerau-Levenshtein) on code points: insertions, deletions,
 * substitutions and swaps of two adjacent characters, no substring edited twice (osa("CA", "ABC") = 3, where unrestricted
 * Damerau-Levenshtein gives 2); DESIGN.md 4.9 gives the recurrence.
 *   counter: int32[n_splits], zeroed by the callee
 * JARO / JARO_WINKLER: jellyfish's definition on code points, from-string first (the reference calls
 * scorer(from_string, to_string), polyfuzz/models/_distance.py:98); DESIGN.md 4.5 gives the recurrence.  */
int pfz_lev_argbest(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids,
                    int32_t n_ids, int32_t n_words, const uint8_t *sym_table, const uint32_t *packed,
                    const int64_t *grp_word_off, const int32_t *slen, const int32_t *sorig, int32_t n_to,
                    int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits,
                    int32_t *part_idx, double *part_score, int32_t *part_dist, int32_t *matrix, int64_t matrix_ld,
                    int32_t *counter, void *stream);
int pfz_lev_merge(const int32_t *part_idx, const double *part_score, const int32_t *part_dist, int32_t n_splits,
                  int32_t n_from, int32_t *best_idx, double *best_score, int32_t *best_dist, void *stream);

/* top-k sibling of pfz_lev_argbest: the k best to-strings per from-string (1 <= k <= 32), same candidates (the cutoff tests
 * above, to-row == from-row + self_shift excluded when exclude_self) and key (score desc, to-index asc).
 * Replaces: rapidfuzz process.extract(query, to_list, scorer, limit=k), and the sort of the scorer values of
 *           polyfuzz/models/_distance.py:98-99 where the reference takes np.argmax.
 *   metric: NORM_LEV, RATIO, JARO, JARO_WINKLER or NORM_OSA; there is no distance output and no matrix.
 *   part_idx / part_score: [n_splits][n_from][k] sorted lists, empty slots (-1, 0.0); merge them with pfz_topk_merge.   */
int pfz_lev_topk(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids,
                 int32_t n_ids, int32_t n_words, const uint8_t *sym_table, const uint32_t *packed,
                 const int64_t *grp_word_off, const int32_t *slen, const int32_t *sorig, int32_t n_to,
                 int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits,
                 int32_t k, int32_t *part_idx, double *part_score, int32_t *counter, void *stream);

/* Unrestricted Damerau-Levenshtein (Lowrance-Wagner with unit costs, on code points): the fewest insertions, deletions,
 * substitutions and swaps of two adjacent characters, where a swapped pair may be edited again (dl("CA", "ABC") = 2).
 * Same parameters, layout, candidates, key and outputs as pfz_lev_argbest / pfz_lev_topk, plus
 *   gate (may be NULL): float64[n_from], per from-row a proven lower bound of its k-th best score (k = 1 for the arg-best) over
 *         the whole to-list; pairs whose score upper bound is below it are skipped.  The k-th best OSA score of the row (the
 *         pfz_lev_* pass with OSA / NORM_OSA and the same cutoff, exclusion and k, merged over the splits) is such a bound, and a
 *         row with fewer than k OSA candidates takes score_cutoff (NORM_DL) or -inf (DL).  NULL: no gate.
 *   metric: DL (raw distance, best = smallest, no cutoff; arg-best only) or NORM_DL (1 - dl/max(|a|,|b|), score >= score_cutoff).
 *   matrix (arg-best only, may be NULL): DL distances of every pair; requires gate == NULL.
 * DESIGN.md 4.10 gives the bounds and the kernel. */
int pfz_dl_argbest(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids,
                   int32_t n_ids, int32_t n_words, const uint8_t *sym_table, const uint32_t *packed,
                   const int64_t *grp_word_off, const int32_t *slen, const int32_t *sorig, int32_t n_to,
                   int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits,
                   int32_t *part_idx, double *part_score, int32_t *part_dist, int32_t *matrix, int64_t matrix_ld,
                   const double *gate, int32_t *counter, void *stream);
int pfz_dl_topk(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids,
                int32_t n_ids, int32_t n_words, const uint8_t *sym_table, const uint32_t *packed,
                const int64_t *grp_word_off, const int32_t *slen, const int32_t *sorig, int32_t n_to,
                int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits,
                int32_t k, int32_t *part_idx, double *part_score, const double *gate, int32_t *counter, void *stream);

/* K3b  rapidfuzz's token / partial / weighted scorers with a fused per-row arg-best (csrc/pfz_fuzz.cu).
 * Replaces: process.extractOne(query, to_list, scorer=fuzz.WRatio | partial_ratio | token_*_ratio | ..., score_cutoff) at
 *           polyfuzz/models/_rapidfuzz.py:48,106-108 and the scorer loop of polyfuzz/models/_distance.py:98.
 * scorer: 0 ratio, 1 QRatio, 2 partial_ratio, 3 token_sort_ratio, 4 token_set_ratio, 5 token_ratio, 6 partial_token_sort_ratio,
 *         7 partial_token_set_ratio, 8 partial_token_ratio, 9 WRatio (rapidfuzz 3.x definitions, processor=None; scores 0..100).
 * ptrs: 38 device pointers -- for the from-side then the to-side: {blob uint32, offsets int64} of s, S(s) = sorted tokens
 *       joined, U(s) = distinct sorted tokens joined; tok_ptr int32[n+1]; tok_ids int32 (distinct token ids per string,
 *       ascending; ids number the tokens of both lists in sorted order); sig uint64[n] (Bloom signature of the ids);
 *       n_tok_all int32[n] (tokens incl. duplicates) -- then from_ids int32[n_ids] (from-rows of this word class: n_words = 1, 2, 4,
 *       8, 16 for from-strings whose longest variant has up to 64, 128, 256, 512, 1024 code points; to-strings of any
 *       length), sym_table uint8[0x110000], for each variant {packed, grp_word_off, slen}
 *       (pfz_lev_pack layouts of b, S(b), U(b) in ONE length order), sorig int32[n_to], tok_blob uint32, tok_off int64[n_tok+1],
 *       part_idx int32[n_splits][n_from], part_score float64[n_splits][n_from], counter int32[n_splits], reserved (NULL).
 * Best = first to-string (lowest index) with the maximal score >= score_cutoff; merge the splits with pfz_lev_merge.
 * The cutoff reaches the scorer as in rapidfuzz: ratio (also inside token_sort_ratio, token_ratio, QRatio, WRatio) keeps
 * ns = 1 - indel/(|a|+|b|) only if ns >= score_cutoff/100, and partial_ratio (also inside the partial_token_* scorers and
 * WRatio) keeps its best window's ns only if ns >= score_cutoff/100 and ns*100 >= score_cutoff; the token-set parts test
 * 100 - 100*dist/lensum >= score_cutoff once.  So a pair is rejected at a cutoff equal to its own score whenever
 * (ns*100)/100 > ns in doubles, and WRatio's internal cutoffs (max(c, end_ratio)/0.9, /0.95) apply the same rule.          */
int pfz_fuzz_argbest(const void *const *ptrs, int32_t n_ptrs, int32_t n_from, int32_t n_ids, int32_t n_words, int32_t n_to,
                     int32_t scorer, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits, void *stream);

/* K3b's token tables, built on the device (csrc/pfz_tok.cu).  Replaces the host derivation of s.split(), sorted(), the token
 * dictionary and the signatures.  Tokens are Python str.split()'s: maximal runs of code points c with not chr(c).isspace().
 *
 * pfz_tok_side: one string list (blob int32 code points, offsets int64[n+1], n_chars = offsets[n] code points) ->
 *   n_all int32[n]                 tokens per string (duplicates counted)
 *   vocab_blob int32, vocab_off int64[n_occ+1]   the list's distinct tokens in Python string order (code points compared in
 *                                  turn, a proper prefix first); entries of vocab_off past the vocabulary hold its total length
 *   tok_ptr int32[n+1], tok_ids int32   each string's distinct token ids (ranks in vocab), ascending
 *   s_off int64[n+1], s_blob int32  S(s) = all tokens in id order joined by single spaces
 *   u_off int64[n+1], u_blob int32  U(s) = the distinct tokens joined the same way
 *   counts_host int64[6] (host memory): n_occ (tokens), vocabulary size, vocabulary code points, S and U code points, tok_ids
 *   entries.  The blob and tok_ids buffers need max(n_chars, 1) entries, vocab_off n_chars + 1.  Synchronises the stream.
 * pfz_tok_union: two sorted vocabularies -> their sorted union (u_blob, u_off int64[n_a+n_b+1], entries past the union hold its
 *   total length; *n_u on the device) and each token's union rank (map_a int32[n_a], map_b int32[n_b]; a monotone map).
 * pfz_tok_remap: ids_out[j] = map[ids_in[j]] (map NULL: the identity) for the ids of the n strings of tok_ptr, and per string
 *   the Bloom signature sig = OR over its ids of 1 << (((id * 0x9E3779B1) >> 13) & 63), the product taken in 64 bits.     */
int pfz_tok_side(const int32_t *blob, const int64_t *offsets, int32_t n, int64_t n_chars, int32_t *n_all, int32_t *vocab_blob,
                 int64_t *vocab_off, int32_t *tok_ptr, int32_t *tok_ids, int64_t *s_off, int32_t *s_blob, int64_t *u_off,
                 int32_t *u_blob, int64_t *counts_host, void *stream);
int pfz_tok_union(const int32_t *a_blob, const int64_t *a_off, int32_t n_a, const int32_t *b_blob, const int64_t *b_off, int32_t n_b,
                  int32_t *map_a, int32_t *map_b, int32_t *u_blob, int64_t *u_off, int32_t *n_u, void *stream);
int pfz_tok_remap(const int32_t *tok_ptr, const int32_t *ids_in, int32_t n, const int32_t *map, int32_t *ids_out, uint64_t *sig,
                  void *stream);

/* top-k sibling of pfz_fuzz_argbest: the k best to-strings per from-string (1 <= k <= 32) under the same candidates and key.
 * Replaces: rapidfuzz process.extract(query, to_list, scorer=..., score_cutoff=..., limit=k), and the sort of the scorer values
 *           of polyfuzz/models/_distance.py:98-99 where the reference takes np.argmax.
 * ptrs: as pfz_fuzz_argbest, except part_idx int32 / part_score float64 are [n_splits][n_from][k] sorted lists with empty slots
 *       (-1, 0.0); merge them with pfz_topk_merge.                                                                               */
int pfz_fuzz_topk(const void *const *ptrs, int32_t n_ptrs, int32_t n_from, int32_t n_ids, int32_t n_words, int32_t n_to,
                  int32_t scorer, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits, int32_t k,
                  void *stream);

/* ------------------------------------------------------------------------------------------------
 * K4  dense cosine top-k for pre-computed embeddings (bf16 wgmma GEMM fed by TMA, top-k fused into the
 * epilogue).  Replaces the dense branch polyfuzz/models/_utils.py:94-102 (sklearn cosine_similarity +
 * argsort) reached from polyfuzz/models/_embeddings.py:127-131.
 * ---------------------------------------------------------------------------------------------- */

/* rows (float32 or float64, row pitch ld elements) -> bf16 [n_rows][d_pad], optionally l2-normalised
 * (sk:metrics/pairwise.py:1744-1750 normalises both sides); columns d..d_pad are zero.  d_pad % 8 == 0.  */
int pfz_rows_to_bf16(const void *x, int32_t is_f64, int64_t ld, int32_t n_rows, int32_t d, int32_t d_pad,
                     int32_t normalize, void *out_bf16, void *stream);

/* top-k of X * Y^T.  x_bf16 [n_from][d], y_bf16 [n_to][d] row-major bf16, d % 8 == 0, 16-byte aligned.
 *   candidate iff score > min_similarity (strict) and not the diagonal (self_match); key (score desc,
 *   index asc) on the fp32 accumulator values; k <= 32; partial lists [n_splits][n_from][k] (idx int32
 *   global, score as float64) -> pfz_topk_merge when n_splits > 1.                                     */
int pfz_dense_cos_topk(const void *x_bf16, const void *y_bf16, int32_t n_from, int32_t n_to, int32_t d, int32_t k,
                       double min_similarity, int32_t self_match, int64_t from_index_base, int64_t to_index_base,
                       int32_t n_splits, int32_t *top_idx, double *top_val, void *stream);

/* K4 exact mode: the canonical fp64 cosine top-k (DESIGN.md 2 and 4.6), bit for bit, from an fp16 tensor-core filter pass,
 * fp64 re-scoring of its candidates with a per-row certificate, and a brute-force pass for the rows not certified.
 * Canonical dot(a, b): lane l = dimension mod 32 sums a[32t+l]*b[32t+l] over ascending t (products rounded, then added, no
 * FMA, from +0), then p[l] += p[l xor o] for o = 16, 8, 4, 2, 1.  Normalisation x~ = x / sqrt(dot(x, x)) (a row with
 * dot(x, x) == 0 stays as it is).  score = dot(x~, y~); candidate iff score > min_similarity (strict) and not the diagonal
 * (self_match); key (score desc, index asc); empty slots (-1, 0.0).
 *
 * prep: rows (float32 or float64, pitch ld) -> out_f64 = x~ and out_f16 = fp16(x~), both [n_rows][d_pad] zero-padded,
 *   d_pad % 8 == 0; norm16[i] >= ||fp16(x~_i)|| and err16[i] >= ||x~_i - fp16(x~_i)|| (float64[n_rows], upward-rounded);
 *   maxima (may be NULL): float64[2] = {max norm16, max err16}, zeroed by the callee.                                     */
int pfz_rows_prep_exact(const void *x, int32_t is_f64, int64_t ld, int32_t n_rows, int32_t d, int32_t d_pad,
                        double *out_f64, void *out_f16, double *norm16, double *err16, double *maxima, void *stream);

/* filter pass: as pfz_dense_cos_topk on fp16 operands (wgmma .f16), except that the candidates are the fp32 scores > t_f,
 * t_f = the largest float <= min_similarity - M_max(d), M_max(d) the a-priori bound on |fp32 filter score - canonical
 * score| of DESIGN.md 4.6.  Every to-row whose canonical score exceeds min_similarity scores above t_f here.           */
int pfz_dense_cos_topk_f16(const void *x_f16, const void *y_f16, int32_t n_from, int32_t n_to, int32_t d, int32_t k,
                           double min_similarity, int32_t self_match, int64_t from_index_base, int64_t to_index_base,
                           int32_t n_splits, int32_t *top_idx, double *top_val, void *stream);

/* re-score + certify: cand_idx / cand_val [n_from][k_cand] = the merged filter lists (global indices) of
 * pfz_dense_cos_topk_f16 with the same min_similarity; x_* from pfz_rows_prep_exact of the from-rows, y_maxima its maxima
 * of the to-rows.  k <= k_cand <= 32.  Writes the canonical top-k of every row to top_idx / top_val [n_from][k]; rows whose
 * result cannot be certified exact are listed in fb_rows (int32[n_from]) with their number in *fb_count (zeroed by the
 * callee); pfz_dense_exact_fallback overwrites them.                                                                     */
int pfz_dense_exact_rescore(const double *x_f64, const double *y_f64, int32_t n_from, int32_t n_to, int32_t d_pad, int32_t k,
                            int32_t k_cand, const int32_t *cand_idx, const double *cand_val, const double *x_norm16,
                            const double *x_err16, const double *y_maxima, double min_similarity, int32_t self_match,
                            int64_t from_index_base, int64_t to_index_base, int32_t *top_idx, double *top_val,
                            int32_t *fb_rows, int32_t *fb_count, void *stream);

/* fallback: canonical top-k over every to-row for the *fb_count rows in fb_rows (the count is read on the device).
 * ws: >= pfz_dense_exact_fallback_ws_bytes(n_from, n_to, k) bytes.                                                       */
int64_t pfz_dense_exact_fallback_ws_bytes(int32_t n_from, int32_t n_to, int32_t k);
int pfz_dense_exact_fallback(const double *x_f64, const double *y_f64, int32_t n_from, int32_t n_to, int32_t d_pad, int32_t k,
                             double min_similarity, int32_t self_match, int64_t from_index_base, int64_t to_index_base,
                             const int32_t *fb_rows, const int32_t *fb_count, int32_t *top_idx, double *top_val, void *ws,
                             void *stream);

/* K4 top_n > 32, both precisions (DESIGN.md 4.7): a bound per row from the UNMERGED lists of a top-16 call with n_splits >= 2k/16
 * (pfz_dense_cos_topk, or pfz_dense_cos_topk_f16 in the exact mode), a threshold pass that appends every to-row scoring above the
 * row's bound, and a per-row select.  Rows are processed in chunks by the caller, so the buffers below stay bounded.
 *
 * bound: row_thr (float[n_from]) from lists [n_lists][n_from][k_list] (global indices, -1 = empty).  exact == 0: the k-th best
 *   score of the row's union; exact != 0: with f_k the k-th best filter score and M_i the row's margin (x_norm16 / x_err16 of
 *   pfz_rows_prep_exact for these rows, y_maxima of the to-rows), tau = f_k - M_i and row_thr = tau - M_i (both rounded down)
 *   when tau > min_similarity.  -inf when no bound exists (fewer than k entries, or tau <= min_similarity).               */
int pfz_dense_topn_bound(const int32_t *list_idx, const double *list_val, int32_t n_lists, int32_t n_from, int32_t k_list,
                         int32_t k, int32_t exact, const double *x_norm16, const double *x_err16, const double *y_maxima,
                         int32_t d_pad, double min_similarity, float *row_thr, void *stream);

/* threshold pass: K4 (bf16, or fp16 with the filter threshold t_f of pfz_dense_cos_topk_f16) appending every (global to-index,
 * fp32 score as float64) with score >= row_thr[i] and score > min_similarity (t_f) to cand_idx / cand_val [n_from][cap] in
 * no particular order.  cand_count (int32[n_from], zeroed by the callee) counts every such to-row, also past cap: a row with
 * cand_count > cap must be re-run with a larger cap.  The diagonal is NOT excluded here (pfz_dense_topn_select does that).
 * The bf16 scores are the same fp32 values pfz_dense_cos_topk ranks.                                                     */
int pfz_dense_cos_cand(const void *x_bf16, const void *y_bf16, int32_t n_from, int32_t n_to, int32_t d, double min_similarity,
                       const float *row_thr, int64_t to_index_base, int32_t n_splits, int32_t cap, int32_t *cand_idx,
                       double *cand_val, int32_t *cand_count, void *stream);
int pfz_dense_cos_cand_f16(const void *x_f16, const void *y_f16, int32_t n_from, int32_t n_to, int32_t d, double min_similarity,
                           const float *row_thr, int64_t to_index_base, int32_t n_splits, int32_t cap, int32_t *cand_idx,
                           double *cand_val, int32_t *cand_count, void *stream);

/* exact mode: replaces each candidate's filter score by its canonical fp64 score.  Row r's from-row is
 * x_f64[row_map ? row_map[r] : r]; y_f64 holds the to-rows of global index to_index_base + local row.                    */
int pfz_dense_topn_exact_rescore(const double *x_f64, const double *y_f64, int32_t n_rows, int32_t d_pad, const int32_t *row_map,
                                 int64_t to_index_base, int32_t cap, const int32_t *cand_idx, double *cand_val,
                                 const int32_t *cand_count, void *stream);

/* select: the top k of each row's min(cand_count, cap) candidates by (score desc, index asc), keeping score > min_similarity
 * and, with self_match, dropping to-index from_index_base + output row; written to output row (row_map ? row_map[r] : r) of
 * top_idx / top_val [..][k], empty slots (-1, 0.0).  Any k and any cap.                                                   */
int pfz_dense_topn_select(const int32_t *cand_idx, const double *cand_val, const int32_t *cand_count, int32_t n_rows, int32_t cap,
                          int32_t k, double min_similarity, int32_t self_match, int64_t from_index_base, const int32_t *row_map,
                          int32_t *top_idx, double *top_val, void *stream);

/* ------------------------------------------------------------------------------------------------
 * K5  frame tail: top-k arrays -> the columns of the result frame (csrc/pfz_assemble.cu).
 * Replaces: polyfuzz/models/_utils.py:104-125 (the per-rank `[to_list[idx] ...]` gathers, the 3-decimal rounding of :102/:143
 *           and the `Similarity < 0.001 -> 0, To -> None` rule of :119-123).  ASCII string lists only (bytes == code points).
 * Column-major entries e = r*n + i (r = rank 0..k-1, i = from-row):
 *   sims    float64[k*n]     np.round(score, 3), 0 where the slot is empty or rounds below 0.001
 *   lens_pos int32[k*n + 1]  on return the EXCLUSIVE prefix of the matched strings' byte lengths (last entry = total bytes)
 *   bitmap  uint32[k * ceil(n/32)]   Arrow validity bits (bit i of column r)
 *   ws: >= pfz_scan_ws_bytes(k*n + 1) bytes.
 * then, with the total known to the caller: offsets int64[k*(n+1)] (relative to each column's start: Arrow large_string, what
 * pandas' Arrow-backed str dtype holds) and the UTF-8 bytes.   */
int pfz_frame_tail_count(const int32_t *top_idx, const double *top_val, int32_t n, int32_t k, const int64_t *to_offsets, double *sims,
                         int32_t *lens_pos, uint32_t *bitmap, void *ws, void *stream);
int pfz_frame_tail_copy(const int32_t *top_idx, int32_t n, int32_t k, const int32_t *to_blob, const int64_t *to_offsets, const int32_t *pos,
                        int64_t *offsets, uint8_t *data, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PFZ_H */
