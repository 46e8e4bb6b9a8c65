// pfz_tfidf.cu -- K1: character n-gram TF-IDF vectoriser on sm_90a.
//
// Replaces the reference's per-string Python loops (polyfuzz/models/_tfidf.py:120-146) and the
// scikit-learn vocabulary / tf-idf / l2 arithmetic they feed (sk:feature_extraction/text.py:1257-1320,
// 1651-1739; sk:utils/sparsefuncs_fast.pyx:578-605).  See include/pfz.h for the staging.
//
// Stage A  ngram_rows   one warp per string: clean -> symbols -> n-gram codes -> bitonic sort -> RLE
// Stage B  df / vocab   direct-addressed document frequency + scan compaction (small code space), or
//                       gather + global bitonic sort + run-length (large code space)
// Stage C  emit         vocabulary lookup, tf*idf, ordered sum of squares, sqrt, divide -> CSR
#include "pfz_common.cuh"

namespace pfz {

constexpr uint64_t KEY_PAD = ~0ull;
constexpr uint32_t SYM_UNKNOWN = 0xffffffffu;
constexpr uint32_t SYM_SPACE = 1u;           // clean alphabet: ' '=1, '0'..'9'=2..11, 'a'..'z'=12..37
constexpr int MAX_N = 8;

// ---- cleaning ------------------------------------------------------------------------------------
// polyfuzz/models/_tfidf.py:142-146: s.lower(); delete [^A-Za-z0-9 ]+; collapse \s+ -> ' '; strip().
// After the first substitution only ASCII alnum and U+0020 survive; the only non-ASCII code points
// whose str.lower() contains a surviving character are U+0130 (-> 'i' + U+0307) and U+212A (-> 'k')
// (tests/golden/clean_survivors.json, exhaustive over all code points).
__device__ __forceinline__ uint32_t clean_symbol(uint32_t c) {
    if (c >= 'A' && c <= 'Z') c += 32;
    if (c >= 'a' && c <= 'z') return 12u + (c - 'a');
    if (c >= '0' && c <= '9') return 2u + (c - '0');
    if (c == ' ') return SYM_SPACE;
    if (c == 0x0130u) return 12u + ('i' - 'a');
    if (c == 0x212Au) return 12u + ('k' - 'a');
    return 0u;  // deleted
}

// One warp turns one string into sorted distinct n-gram codes + counts.
//   sym  : smem uint32[cap_sym]   (symbols, compacted in place)
//   keys : smem uint64[cap_keys]  (cap_keys power of two)
template <bool CLEAN>
__device__ void process_row(const uint32_t *__restrict__ blob, int64_t beg, int L, int lo, int hi, bool remove_space,
                            const uint32_t *__restrict__ sym_table, uint64_t base, uint32_t *sym, uint64_t *keys,
                            int cap_keys, uint64_t *__restrict__ out_codes, int32_t *__restrict__ out_tf,
                            int32_t *out_cnt) {
    const int lane = lane_id();
    const unsigned lt = (1u << lane) - 1u;
    int Lc = 0;
    if (CLEAN) {
        // pass 1: map + drop deleted characters
        int kept = 0;
        for (int p0 = 0; p0 < L; p0 += 32) {
            int p = p0 + lane;
            uint32_t s = (p < L) ? clean_symbol(blob[beg + p]) : 0u;
            unsigned m = __ballot_sync(FULL, s != 0u);
            if (s != 0u) sym[kept + __popc(m & lt)] = s;
            kept += __popc(m);
        }
        __syncwarp();
        // pass 2: collapse space runs, strip both ends (in place: destination index <= source index,
        // processed in ascending 32-chunks with the chunk read before any write of that chunk)
        int last_ns = -1;
        for (int p0 = 0; p0 < kept; p0 += 32) {
            int p = p0 + lane;
            bool ns = (p < kept) && sym[p] != SYM_SPACE;
            unsigned m = __ballot_sync(FULL, ns);
            if (m) last_ns = p0 + 31 - __clz(m);
        }
        int outn = 0;
        for (int p0 = 0; p0 < kept; p0 += 32) {
            int p = p0 + lane;
            uint32_t s = (p < kept) ? sym[p] : 0u;
            uint32_t prev = (p > 0 && p < kept) ? sym[p - 1] : SYM_SPACE;   // original neighbour
            __syncwarp();
            bool keep = (p < kept) && (s != SYM_SPACE || (prev != SYM_SPACE && p < last_ns));
            unsigned m = __ballot_sync(FULL, keep);
            // NOTE: prev must be the ORIGINAL previous symbol; writes land at index <= p0+lane and
            // only for indices < p0 + popc, while sym[p0-1] was read by lane 0 before this chunk's writes.
            if (keep) sym[outn + __popc(m & lt)] = s;
            outn += __popc(m);
            __syncwarp();
        }
        Lc = outn;
    } else {
        for (int p0 = 0; p0 < L; p0 += 32) {
            int p = p0 + lane;
            if (p < L) {
                uint32_t c = blob[beg + p];
                sym[p] = (c < 0x110000u) ? sym_table[c] : SYM_UNKNOWN;
            }
        }
        Lc = L;
        __syncwarp();
    }

    // n-gram codes
    uint64_t pw[MAX_N];
    {
        uint64_t q = 1;
#pragma unroll
        for (int d = MAX_N - 1; d >= 0; --d) {
            if (d < hi) { pw[d] = q; q *= base; } else pw[d] = 0;   // pw[d] = base^(hi-1-d)
        }
    }
    // In raw mode the space symbol is whatever the fitted alphabet assigned to U+0020.
    const uint32_t space_sym = CLEAN ? SYM_SPACE : sym_table[0x20];
    int cnt = 0;
    for (int n = lo; n <= hi; ++n) {
        const int nst = Lc - n + 1;
        for (int i0 = 0; i0 < nst; i0 += 32) {
            int i = i0 + lane;
            bool ok = i < nst;
            uint64_t code = 0;
            if (ok) {
#pragma unroll
                for (int d = 0; d < MAX_N; ++d) {
                    if (d < n) {
                        uint32_t s = sym[i + d];
                        if (s == SYM_UNKNOWN || (remove_space && s == space_sym)) ok = false;
                        code += (uint64_t)s * pw[d];
                    }
                }
            }
            unsigned m = __ballot_sync(FULL, ok);
            if (ok) keys[cnt + __popc(m & lt)] = code;
            cnt += __popc(m);
        }
    }
    // pad to a power of two and sort (bitonic, ascending)
    int P = 1;
    while (P < cnt) P <<= 1;
    if (P > cap_keys) P = cap_keys;
    for (int q = cnt + lane; q < P; q += 32) keys[q] = KEY_PAD;
    __syncwarp();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = lane; t < (P >> 1); t += 32) {
                int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));   // index with bit j clear
                int ix = i | j;
                uint64_t a = keys[i], b = keys[ix];
                bool up = (i & k) == 0;
                if ((a > b) == up) { keys[i] = b; keys[ix] = a; }
            }
            __syncwarp();
        }
    }
    // run-length encode
    int nd = 0;
    for (int q0 = 0; q0 < cnt; q0 += 32) {
        int q = q0 + lane;
        bool head = false;
        uint64_t c = 0;
        if (q < cnt) { c = keys[q]; head = (q == 0) || keys[q - 1] != c; }
        unsigned m = __ballot_sync(FULL, head);
        if (head) {
            int len = 1;
            while (q + len < cnt && keys[q + len] == c) ++len;
            int pos = nd + __popc(m & lt);
            out_codes[pos] = c;
            out_tf[pos] = len;
        }
        nd += __popc(m);
    }
    if (lane == 0) *out_cnt = nd;
}

template <bool CLEAN>
__global__ void __launch_bounds__(256) ngram_rows_warp_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ offsets,
                                                              int n_rows, int lo, int hi, int remove_space,
                                                              const uint32_t *__restrict__ sym_table, uint64_t base,
                                                              const int64_t *__restrict__ occ_ptr, uint64_t *__restrict__ codes,
                                                              int32_t *__restrict__ tf, int32_t *__restrict__ row_cnt) {
    constexpr int WPB = 8;
    constexpr int CAP = PFZ_WARP_ROW_SLOTS;
    __shared__ uint64_t s_keys[WPB][CAP];
    __shared__ uint32_t s_sym[WPB][CAP + MAX_N];
    const int w = threadIdx.x >> 5;
    for (int r = blockIdx.x * WPB + w; r < n_rows; r += gridDim.x * WPB) {
        const int64_t o0 = occ_ptr[r];
        const int64_t slots = occ_ptr[r + 1] - o0;
        if (slots > CAP) continue;                      // handled by the long-row kernel
        const int64_t beg = offsets[r];
        const int L = (int)(offsets[r + 1] - beg);
        if (slots == 0) { if (lane_id() == 0) row_cnt[r] = 0; continue; }
        process_row<CLEAN>(blob, beg, L, lo, hi, remove_space != 0, sym_table, base, s_sym[w], s_keys[w], CAP,
                           codes + o0, tf + o0, row_cnt + r);
        __syncwarp();
    }
}

// long rows: one warp per block with a large dynamic smem arena
template <bool CLEAN>
__global__ void __launch_bounds__(32) ngram_rows_long_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ offsets,
                                                             const int32_t *__restrict__ long_rows, int n_long, int lo, int hi,
                                                             int remove_space, const uint32_t *__restrict__ sym_table, uint64_t base,
                                                             const int64_t *__restrict__ occ_ptr, uint64_t *__restrict__ codes,
                                                             int32_t *__restrict__ tf, int32_t *__restrict__ row_cnt) {
    extern __shared__ __align__(16) unsigned char dyn[];
    uint64_t *s_keys = reinterpret_cast<uint64_t *>(dyn);
    uint32_t *s_sym = reinterpret_cast<uint32_t *>(dyn + (size_t)PFZ_MAX_ROW_SLOTS * 8);
    for (int q = blockIdx.x; q < n_long; q += gridDim.x) {
        const int r = long_rows[q];
        const int64_t o0 = occ_ptr[r];
        const int64_t beg = offsets[r];
        const int L = (int)(offsets[r + 1] - beg);
        process_row<CLEAN>(blob, beg, L, lo, hi, remove_space != 0, sym_table, base, s_sym, s_keys, PFZ_MAX_ROW_SLOTS,
                           codes + o0, tf + o0, row_cnt + r);
        __syncwarp();
    }
}

__global__ void alphabet_mark_kernel(const uint32_t *__restrict__ blob, int64_t n, uint8_t *__restrict__ present) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t c = blob[i];
        if (c < 0x110000u) present[c] = 1;
    }
}

// ---- Stage B -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) df_dense_kernel(const uint64_t *__restrict__ codes, const int64_t *__restrict__ occ_ptr,
                                                       const int32_t *__restrict__ row_cnt, int n_rows, int32_t *__restrict__ df_dense) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const int64_t o0 = occ_ptr[r];
        const int c = row_cnt[r];
        for (int q = lane; q < c; q += 32) atomicAdd(&df_dense[codes[o0 + q]], 1);
    }
}

__global__ void flag_positive_kernel(const int32_t *__restrict__ df_dense, int64_t n, int32_t *__restrict__ flag) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = df_dense[i] > 0;
}

__global__ void vocab_compact_kernel(const int32_t *__restrict__ df_dense, int64_t n, int32_t *__restrict__ rank,
                                     uint64_t *__restrict__ vocab_keys, int32_t *__restrict__ df, int32_t *__restrict__ n_vocab) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t d = df_dense[i];
        const int32_t pos = rank[i];
        if (i == n - 1) *n_vocab = pos + (d > 0);
        if (d > 0) { vocab_keys[pos] = (uint64_t)i; df[pos] = d; }
        else rank[i] = -1;
    }
}

__global__ void __launch_bounds__(256) gather_codes_kernel(const uint64_t *__restrict__ codes, const int64_t *__restrict__ occ_ptr,
                                                           const int32_t *__restrict__ row_cnt, int n_rows, uint64_t *__restrict__ keys,
                                                           unsigned long long *__restrict__ cursor) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const int64_t o0 = occ_ptr[r];
        const int c = row_cnt[r];
        if (c == 0) continue;
        unsigned long long dst = 0;
        if (lane == 0) dst = atomicAdd(cursor, (unsigned long long)c);
        dst = __shfl_sync(FULL, dst, 0);
        for (int q = lane; q < c; q += 32) keys[dst + q] = codes[o0 + q];
    }
}

// idf[v] = table[df[v]] for v < *n_vocab (the table holds sklearn's idf for every possible df, computed by numpy on the host)
__global__ void idf_lookup_kernel(const int32_t *__restrict__ df, const int32_t *__restrict__ n_vocab, int64_t cap, const double *__restrict__ table,
                                  int64_t n_table, double *__restrict__ idf) {
    const int64_t nv = min((int64_t)*n_vocab, cap);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t d = df[i];
        idf[i] = table[d < n_table ? d : n_table - 1];
    }
}

// global bitonic sort of uint64 keys (n power of two)
constexpr int BS_TILE = 4096;      // keys per block for the shared-memory stages (32 KB)
constexpr int BS_THREADS = 512;

__global__ void __launch_bounds__(BS_THREADS) bitonic_local_kernel(uint64_t *__restrict__ keys, int64_t n, int64_t k_first, int64_t k_last,
                                                                   int64_t j_first) {
    // performs, for k = k_first .. k_last (doubling): j = (k == k_first ? j_first : k/2) .. 1 inside one tile
    __shared__ uint64_t s[BS_TILE];
    const int64_t base = (int64_t)blockIdx.x * BS_TILE;
    for (int t = threadIdx.x; t < BS_TILE; t += BS_THREADS) s[t] = (base + t < n) ? keys[base + t] : KEY_PAD;
    __syncthreads();
    for (int64_t k = k_first; k <= k_last; k <<= 1) {
        int64_t j0 = (k == k_first) ? j_first : (k >> 1);
        for (int64_t j = j0; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < BS_TILE / 2; t += BS_THREADS) {
                int i = ((t & ~((int)j - 1)) << 1) | (t & ((int)j - 1));
                int ix = i | (int)j;
                uint64_t a = s[i], b = s[ix];
                bool up = ((base + i) & k) == 0;
                if ((a > b) == up) { s[i] = b; s[ix] = a; }
            }
            __syncthreads();
        }
    }
    for (int t = threadIdx.x; t < BS_TILE; t += BS_THREADS) if (base + t < n) keys[base + t] = s[t];
}

__global__ void bitonic_global_kernel(uint64_t *__restrict__ keys, int64_t n, int64_t k, int64_t j) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (n >> 1); t += (int64_t)gridDim.x * blockDim.x) {
        int64_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        int64_t ix = i | j;
        uint64_t a = keys[i], b = keys[ix];
        bool up = (i & k) == 0;
        if ((a > b) == up) { keys[i] = b; keys[ix] = a; }
    }
}

__global__ void sorted_heads_kernel(const uint64_t *__restrict__ keys, int64_t cap, const int64_t *__restrict__ n_keys, int32_t *__restrict__ flag) {
    const int64_t n = *n_keys;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = (i < n) && (i == 0 || keys[i] != keys[i - 1]);
}

__global__ void sorted_compact_kernel(const uint64_t *__restrict__ keys, int64_t cap, const int64_t *__restrict__ n_keys,
                                      const int32_t *__restrict__ pos, uint64_t *__restrict__ vocab_keys, int32_t *__restrict__ head_at,
                                      int32_t *__restrict__ n_vocab) {
    const int64_t n = *n_keys;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
        bool head = (i < n) && (i == 0 || keys[i] != keys[i - 1]);
        if (head) { vocab_keys[pos[i]] = keys[i]; head_at[pos[i]] = (int32_t)i; }
        if (i == cap - 1) { int32_t v = pos[i] + (head ? 1 : 0); *n_vocab = v; }
    }
}

__global__ void head_diff_kernel(const int32_t *__restrict__ head_at, const int32_t *__restrict__ n_vocab, const int64_t *__restrict__ n_keys,
                                 int32_t *__restrict__ df, int64_t cap) {
    const int32_t V = *n_vocab;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V && i < cap; i += (int64_t)gridDim.x * blockDim.x) {
        int32_t nxt = (i + 1 < V) ? head_at[i + 1] : (int32_t)(*n_keys);
        df[i] = nxt - head_at[i];
    }
}

// ---- Stage C -------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t lookup_col(uint64_t code, const int32_t *__restrict__ rank_dense, const uint64_t *__restrict__ vocab_keys,
                                              int32_t n_vocab) {
    if (rank_dense) return rank_dense[code];
    int32_t lo = 0, hi = n_vocab;
    while (lo < hi) {
        int32_t mid = (lo + hi) >> 1;
        if (vocab_keys[mid] < code) lo = mid + 1; else hi = mid;
    }
    return (lo < n_vocab && vocab_keys[lo] == code) ? lo : -1;
}

__global__ void __launch_bounds__(256) emit_count_kernel(const uint64_t *__restrict__ codes, const int64_t *__restrict__ occ_ptr,
                                                         const int32_t *__restrict__ row_cnt, int n_rows, const int32_t *__restrict__ rank_dense,
                                                         const uint64_t *__restrict__ vocab_keys, int32_t n_vocab, int32_t *__restrict__ row_nnz) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r <= n_rows; r += nw) {
        if (r == n_rows) { if (lane == 0) row_nnz[r] = 0; continue; }
        const int64_t o0 = occ_ptr[r];
        const int c = row_cnt[r];
        int tot = 0;
        for (int q0 = 0; q0 < c; q0 += 32) {
            int q = q0 + lane;
            bool ok = (q < c) && lookup_col(codes[o0 + q], rank_dense, vocab_keys, n_vocab) >= 0;
            tot += __popc(__ballot_sync(FULL, ok));
        }
        if (lane == 0) row_nnz[r] = tot;
    }
}

// tf*idf, ordered sum of squares (column order, product rounded before the add), sqrt, divide:
// sk:feature_extraction/text.py:1734 (X.data *= idf[X.indices]) and sk:utils/sparsefuncs_fast.pyx:578-605.
__global__ void __launch_bounds__(256) emit_write_kernel(const uint64_t *__restrict__ codes, const int32_t *__restrict__ tf,
                                                         const int64_t *__restrict__ occ_ptr, const int32_t *__restrict__ row_cnt, int n_rows,
                                                         const int32_t *__restrict__ rank_dense, const uint64_t *__restrict__ vocab_keys,
                                                         int32_t n_vocab, const double *__restrict__ idf, const int32_t *__restrict__ indptr,
                                                         int32_t *__restrict__ indices, double *__restrict__ data) {
    const int lane = lane_id();
    const unsigned lt = (1u << lane) - 1u;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const int64_t o0 = occ_ptr[r];
        const int c = row_cnt[r];
        const int32_t w0 = indptr[r];
        double ss = 0.0;
        for (int q0 = 0; q0 < c; q0 += 32) {
            int q = q0 + lane;
            int32_t col = (q < c) ? lookup_col(codes[o0 + q], rank_dense, vocab_keys, n_vocab) : -1;
            double x2 = 0.0;
            if (col >= 0) { double x = __dmul_rn((double)tf[o0 + q], idf[col]); x2 = __dmul_rn(x, x); }
            unsigned m = __ballot_sync(FULL, col >= 0);
            while (m) {                              // ascending lane == ascending column
                int l = __ffs(m) - 1; m &= m - 1;
                ss = __dadd_rn(ss, shfl_d(x2, l));
            }
        }
        const double norm = __dsqrt_rn(ss);
        int wrote = 0;
        for (int q0 = 0; q0 < c; q0 += 32) {
            int q = q0 + lane;
            int32_t col = (q < c) ? lookup_col(codes[o0 + q], rank_dense, vocab_keys, n_vocab) : -1;
            unsigned m = __ballot_sync(FULL, col >= 0);
            if (col >= 0) {
                double x = __dmul_rn((double)tf[o0 + q], idf[col]);
                int p = w0 + wrote + __popc(m & lt);
                indices[p] = col;
                data[p] = (norm != 0.0) ? __ddiv_rn(x, norm) : x;
            }
            wrote += __popc(m);
        }
    }
}

static int grid_for(int64_t work_items, int threads, int cap = SM_COUNT * 16) {
    int64_t g = (work_items + threads - 1) / threads;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_alphabet_mark(const uint32_t *blob, int64_t n_chars, uint8_t *present, void *stream) {
    if (n_chars <= 0) return 0;
    alphabet_mark_kernel<<<grid_for(n_chars, 256), 256, 0, as_stream(stream)>>>(blob, n_chars, present);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_ngram_rows(const uint32_t *blob, const int64_t *offsets, int32_t n_rows, int32_t lo, int32_t hi, int32_t flags,
                   const uint32_t *sym_table, uint32_t base, const int64_t *occ_ptr, const int32_t *long_rows, int32_t n_long,
                   uint64_t *codes, int32_t *tf, int32_t *row_cnt, void *stream) {
    PFZ_REQUIRE(lo >= 1 && hi >= lo && hi <= MAX_N, "pfz_ngram_rows: n-gram range (%d,%d) unsupported (1 <= lo <= hi <= %d)", lo, hi, MAX_N);
    const bool clean = flags & PFZ_FLAG_CLEAN;
    PFZ_REQUIRE(clean || sym_table, "pfz_ngram_rows: raw mode needs sym_table");
    {   // code must fit 64 bits
        long double cs = 1; for (int i = 0; i < hi; ++i) cs *= (long double)base;
        PFZ_REQUIRE(cs < 18446744073709551615.0L, "pfz_ngram_rows: alphabet %u ^ n %d exceeds 64-bit n-gram codes", base, hi);
    }
    if (n_rows <= 0) return 0;
    const int rs = (flags & PFZ_FLAG_REMOVE_SPACE) ? 1 : 0;
    cudaStream_t st = as_stream(stream);
    int grid = grid_for((int64_t)n_rows * 32, 256, SM_COUNT * 8);
    if (clean) ngram_rows_warp_kernel<true><<<grid, 256, 0, st>>>(blob, offsets, n_rows, lo, hi, rs, sym_table, base, occ_ptr, codes, tf, row_cnt);
    else       ngram_rows_warp_kernel<false><<<grid, 256, 0, st>>>(blob, offsets, n_rows, lo, hi, rs, sym_table, base, occ_ptr, codes, tf, row_cnt);
    PFZ_LAUNCH_OK();
    if (n_long > 0) {
        PFZ_REQUIRE(long_rows, "pfz_ngram_rows: n_long > 0 but long_rows is NULL");
        const size_t smem = (size_t)PFZ_MAX_ROW_SLOTS * 8 + ((size_t)PFZ_MAX_ROW_SLOTS + MAX_N + 8) * 4;
        if (clean) {
            PFZ_CUDA_OK(cudaFuncSetAttribute(ngram_rows_long_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ngram_rows_long_kernel<true><<<n_long < 592 ? n_long : 592, 32, smem, st>>>(blob, offsets, long_rows, n_long, lo, hi, rs, sym_table, base, occ_ptr, codes, tf, row_cnt);
        } else {
            PFZ_CUDA_OK(cudaFuncSetAttribute(ngram_rows_long_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ngram_rows_long_kernel<false><<<n_long < 592 ? n_long : 592, 32, smem, st>>>(blob, offsets, long_rows, n_long, lo, hi, rs, sym_table, base, occ_ptr, codes, tf, row_cnt);
        }
        PFZ_LAUNCH_OK();
    }
    return 0;
}

int pfz_df_dense(const uint64_t *codes, const int64_t *occ_ptr, const int32_t *row_cnt, int32_t n_rows, int32_t *df_dense, void *stream) {
    if (n_rows <= 0) return 0;
    df_dense_kernel<<<grid_for((int64_t)n_rows * 32, 256), 256, 0, as_stream(stream)>>>(codes, occ_ptr, row_cnt, n_rows, df_dense);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_vocab_compact_dense(const int32_t *df_dense, int64_t code_space, uint64_t *vocab_keys, int32_t *df, int32_t *rank_dense,
                            int32_t *n_vocab_dev, void *ws, void *stream) {
    PFZ_REQUIRE(code_space > 0 && code_space < (1ll << 31), "pfz_vocab_compact_dense: bad code space %lld", (long long)code_space);
    cudaStream_t st = as_stream(stream);
    flag_positive_kernel<<<grid_for(code_space, 256), 256, 0, st>>>(df_dense, code_space, rank_dense);
    PFZ_LAUNCH_OK();
    if (scan_exclusive_i32(rank_dense, rank_dense, code_space, ws, st)) return 1;
    vocab_compact_kernel<<<grid_for(code_space, 256), 256, 0, st>>>(df_dense, code_space, rank_dense, vocab_keys, df, n_vocab_dev);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_gather_codes(const uint64_t *codes, const int64_t *occ_ptr, const int32_t *row_cnt, int32_t n_rows, uint64_t *keys,
                     int64_t *cursor_dev, void *stream) {
    if (n_rows <= 0) return 0;
    gather_codes_kernel<<<grid_for((int64_t)n_rows * 32, 256), 256, 0, as_stream(stream)>>>(codes, occ_ptr, row_cnt, n_rows, keys,
                                                                                             reinterpret_cast<unsigned long long *>(cursor_dev));
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_idf_lookup(const int32_t *df, const int32_t *n_vocab_dev, int64_t cap, const double *table, int64_t n_table, double *idf, void *stream) {
    if (cap <= 0) return 0;
    PFZ_REQUIRE(n_table >= 1, "pfz_idf_lookup: empty table");
    idf_lookup_kernel<<<grid_for(cap, 256), 256, 0, as_stream(stream)>>>(df, n_vocab_dev, cap, table, n_table, idf);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_sort_u64(uint64_t *keys, int64_t n, void *stream) {
    PFZ_REQUIRE(n > 0 && (n & (n - 1)) == 0, "pfz_sort_u64: n=%lld must be a power of two", (long long)n);
    cudaStream_t st = as_stream(stream);
    const int64_t nblk = (n + BS_TILE - 1) / BS_TILE;
    const int64_t kloc = n < BS_TILE ? n : BS_TILE;
    bitonic_local_kernel<<<(unsigned)nblk, BS_THREADS, 0, st>>>(keys, n, 2, kloc, 1);
    PFZ_LAUNCH_OK();
    for (int64_t k = (int64_t)BS_TILE * 2; k <= n; k <<= 1) {
        int64_t j = k >> 1;
        for (; j >= BS_TILE; j >>= 1) {
            bitonic_global_kernel<<<grid_for(n >> 1, 256, SM_COUNT * 32), 256, 0, st>>>(keys, n, k, j);
            PFZ_LAUNCH_OK();
        }
        bitonic_local_kernel<<<(unsigned)nblk, BS_THREADS, 0, st>>>(keys, n, k, k, j);
        PFZ_LAUNCH_OK();
    }
    return 0;
}

int pfz_vocab_from_sorted(const uint64_t *sorted_keys, int64_t cap, const int64_t *n_keys_dev, uint64_t *vocab_keys, int32_t *df,
                          int32_t *n_vocab_dev, void *ws, void *stream) {
    PFZ_REQUIRE(cap > 0 && cap < (1ll << 31), "pfz_vocab_from_sorted: bad capacity %lld", (long long)cap);
    cudaStream_t st = as_stream(stream);
    // ws layout: pos int32[cap] | head_at int32[cap] | scan ws
    int32_t *pos = reinterpret_cast<int32_t *>(ws);
    int32_t *head_at = pos + cap;
    void *sws = reinterpret_cast<char *>(ws) + (((size_t)cap * 8 + 255) / 256) * 256;
    sorted_heads_kernel<<<grid_for(cap, 256), 256, 0, st>>>(sorted_keys, cap, n_keys_dev, pos);
    PFZ_LAUNCH_OK();
    if (scan_exclusive_i32(pos, pos, cap, sws, st)) return 1;
    sorted_compact_kernel<<<grid_for(cap, 256), 256, 0, st>>>(sorted_keys, cap, n_keys_dev, pos, vocab_keys, head_at, n_vocab_dev);
    PFZ_LAUNCH_OK();
    head_diff_kernel<<<grid_for(cap, 256), 256, 0, st>>>(head_at, n_vocab_dev, n_keys_dev, df, cap);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_tfidf_emit(const uint64_t *codes, const int32_t *tf, const int64_t *occ_ptr, const int32_t *row_cnt, int32_t n_rows,
                   const int32_t *rank_dense, const uint64_t *vocab_keys, int32_t n_vocab, const double *idf, int32_t *indptr,
                   int32_t *indices, double *data, void *ws, void *stream) {
    PFZ_REQUIRE(n_rows >= 0, "pfz_tfidf_emit: n_rows < 0");
    cudaStream_t st = as_stream(stream);
    emit_count_kernel<<<grid_for((int64_t)(n_rows + 1) * 32, 256), 256, 0, st>>>(codes, occ_ptr, row_cnt, n_rows, rank_dense, vocab_keys, n_vocab, indptr);
    PFZ_LAUNCH_OK();
    if (scan_exclusive_i32(indptr, indptr, (int64_t)n_rows + 1, ws, st)) return 1;
    if (n_rows > 0) {
        emit_write_kernel<<<grid_for((int64_t)n_rows * 32, 256), 256, 0, st>>>(codes, tf, occ_ptr, row_cnt, n_rows, rank_dense, vocab_keys, n_vocab,
                                                                                  idf, indptr, indices, data);
        PFZ_LAUNCH_OK();
    }
    return 0;
}
}
