// pfz_wordvec.cu -- K6: word-vector lookup and mean pooling on the device.
// Replaces GensimEmbeddings._embed (polyfuzz/models/_gensim.py:118-140): every string is split on U+0020, each token is looked
// up in the KeyedVectors table (a zero vector when it is missing) and the token vectors are averaged with np.mean(axis=0).
//
//   table build  one thread per key, open addressing with linear probing, atomicCAS inserts into int32 table[cap] (-1 = empty);
//                the keys are distinct, so what a lookup returns does not depend on the order of the inserts
//   lookup       count kernel (spaces + 1 per string), in-place CUB scan -> tok_off, then one warp per string: a ballot over
//                32 code points at a time marks the token ends, and each lane that ends a token hashes it and probes the
//                table, comparing the full code-point sequence of every key whose slot it meets
//   pool         one warp per string, lanes over columns: numpy's sequential axis-0 sum in the dtype of the token list, and
//                one division by the token count (DESIGN.md 4.11 states the rule)
//   FastText     pfz_ft_pool: the pool with every token in float32, a token missing from the vocabulary replaced by gensim's
//                subword vector, hashed and gathered in place by the string's warp (DESIGN.md 4.14)
#include <cub/device/device_scan.cuh>
#include "pfz_common.cuh"

namespace pfz {

constexpr int WV_THREADS = 256;
constexpr int WV_COLS = 8;          // columns per lane in one pass of the pool kernel: 256 columns per pass

// FNV-1a over the code points, then murmur3's finaliser so that the slot bits depend on every code point
__device__ __forceinline__ uint32_t wv_hash(const uint32_t *__restrict__ cp, int64_t len) {
    uint32_t h = 2166136261u;
    for (int64_t i = 0; i < len; ++i) { h ^= cp[i]; h *= 16777619u; }
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}

__global__ void __launch_bounds__(WV_THREADS) wv_insert_kernel(const uint32_t *__restrict__ key_blob, const int64_t *__restrict__ key_off,
                                                              int32_t n_keys, int32_t *table, uint32_t mask) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_keys; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = key_off[i];
        uint32_t s = wv_hash(key_blob + b, key_off[i + 1] - b) & mask;
        while (atomicCAS(&table[s], -1, (int)i) != -1) s = (s + 1) & mask;      // cap > n_keys: an empty slot exists
    }
}

// position of the key equal to tok[0..len) in the key list, or -1
__device__ __forceinline__ int32_t wv_find(const uint32_t *__restrict__ tok, int64_t len, const uint32_t *__restrict__ key_blob,
                                           const int64_t *__restrict__ key_off, const int32_t *__restrict__ table, uint32_t mask) {
    uint32_t s = wv_hash(tok, len) & mask;
    for (;;) {
        const int32_t p = table[s];
        if (p < 0) return -1;
        const int64_t b = key_off[p];
        if (key_off[p + 1] - b == len) {
            int64_t i = 0;
            while (i < len && key_blob[b + i] == tok[i]) ++i;
            if (i == len) return p;
        }
        s = (s + 1) & mask;
    }
}

// ntok[r] = (number of U+0020 in string r) + 1, ntok[n] = 0 (the scan turns ntok into the token offsets)
__global__ void __launch_bounds__(WV_THREADS) wv_count_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ off, int32_t n,
                                                             int64_t *__restrict__ ntok) {
    const int lane = lane_id();
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    if (blockIdx.x == 0 && threadIdx.x == 0) ntok[n] = 0;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
        const int64_t e = off[r + 1];
        unsigned long long c = 0;
        for (int64_t i = off[r] + lane; i < e; i += 32) c += blob[i] == 32u;
#pragma unroll
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
        if (lane == 0) ntok[r] = (int64_t)c + 1;
    }
}

// tok_row[tok_off[r] + j] = key_row of token j of string r, or -1.  The end of the string acts as one more space, so a string
// of s spaces gives s + 1 tokens, empty ones included.
__global__ void __launch_bounds__(WV_THREADS) wv_lookup_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ off, int32_t n,
                                                              const int64_t *__restrict__ tok_off, const uint32_t *__restrict__ key_blob,
                                                              const int64_t *__restrict__ key_off, const int32_t *__restrict__ key_row,
                                                              const int32_t *__restrict__ table, uint32_t mask, int32_t *__restrict__ tok_row) {
    const int lane = lane_id();
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
        const int64_t e = off[r + 1];
        int64_t start = off[r], t = tok_off[r];          // the current token's first code point and its slot (warp-uniform)
        for (int64_t c0 = off[r]; c0 <= e; c0 += 32) {
            const int64_t i = c0 + lane;
            const bool brk = i < e ? blob[i] == 32u : i == e;
            const unsigned m = __ballot_sync(FULL, brk);
            if (brk) {
                const unsigned below = m & ((1u << lane) - 1u);
                const int64_t s0 = below ? c0 + (32 - __clz(below)) : start;
                const int32_t p = wv_find(blob + s0, i - s0, key_blob, key_off, table, mask);
                tok_row[t + __popc(below)] = p < 0 ? -1 : key_row[p];
            }
            if (m) { start = c0 + (32 - __clz(m)); t += __popc(m); }
        }
    }
}

// One string's mean in the accumulator type A (float: every token found in a float32 table; double otherwise).  Per column
// s_0 = +0.0, s_j = s_{j-1} + v_j rounded to A (so a column of -0.0 values sums to +0.0, as numpy's does), then s_n / n: numpy divides the float32 sum by the intp count in double and
// rounds the quotient to float32, which is the correctly rounded float32 quotient (53 >= 2*24 + 2) and what is done here.
template <typename T, typename A>
__device__ __forceinline__ void wv_pool_row(const T *__restrict__ V, int32_t d, const int32_t *__restrict__ rows, int64_t nt,
                                            double *__restrict__ out) {
    const int lane = lane_id();
    for (int c0 = 0; c0 < d; c0 += 32 * WV_COLS) {
        A s[WV_COLS];
#pragma unroll
        for (int u = 0; u < WV_COLS; ++u) s[u] = (A)0;                   // numpy's add.reduce starts from +0.0
        for (int64_t j0 = 0; j0 < nt; j0 += 32) {
            const int32_t mine = j0 + lane < nt ? rows[j0 + lane] : -1;
            const int cnt = (int)min((int64_t)32, nt - j0);
            for (int q = 0; q < cnt; ++q) {
                const int32_t row = __shfl_sync(FULL, mine, q);
                const T *vr = V + (int64_t)row * d;
#pragma unroll
                for (int u = 0; u < WV_COLS; ++u) {
                    const int c = c0 + u * 32 + lane;
                    if (c < d) {
                        const A v = row >= 0 ? (A)vr[c] : (A)0;          // a missing token is +0.0 (np.zeros)
                        if constexpr (sizeof(A) == 4) s[u] = __fadd_rn(s[u], v);
                        else s[u] = __dadd_rn(s[u], v);
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < WV_COLS; ++u) {
            const int c = c0 + u * 32 + lane;
            if (c < d) {
                const double q = __ddiv_rn((double)s[u], (double)nt);
                out[c] = sizeof(A) == 4 ? (double)__double2float_rn(q) : q;
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(WV_THREADS) wv_pool_kernel(const T *__restrict__ V, int32_t d, const int64_t *__restrict__ tok_off,
                                                            const int32_t *__restrict__ tok_row, int32_t n, double *__restrict__ out,
                                                            int64_t ld) {
    const int lane = lane_id();
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
        const int64_t t0 = tok_off[r], nt = tok_off[r + 1] - t0;
        const int32_t *rows = tok_row + t0;
        if constexpr (sizeof(T) == 4) {
            // one missing token makes the list a float64 array (np.zeros(d) among float32 rows): the whole row pools in fp64
            bool miss = false;
            for (int64_t j = lane; j < nt; j += 32) miss |= rows[j] < 0;
            if (!__any_sync(FULL, miss)) { wv_pool_row<T, float>(V, d, rows, nt, out + r * ld); continue; }
        }
        wv_pool_row<T, double>(V, d, rows, nt, out + r * ld);
    }
}

// ---- FastText subword vectors (DESIGN.md 4.14) ------------------------------------------------------------------------------------
// gensim's FastTextKeyedVectors.get_vector(word) for a word outside the vocabulary: the n-grams of "<" + word + ">" (characters,
// i ascending, n = 1..max_n ascending, kept when n >= min_n and not the lone "<" or ">"), each hashed by 32-bit FNV-1a over its
// UTF-8 bytes sign-extended, bucket = h % bucket; the vector is fl32(sum) / count in float32, +0.0 without n-grams.
constexpr int FT_COLS = 10;         // columns per lane in one pass of the FastText pool kernel: 320 columns, d = 300 in one pass

// character k of "<" + tok[0..len) + ">"
__device__ __forceinline__ uint32_t ft_char(const uint32_t *__restrict__ tok, int64_t len, int64_t k) {
    return k == 0 ? 60u : k == len + 1 ? 62u : tok[k - 1];
}

__device__ __forceinline__ uint32_t ft_fnv_byte(uint32_t h, uint32_t b) {
    return (h ^ (b >= 0x80u ? 0xFFFFFF00u | b : b)) * 16777619u;      // the byte as int8, sign-extended to 32 bits
}

// FNV-1a over the UTF-8 encoding of characters [i, i + n) of "<" + tok + ">" (no surrogates: the host refuses them)
__device__ __forceinline__ uint32_t ft_hash(const uint32_t *__restrict__ tok, int64_t len, int64_t i, int64_t n) {
    uint32_t h = 2166136261u;
    for (int64_t k = i; k < i + n; ++k) {
        const uint32_t c = ft_char(tok, len, k);
        if (c < 0x80u) {
            h = ft_fnv_byte(h, c);
        } else if (c < 0x800u) {
            h = ft_fnv_byte(h, 0xC0u | (c >> 6));
            h = ft_fnv_byte(h, 0x80u | (c & 0x3Fu));
        } else if (c < 0x10000u) {
            h = ft_fnv_byte(h, 0xE0u | (c >> 12));
            h = ft_fnv_byte(h, 0x80u | ((c >> 6) & 0x3Fu));
            h = ft_fnv_byte(h, 0x80u | (c & 0x3Fu));
        } else {
            h = ft_fnv_byte(h, 0xF0u | (c >> 18));
            h = ft_fnv_byte(h, 0x80u | ((c >> 12) & 0x3Fu));
            h = ft_fnv_byte(h, 0x80u | ((c >> 6) & 0x3Fu));
            h = ft_fnv_byte(h, 0x80u | (c & 0x3Fu));
        }
    }
    return h;
}

// The subword vector of tok[0..len) for columns c0 + u*32 + lane, added to s (the string's float32 sum).  The n-grams are the
// cells (i, n) of a grid of width W = min(max_n, len + 2) - nlo + 1, walked 32 cells at a time in list order; each lane hashes
// one cell, the kept cells' bucket ids are broadcast in order and every lane adds its columns of those rows in that order.
__device__ __forceinline__ void ft_add_subword(const uint32_t *__restrict__ tok, int64_t len, const float *__restrict__ NG, int32_t d,
                                               uint32_t bucket, int32_t min_n, int32_t max_n, int c0, float (&s)[FT_COLS]) {
    const int lane = lane_id();
    const int64_t lc = len + 2;                                        // characters of "<" + tok + ">"
    const int64_t nlo = min_n > 1 ? min_n : 1;
    const int64_t w = min((int64_t)max_n, lc) - nlo + 1;                 // < 2^31: max_n is an int32
    float acc[FT_COLS];
#pragma unroll
    for (int u = 0; u < FT_COLS; ++u) acc[u] = 0.f;                  // gensim's word_vec = np.zeros(d, float32)
    int64_t cnt = 0;
    if (w > 0) {
        const uint32_t W = (uint32_t)w;
        // the chunk starts at cell (i0, j0); j0 < W, so j0 + 32 fits 32 bits and the divisions stay 32-bit
        int64_t i0 = 0;
        for (uint32_t j0 = 0; i0 < lc; i0 += (j0 + 32u) / W, j0 = (j0 + 32u) % W) {
            const uint32_t j = j0 + (uint32_t)lane;
            const int64_t i = i0 + j / W, n = nlo + j % W;
            const bool keep = i + n <= lc && !(n == 1 && (i == 0 || i == lc - 1));
            const uint32_t bid = keep ? ft_hash(tok, len, i, n) % bucket : 0u;
            unsigned m = __ballot_sync(FULL, keep);
            cnt += __popc(m);
            while (m) {
                const int q = __ffs(m) - 1;
                m &= m - 1;
                const float *nr = NG + (int64_t)__shfl_sync(FULL, bid, q) * d;
#pragma unroll
                for (int u = 0; u < FT_COLS; ++u) {
                    const int c = c0 + u * 32 + lane;
                    if (c < d) acc[u] = __fadd_rn(acc[u], nr[c]);
                }
            }
        }
    }
    // word_vec / len(ngram_hashes): a float32 array over a Python int, divided in float32; no n-grams leaves the zero vector
    const float fc = __ll2float_rn(cnt);
#pragma unroll
    for (int u = 0; u < FT_COLS; ++u) s[u] = __fadd_rn(s[u], cnt ? __fdiv_rn(acc[u], fc) : 0.f);
}

// One warp per string, lanes over columns: every token resolves to a float32 vector (its row of V, or its subword vector when
// tok_row is -1), so every string pools on numpy's float32 path.  The tokens are found again by the lookup kernel's ballot walk
// over the U+0020 breaks, in the order of tok_row.
__global__ void __launch_bounds__(WV_THREADS) ft_pool_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ off, int32_t n,
                                                            const int64_t *__restrict__ tok_off, const int32_t *__restrict__ tok_row,
                                                            const float *__restrict__ V, const float *__restrict__ NG, int32_t d,
                                                            uint32_t bucket, int32_t min_n, int32_t max_n, double *__restrict__ out,
                                                            int64_t ld) {
    const int lane = lane_id();
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += warps) {
        const int64_t e = off[r + 1], nt = tok_off[r + 1] - tok_off[r];
        for (int c0 = 0; c0 < d; c0 += 32 * FT_COLS) {
            float s[FT_COLS];
#pragma unroll
            for (int u = 0; u < FT_COLS; ++u) s[u] = 0.f;              // numpy's add.reduce starts from +0.0
            int64_t start = off[r], t = tok_off[r];
            for (int64_t b0 = off[r]; b0 <= e; b0 += 32) {
                const int64_t i = b0 + lane;
                const bool brk = i < e ? blob[i] == 32u : i == e;
                unsigned m = __ballot_sync(FULL, brk);
                while (m) {                                            // the tokens ending in this chunk, in order
                    const int64_t end = b0 + (__ffs(m) - 1);
                    m &= m - 1;
                    const int32_t row = tok_row[t++];
                    if (row >= 0) {
                        const float *vr = V + (int64_t)row * d;
#pragma unroll
                        for (int u = 0; u < FT_COLS; ++u) {
                            const int c = c0 + u * 32 + lane;
                            if (c < d) s[u] = __fadd_rn(s[u], vr[c]);
                        }
                    } else {
                        ft_add_subword(blob + start, end - start, NG, d, bucket, min_n, max_n, c0, s);
                    }
                    start = end + 1;
                }
            }
#pragma unroll
            for (int u = 0; u < FT_COLS; ++u) {
                const int c = c0 + u * 32 + lane;
                if (c < d) out[r * ld + c] = (double)__double2float_rn(__ddiv_rn((double)s[u], (double)nt));
            }
        }
    }
}

static int wv_grid(int64_t warps_needed) {
    int64_t g = (warps_needed + WV_THREADS / 32 - 1) / (WV_THREADS / 32);
    if (g > SM_COUNT * 16) g = SM_COUNT * 16;
    return g < 1 ? 1 : (int)g;
}

static bool pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_wv_table_build(const uint32_t *key_blob, const int64_t *key_off, int32_t n_keys, int32_t *table, int64_t cap, void *stream) {
    PFZ_REQUIRE(n_keys >= 0 && pow2(cap) && cap > n_keys && cap <= (1ll << 31),
                "pfz_wv_table_build: cap (%lld) must be a power of two above n_keys (%d), at most 2^31", (long long)cap, n_keys);
    cudaStream_t st = as_stream(stream);
    PFZ_CUDA_OK(cudaMemsetAsync(table, 0xFF, sizeof(int32_t) * (size_t)cap, st));
    if (n_keys == 0) return 0;
    int grid = (int)((n_keys + WV_THREADS - 1) / WV_THREADS); if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    wv_insert_kernel<<<grid, WV_THREADS, 0, st>>>(key_blob, key_off, n_keys, table, (uint32_t)(cap - 1));
    PFZ_LAUNCH_OK();
    return 0;
}

int64_t pfz_wv_lookup_ws_bytes(int32_t n) {
    size_t bytes = 0;
    if (n < 0 || cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int64_t *)nullptr, (int64_t)n + 1) != cudaSuccess) return -1;
    return (int64_t)bytes;
}

int pfz_wv_lookup(const uint32_t *blob, const int64_t *offsets, int32_t n, const uint32_t *key_blob, const int64_t *key_off,
                  const int32_t *key_row, const int32_t *table, int64_t cap, int64_t *tok_off, int32_t *tok_row, void *ws, int64_t ws_bytes,
                  void *stream) {
    PFZ_REQUIRE(n >= 0 && pow2(cap) && cap <= (1ll << 31), "pfz_wv_lookup: n (%d) or cap (%lld) out of range", n, (long long)cap);
    if (n == 0) return 0;
    cudaStream_t st = as_stream(stream);
    const int grid = wv_grid(n);
    wv_count_kernel<<<grid, WV_THREADS, 0, st>>>(blob, offsets, n, tok_off);
    PFZ_LAUNCH_OK();
    size_t bytes = (size_t)ws_bytes;
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(ws, bytes, tok_off, (int64_t)n + 1, st));
    wv_lookup_kernel<<<grid, WV_THREADS, 0, st>>>(blob, offsets, n, tok_off, key_blob, key_off, key_row, table, (uint32_t)(cap - 1), tok_row);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_wv_pool(const void *vectors, int32_t is_f64, int32_t d, const int64_t *tok_off, const int32_t *tok_row, int32_t n, double *out,
                int64_t ld, void *stream) {
    PFZ_REQUIRE(d >= 2 && ld >= d && n >= 0, "pfz_wv_pool: d (%d) must be >= 2 and ld (%lld) >= d", d, (long long)ld);
    if (n == 0) return 0;
    cudaStream_t st = as_stream(stream);
    const int grid = wv_grid(n);
    if (is_f64) wv_pool_kernel<double><<<grid, WV_THREADS, 0, st>>>((const double *)vectors, d, tok_off, tok_row, n, out, ld);
    else wv_pool_kernel<float><<<grid, WV_THREADS, 0, st>>>((const float *)vectors, d, tok_off, tok_row, n, out, ld);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_ft_pool(const uint32_t *blob, const int64_t *offsets, int32_t n, const int64_t *tok_off, const int32_t *tok_row, const float *vectors,
                const float *vectors_ngrams, int32_t d, int64_t bucket, int32_t min_n, int32_t max_n, double *out, int64_t ld, void *stream) {
    PFZ_REQUIRE(d >= 2 && ld >= d && n >= 0, "pfz_ft_pool: d (%d) must be >= 2 and ld (%lld) >= d", d, (long long)ld);
    PFZ_REQUIRE(bucket >= 1 && bucket < (1ll << 32) && min_n >= 0 && max_n >= 0,
                "pfz_ft_pool: bucket (%lld) must be in [1, 2^32) and min_n (%d), max_n (%d) >= 0", (long long)bucket, min_n, max_n);
    if (n == 0) return 0;
    cudaStream_t st = as_stream(stream);
    ft_pool_kernel<<<wv_grid(n), WV_THREADS, 0, st>>>(blob, offsets, n, tok_off, tok_row, vectors, vectors_ngrams, d, (uint32_t)bucket,
                                                       min_n, max_n, out, ld);
    PFZ_LAUNCH_OK();
    return 0;
}
}
