// pfz_tok.cu -- K3b's token tables on the device: Python str.split() tokens, a sorted vocabulary per list, the per-string
// S(s) / U(s) strings, distinct token ids and Bloom signatures (include/pfz.h, pfz_tok_*).
//
// A list is tokenised on its own (pfz_tok_side): every token occurrence is sorted by its code points (CUB merge sort with a
// comparator that reads the blob, so tokens of any length sort exactly), equal neighbours share a rank, and the ranks number
// the list's own vocabulary.  Two lists are joined afterwards (pfz_tok_union) by binary searches of each vocabulary in the other
// vocabulary: the rank of a to-token is its rank in its own vocabulary plus the number of from-only tokens that sort before
// it, a monotone map, so a kept to-side is renumbered for each new from-list without being tokenised again (pfz_tok_remap).
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "pfz_common.cuh"

namespace pfz {
namespace {

constexpr int TPB = 256;

static unsigned grid_of(int64_t n) { return (unsigned)((n + TPB - 1) / TPB > 0 ? (n + TPB - 1) / TPB : 1); }

// chr(c).isspace(): the 29 code points Python's str.split() breaks on
__device__ __forceinline__ bool py_space(int32_t c) {
    if (c <= 0x20) return c == 0x20 || (c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x1F);
    if (c < 0x85) return false;
    return c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) || c == 0x2028 || c == 0x2029 || c == 0x202F ||
           c == 0x205F || c == 0x3000;
}

// Python string order: code points compared in turn, a proper prefix first
__device__ __forceinline__ int cp_cmp(const int32_t *a, int la, const int32_t *b, int lb) {
    const int m = la < lb ? la : lb;
    for (int i = 0; i < m; ++i) {
        const int32_t x = a[i], y = b[i];
        if (x != y) return x < y ? -1 : 1;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

// a token occurrence and its first three code points (+1, 21 bits each; 0 pads a shorter token), which decide most comparisons
struct TokKey {
    uint64_t pre;
    int32_t occ;
};

__device__ __forceinline__ uint64_t prefix_key(const int32_t *t, int len) {
    uint64_t k = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) k = (k << 21) | (i < len ? (uint64_t)(t[i] + 1) : 0ull);
    return k;
}

struct TokOrder {
    const int32_t *blob; const int64_t *start; const int32_t *len;
    // equal prefixes: either both tokens are shorter than 3 and equal, or both share their first 3 code points
    __device__ __forceinline__ int cmp(const TokKey &a, const TokKey &b) const {
        if (a.pre != b.pre) return a.pre < b.pre ? -1 : 1;
        const int la = len[a.occ], lb = len[b.occ];
        if (la <= 3 || lb <= 3) return la < lb ? -1 : (la > lb ? 1 : 0);
        return cp_cmp(blob + start[a.occ] + 3, la - 3, blob + start[b.occ] + 3, lb - 3);
    }
    __device__ __forceinline__ bool operator()(const TokKey &a, const TokKey &b) const { return cmp(a, b) < 0; }
};

// stream-ordered scratch, released on the stream when the entry point returns
struct Scratch {
    cudaStream_t st;
    void *ptrs[64]; int n = 0;
    explicit Scratch(cudaStream_t s) : st(s) {}
    ~Scratch() { for (int i = 0; i < n; ++i) cudaFreeAsync(ptrs[i], st); }
    template <typename T> cudaError_t get(T **p, int64_t count) {
        void *q = nullptr;
        if (n == 64) return cudaErrorMemoryAllocation;
        cudaError_t e = cudaMallocAsync(&q, (size_t)(count > 0 ? count : 1) * sizeof(T), st);
        if (e == cudaSuccess) ptrs[n++] = q;
        *p = (T *)q;
        return e;
    }
};

template <typename T>
static int excl_sum(Scratch &ws, const T *in, T *out, int64_t n) {
    size_t bytes = 0;
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, ws.st));
    void *tmp = nullptr;
    PFZ_CUDA_OK(ws.get((char **)&tmp, (int64_t)bytes));
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, n, ws.st));
    return 0;
}

// bit 0: first code point of its string, bit 1: last
__global__ void string_ends_kernel(const int64_t *__restrict__ off, int32_t n, uint8_t *__restrict__ ends) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int64_t a = off[s], b = off[s + 1];
    if (b - a == 1) ends[a] = 3;
    else if (b > a) { ends[a] = 1; ends[b - 1] = 2; }
}

// start[c] = 1 where a token starts (c is not whitespace, and begins its string or follows whitespace); start[n_chars] = 0
__global__ void token_starts_kernel(const int32_t *__restrict__ blob, const uint8_t *__restrict__ ends, int64_t n_chars,
                                    int32_t *__restrict__ start) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c > n_chars) return;
    if (c == n_chars) { start[c] = 0; return; }
    start[c] = !py_space(blob[c]) && ((ends[c] & 1) || py_space(blob[c - 1]));
}

// occurrence k (numbered by the scan of start) spans [tok_start[k], tok_start[k] + tok_len[k])
__global__ void token_spans_kernel(const int32_t *__restrict__ blob, const uint8_t *__restrict__ ends, int64_t n_chars,
                                   const int32_t *__restrict__ start, const int32_t *__restrict__ occx, int64_t *__restrict__ tok_start,
                                   int64_t *__restrict__ tok_end) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chars) return;
    const int32_t x = blob[c];
    if (py_space(x)) return;
    if (start[c]) tok_start[occx[c]] = c;
    if ((ends[c] & 2) || py_space(blob[c + 1])) tok_end[occx[c] + start[c] - 1] = c + 1;
}

// per string: its first occurrence, token count, and the string of each of its occurrences
__global__ void string_tokens_kernel(const int64_t *__restrict__ off, int32_t n, const int32_t *__restrict__ occx,
                                     int32_t *__restrict__ occ_ptr, int32_t *__restrict__ n_all, int32_t *__restrict__ tok_str) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int32_t a = occx[off[s]], b = occx[off[s + 1]];
    occ_ptr[s] = a; n_all[s] = b - a;
    if (s == n - 1) occ_ptr[n] = b;
    for (int32_t k = a; k < b; ++k) tok_str[k] = s;
}

__global__ void token_keys_kernel(const int32_t *__restrict__ blob, const int64_t *__restrict__ tok_start,
                                  const int64_t *__restrict__ tok_end, int32_t n_occ, int32_t *__restrict__ tok_len,
                                  TokKey *__restrict__ keys) {
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_occ) return;
    const int len = (int)(tok_end[k] - tok_start[k]);
    tok_len[k] = len;
    keys[k] = TokKey{prefix_key(blob + tok_start[k], len), k};
}

// head[i] = 1 where sorted occurrence i differs from its predecessor; head[n_occ] = 0
__global__ void token_heads_kernel(const TokKey *__restrict__ keys, int32_t n_occ, TokOrder ord, int32_t *__restrict__ head) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_occ) return;
    head[i] = i == n_occ ? 0 : (i == 0 || ord.cmp(keys[i - 1], keys[i]) != 0);
}

// rank of each occurrence; the vocabulary's representative occurrence and length per rank
__global__ void token_ranks_kernel(const TokKey *__restrict__ keys, int32_t n_occ, const int32_t *__restrict__ head,
                                   const int32_t *__restrict__ hx, const int32_t *__restrict__ tok_len, int32_t *__restrict__ local_id,
                                   int32_t *__restrict__ vrep, int64_t *__restrict__ vlen) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_occ) return;
    const int32_t occ = keys[i].occ, r = hx[i] + head[i] - 1;
    local_id[occ] = r;
    if (head[i]) { vrep[r] = occ; vlen[r] = tok_len[occ]; }
}

__global__ void vocab_copy_kernel(const int32_t *__restrict__ blob, const int64_t *__restrict__ tok_start, const int32_t *__restrict__ tok_len,
                                  const int32_t *__restrict__ vrep, const int32_t *__restrict__ n_vocab, const int64_t *__restrict__ vocab_off,
                                  int32_t *__restrict__ vocab_blob) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= *n_vocab) return;
    const int32_t occ = vrep[r];
    const int32_t *src = blob + tok_start[occ];
    int32_t *dst = vocab_blob + vocab_off[r];
    for (int i = 0; i < tok_len[occ]; ++i) dst[i] = src[i];
}

__global__ void pair_keys_kernel(const int32_t *__restrict__ tok_str, const int32_t *__restrict__ local_id, int32_t n_occ,
                                 uint64_t *__restrict__ pairs) {
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_occ) return;
    pairs[k] = ((uint64_t)tok_str[k] << 32) | (uint32_t)local_id[k];
}

// (string, id) pairs in order: the width of each in S(s) and U(s) (token + separator) and whether it is the string's first of its id
__global__ void pair_widths_kernel(const uint64_t *__restrict__ pairs, int32_t n_occ, const int32_t *__restrict__ occ_ptr,
                                   const int64_t *__restrict__ vocab_off, int64_t *__restrict__ ws, int64_t *__restrict__ wu,
                                   int32_t *__restrict__ wd) {
    const int32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n_occ) return;
    if (p == n_occ) { ws[p] = 0; wu[p] = 0; wd[p] = 0; return; }
    const int32_t s = (int32_t)(pairs[p] >> 32), id = (int32_t)(uint32_t)pairs[p];
    const bool distinct = p == occ_ptr[s] || (int32_t)(uint32_t)pairs[p - 1] != id;
    const int64_t w = vocab_off[id + 1] - vocab_off[id] + 1;
    ws[p] = w; wu[p] = distinct ? w : 0; wd[p] = distinct;
}

// per string: |S(s)|, |U(s)| (the widths less the last separator) and the first distinct id
__global__ void string_lens_kernel(int32_t n, int32_t n_occ, const int32_t *__restrict__ occ_ptr, const int64_t *__restrict__ xs,
                                   const int64_t *__restrict__ xu, const int32_t *__restrict__ xd, int64_t *__restrict__ s_len,
                                   int64_t *__restrict__ u_len, int32_t *__restrict__ tok_ptr) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n) return;
    if (s == n) { s_len[s] = 0; u_len[s] = 0; tok_ptr[n] = xd[n_occ]; return; }
    const int32_t a = occ_ptr[s], b = occ_ptr[s + 1];
    s_len[s] = b > a ? xs[b] - xs[a] - 1 : 0;
    u_len[s] = b > a ? xu[b] - xu[a] - 1 : 0;
    tok_ptr[s] = xd[a];
}

__global__ void pair_fill_kernel(const uint64_t *__restrict__ pairs, int32_t n_occ, const int32_t *__restrict__ occ_ptr,
                                 const int32_t *__restrict__ vocab_blob, const int64_t *__restrict__ vocab_off,
                                 const int64_t *__restrict__ xs, const int64_t *__restrict__ xu, const int32_t *__restrict__ xd,
                                 const int32_t *__restrict__ wd, const int64_t *__restrict__ s_off, const int64_t *__restrict__ u_off,
                                 int32_t *__restrict__ s_blob, int32_t *__restrict__ u_blob, int32_t *__restrict__ tok_ids) {
    const int32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_occ) return;
    const int32_t s = (int32_t)(pairs[p] >> 32), id = (int32_t)(uint32_t)pairs[p];
    const int32_t a = occ_ptr[s];
    const int32_t *src = vocab_blob + vocab_off[id];
    const int len = (int)(vocab_off[id + 1] - vocab_off[id]);
    int64_t pos = s_off[s] + xs[p] - xs[a];
    for (int i = 0; i < len; ++i) s_blob[pos + i] = src[i];
    if (pos + len < s_off[s + 1]) s_blob[pos + len] = 0x20;
    if (wd[p]) {
        pos = u_off[s] + xu[p] - xu[a];
        for (int i = 0; i < len; ++i) u_blob[pos + i] = src[i];
        if (pos + len < u_off[s + 1]) u_blob[pos + len] = 0x20;
        tok_ids[xd[p]] = id;
    }
}

__global__ void side_counts_kernel(int32_t n, int32_t n_occ, const int32_t *__restrict__ hx, const int64_t *__restrict__ vocab_off,
                                   const int64_t *__restrict__ s_off, const int64_t *__restrict__ u_off, const int32_t *__restrict__ xd,
                                   int64_t *__restrict__ out) {
    out[0] = n_occ; out[1] = hx[n_occ]; out[2] = vocab_off[hx[n_occ]]; out[3] = s_off[n]; out[4] = u_off[n]; out[5] = xd[n_occ];
}

// lower bound of token t in the sorted vocabulary (v_blob, v_off, n_v)
__device__ __forceinline__ int32_t vocab_lower_bound(const int32_t *t, int lt, const int32_t *v_blob, const int64_t *v_off, int32_t n_v,
                                                     bool *found) {
    int32_t lo = 0, hi = n_v;
    while (lo < hi) {
        const int32_t mid = lo + ((hi - lo) >> 1);
        const int c = cp_cmp(v_blob + v_off[mid], (int)(v_off[mid + 1] - v_off[mid]), t, lt);
        if (c < 0) lo = mid + 1; else hi = mid;
    }
    *found = lo < n_v && cp_cmp(v_blob + v_off[lo], (int)(v_off[lo + 1] - v_off[lo]), t, lt) == 0;
    return lo;
}

// Union ranks.  The union rank of a token x is (tokens of b before x) + (tokens of a before x that b lacks).  Pass 1 over a:
// each token's lower bound in b and whether b has it (shared[i]); the exclusive scan of shared counts the shared tokens of a
// before a given rank.
__global__ void union_probe_kernel(const int32_t *__restrict__ a_blob, const int64_t *__restrict__ a_off, int32_t n_a,
                                   const int32_t *__restrict__ b_blob, const int64_t *__restrict__ b_off, int32_t n_b,
                                   int32_t *__restrict__ lb_b, int32_t *__restrict__ shared) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_a) return;
    if (i == n_a) { shared[i] = 0; return; }
    bool found = false;
    lb_b[i] = vocab_lower_bound(a_blob + a_off[i], (int)(a_off[i + 1] - a_off[i]), b_blob, b_off, n_b, &found);
    shared[i] = found;
}

// pass 2 over a: rank = lb_b + (i - shared tokens of a before i); a token b lacks is written by a
__global__ void union_rank_a_kernel(const int64_t *__restrict__ a_off, int32_t n_a, const int32_t *__restrict__ lb_b,
                                    const int32_t *__restrict__ shared, const int32_t *__restrict__ shared_x, int32_t *__restrict__ map,
                                    int64_t *__restrict__ u_len) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_a) return;
    const int32_t r = lb_b[i] + i - shared_x[i];
    map[i] = r;
    if (!shared[i]) u_len[r] = a_off[i + 1] - a_off[i];
}

// over b: rank = j + (tokens of a before b[j]) - (shared ones among them); b writes every token it has
__global__ void union_rank_b_kernel(const int32_t *__restrict__ b_blob, const int64_t *__restrict__ b_off, int32_t n_b,
                                    const int32_t *__restrict__ a_blob, const int64_t *__restrict__ a_off, int32_t n_a,
                                    const int32_t *__restrict__ shared_x, int32_t *__restrict__ map, int64_t *__restrict__ u_len) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_b) return;
    bool found = false;
    const int len = (int)(b_off[j + 1] - b_off[j]);
    const int32_t la = vocab_lower_bound(b_blob + b_off[j], len, a_blob, a_off, n_a, &found);
    const int32_t r = j + la - shared_x[la];
    map[j] = r;
    u_len[r] = len;
}

__global__ void union_copy_kernel(const int32_t *__restrict__ x_blob, const int64_t *__restrict__ x_off, int32_t n_x,
                                  const int32_t *__restrict__ map, const int32_t *__restrict__ skip, const int64_t *__restrict__ u_off,
                                  int32_t *__restrict__ u_blob) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_x || (skip && skip[i])) return;
    const int32_t *src = x_blob + x_off[i];
    int32_t *dst = u_blob + u_off[map[i]];
    for (int64_t c = 0; c < x_off[i + 1] - x_off[i]; ++c) dst[c] = src[c];
}

__global__ void union_size_kernel(int32_t n_a, int32_t n_b, const int32_t *__restrict__ shared_x, int32_t *__restrict__ n_u) {
    *n_u = n_a + n_b - shared_x[n_a];
}

// one string per thread: ids through the map, and OR of 1 << (((id * 0x9E3779B1) >> 13) & 63) over them (a 64-bit product)
__global__ void remap_sig_kernel(const int32_t *__restrict__ tok_ptr, const int32_t *__restrict__ ids_in, int32_t n,
                                 const int32_t *__restrict__ map, int32_t *__restrict__ ids_out, uint64_t *__restrict__ sig) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    uint64_t b = 0;
    for (int32_t j = tok_ptr[s]; j < tok_ptr[s + 1]; ++j) {
        const int32_t id = map ? map[ids_in[j]] : ids_in[j];
        ids_out[j] = id;
        b |= 1ull << ((((uint64_t)(uint32_t)id * 0x9E3779B1ull) >> 13) & 63);
    }
    sig[s] = b;
}

}  // namespace
}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_tok_side(const int32_t *blob, const int64_t *offsets, int32_t n, int64_t n_chars, int32_t *n_all, int32_t *vocab_blob,
                 int64_t *vocab_off, int32_t *tok_ptr, int32_t *tok_ids, int64_t *s_off, int32_t *s_blob, int64_t *u_off,
                 int32_t *u_blob, int64_t *counts_host, void *stream) {
    PFZ_REQUIRE(n >= 0 && n_chars >= 0 && n_chars < INT32_MAX, "pfz_tok_side: %lld code points (at most 2^31 - 2)", (long long)n_chars);
    const cudaStream_t st = as_stream(stream);
    Scratch ws(st);
    uint8_t *ends; int32_t *start, *occx;
    PFZ_CUDA_OK(ws.get(&ends, n_chars)); PFZ_CUDA_OK(ws.get(&start, n_chars + 1)); PFZ_CUDA_OK(ws.get(&occx, n_chars + 1));
    PFZ_CUDA_OK(cudaMemsetAsync(ends, 0, (size_t)(n_chars > 0 ? n_chars : 1), st));
    if (n > 0) { string_ends_kernel<<<grid_of(n), TPB, 0, st>>>(offsets, n, ends); PFZ_LAUNCH_OK(); }
    token_starts_kernel<<<grid_of(n_chars + 1), TPB, 0, st>>>(blob, ends, n_chars, start); PFZ_LAUNCH_OK();
    if (excl_sum(ws, start, occx, n_chars + 1)) return 1;
    int32_t n_occ = 0;
    PFZ_CUDA_OK(cudaMemcpyAsync(&n_occ, occx + n_chars, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PFZ_CUDA_OK(cudaStreamSynchronize(st));

    int64_t *tok_start, *tok_end; int32_t *tok_len, *tok_str, *occ_ptr, *local_id, *head, *hx, *vrep, *xd, *wd;
    TokKey *keys; uint64_t *pairs, *pairs_sorted; int64_t *vlen, *w_s, *w_u, *x_s, *x_u, *l_s, *l_u, *cnt;
    PFZ_CUDA_OK(ws.get(&tok_start, n_occ)); PFZ_CUDA_OK(ws.get(&tok_end, n_occ)); PFZ_CUDA_OK(ws.get(&tok_len, n_occ));
    PFZ_CUDA_OK(ws.get(&tok_str, n_occ)); PFZ_CUDA_OK(ws.get(&occ_ptr, (int64_t)n + 1)); PFZ_CUDA_OK(ws.get(&local_id, n_occ));
    PFZ_CUDA_OK(ws.get(&head, n_occ + 1)); PFZ_CUDA_OK(ws.get(&hx, n_occ + 1)); PFZ_CUDA_OK(ws.get(&vrep, n_occ));
    PFZ_CUDA_OK(ws.get(&keys, n_occ)); PFZ_CUDA_OK(ws.get(&pairs, n_occ)); PFZ_CUDA_OK(ws.get(&pairs_sorted, n_occ));
    PFZ_CUDA_OK(ws.get(&vlen, n_occ + 1)); PFZ_CUDA_OK(ws.get(&w_s, n_occ + 1)); PFZ_CUDA_OK(ws.get(&w_u, n_occ + 1));
    PFZ_CUDA_OK(ws.get(&wd, n_occ + 1)); PFZ_CUDA_OK(ws.get(&x_s, n_occ + 1)); PFZ_CUDA_OK(ws.get(&x_u, n_occ + 1));
    PFZ_CUDA_OK(ws.get(&xd, n_occ + 1)); PFZ_CUDA_OK(ws.get(&l_s, (int64_t)n + 1)); PFZ_CUDA_OK(ws.get(&l_u, (int64_t)n + 1));
    PFZ_CUDA_OK(ws.get(&cnt, 6));

    token_spans_kernel<<<grid_of(n_chars), TPB, 0, st>>>(blob, ends, n_chars, start, occx, tok_start, tok_end); PFZ_LAUNCH_OK();
    if (n > 0) { string_tokens_kernel<<<grid_of(n), TPB, 0, st>>>(offsets, n, occx, occ_ptr, n_all, tok_str); PFZ_LAUNCH_OK(); }
    else PFZ_CUDA_OK(cudaMemsetAsync(occ_ptr, 0, sizeof(int32_t), st));
    token_keys_kernel<<<grid_of(n_occ), TPB, 0, st>>>(blob, tok_start, tok_end, n_occ, tok_len, keys); PFZ_LAUNCH_OK();
    const TokOrder ord{blob, tok_start, tok_len};
    if (n_occ > 1) {
        size_t bytes = 0;
        PFZ_CUDA_OK(cub::DeviceMergeSort::SortKeys(nullptr, bytes, keys, (int64_t)n_occ, ord, st));
        char *tmp;
        PFZ_CUDA_OK(ws.get(&tmp, (int64_t)bytes));
        PFZ_CUDA_OK(cub::DeviceMergeSort::SortKeys(tmp, bytes, keys, (int64_t)n_occ, ord, st));
    }
    token_heads_kernel<<<grid_of(n_occ + 1), TPB, 0, st>>>(keys, n_occ, ord, head); PFZ_LAUNCH_OK();
    if (excl_sum(ws, head, hx, (int64_t)n_occ + 1)) return 1;
    PFZ_CUDA_OK(cudaMemsetAsync(vlen, 0, sizeof(int64_t) * ((size_t)n_occ + 1), st));
    token_ranks_kernel<<<grid_of(n_occ), TPB, 0, st>>>(keys, n_occ, head, hx, tok_len, local_id, vrep, vlen); PFZ_LAUNCH_OK();
    // vocab_off has n_occ + 1 entries; those past the vocabulary's size all hold its total length
    if (excl_sum(ws, vlen, vocab_off, (int64_t)n_occ + 1)) return 1;
    vocab_copy_kernel<<<grid_of(n_occ), TPB, 0, st>>>(blob, tok_start, tok_len, vrep, hx + n_occ, vocab_off, vocab_blob); PFZ_LAUNCH_OK();

    // (string, id) pairs sorted: each string's ids ascending, duplicates adjacent
    pair_keys_kernel<<<grid_of(n_occ), TPB, 0, st>>>(tok_str, local_id, n_occ, pairs); PFZ_LAUNCH_OK();
    if (n_occ > 0) {
        size_t bytes = 0;
        PFZ_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, pairs, pairs_sorted, (int64_t)n_occ, 0, 64, st));
        char *tmp;
        PFZ_CUDA_OK(ws.get(&tmp, (int64_t)bytes));
        PFZ_CUDA_OK(cub::DeviceRadixSort::SortKeys(tmp, bytes, pairs, pairs_sorted, (int64_t)n_occ, 0, 64, st));
    }
    pair_widths_kernel<<<grid_of(n_occ + 1), TPB, 0, st>>>(pairs_sorted, n_occ, occ_ptr, vocab_off, w_s, w_u, wd); PFZ_LAUNCH_OK();
    if (excl_sum(ws, w_s, x_s, (int64_t)n_occ + 1) || excl_sum(ws, w_u, x_u, (int64_t)n_occ + 1) || excl_sum(ws, wd, xd, (int64_t)n_occ + 1))
        return 1;
    string_lens_kernel<<<grid_of((int64_t)n + 1), TPB, 0, st>>>(n, n_occ, occ_ptr, x_s, x_u, xd, l_s, l_u, tok_ptr); PFZ_LAUNCH_OK();
    if (excl_sum(ws, l_s, s_off, (int64_t)n + 1) || excl_sum(ws, l_u, u_off, (int64_t)n + 1)) return 1;
    pair_fill_kernel<<<grid_of(n_occ), TPB, 0, st>>>(pairs_sorted, n_occ, occ_ptr, vocab_blob, vocab_off, x_s, x_u, xd, wd, s_off, u_off,
                                                     s_blob, u_blob, tok_ids);
    PFZ_LAUNCH_OK();
    side_counts_kernel<<<1, 1, 0, st>>>(n, n_occ, hx, vocab_off, s_off, u_off, xd, cnt); PFZ_LAUNCH_OK();
    PFZ_CUDA_OK(cudaMemcpyAsync(counts_host, cnt, 6 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    PFZ_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

int pfz_tok_union(const int32_t *a_blob, const int64_t *a_off, int32_t n_a, const int32_t *b_blob, const int64_t *b_off, int32_t n_b,
                  int32_t *map_a, int32_t *map_b, int32_t *u_blob, int64_t *u_off, int32_t *n_u, void *stream) {
    PFZ_REQUIRE(n_a >= 0 && n_b >= 0, "pfz_tok_union: negative vocabulary size");
    const cudaStream_t st = as_stream(stream);
    Scratch ws(st);
    const int64_t cap = (int64_t)n_a + n_b;
    int64_t *u_len; int32_t *lb_b, *shared, *shared_x;
    PFZ_CUDA_OK(ws.get(&u_len, cap + 1)); PFZ_CUDA_OK(ws.get(&lb_b, n_a)); PFZ_CUDA_OK(ws.get(&shared, (int64_t)n_a + 1));
    PFZ_CUDA_OK(ws.get(&shared_x, (int64_t)n_a + 1));
    PFZ_CUDA_OK(cudaMemsetAsync(u_len, 0, sizeof(int64_t) * (size_t)(cap + 1), st));
    union_probe_kernel<<<grid_of((int64_t)n_a + 1), TPB, 0, st>>>(a_blob, a_off, n_a, b_blob, b_off, n_b, lb_b, shared); PFZ_LAUNCH_OK();
    if (excl_sum(ws, shared, shared_x, (int64_t)n_a + 1)) return 1;
    if (n_a) { union_rank_a_kernel<<<grid_of(n_a), TPB, 0, st>>>(a_off, n_a, lb_b, shared, shared_x, map_a, u_len); PFZ_LAUNCH_OK(); }
    if (n_b) { union_rank_b_kernel<<<grid_of(n_b), TPB, 0, st>>>(b_blob, b_off, n_b, a_blob, a_off, n_a, shared_x, map_b, u_len); PFZ_LAUNCH_OK(); }
    // u_off has n_a + n_b + 1 entries; those past the union's size all hold its total length
    if (excl_sum(ws, u_len, u_off, cap + 1)) return 1;
    if (n_a) { union_copy_kernel<<<grid_of(n_a), TPB, 0, st>>>(a_blob, a_off, n_a, map_a, shared, u_off, u_blob); PFZ_LAUNCH_OK(); }
    if (n_b) { union_copy_kernel<<<grid_of(n_b), TPB, 0, st>>>(b_blob, b_off, n_b, map_b, nullptr, u_off, u_blob); PFZ_LAUNCH_OK(); }
    union_size_kernel<<<1, 1, 0, st>>>(n_a, n_b, shared_x, n_u); PFZ_LAUNCH_OK();
    return 0;
}

int pfz_tok_remap(const int32_t *tok_ptr, const int32_t *ids_in, int32_t n, const int32_t *map, int32_t *ids_out, uint64_t *sig,
                  void *stream) {
    if (n <= 0) return 0;
    remap_sig_kernel<<<grid_of(n), TPB, 0, as_stream(stream)>>>(tok_ptr, ids_in, n, map, ids_out, sig);
    PFZ_LAUNCH_OK();
    return 0;
}

}  // extern "C"
