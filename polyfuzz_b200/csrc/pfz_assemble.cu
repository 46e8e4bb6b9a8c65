// pfz_assemble.cu -- K5: the frame tail on the device.  From the top-k arrays to the COLUMNS of the result frame:
// per rank r the rounded similarities, the validity bitmap and the matched to-strings gathered into one Arrow string
// column (int64 offsets -- Arrow large_string, the layout pandas' str dtype holds, so that the host wraps it without a cast --
// + UTF-8 bytes), ready to be wrapped zero-copy by the host.
//
// Replaces the tail of polyfuzz/models/_utils.py:104-125: `matches = [[to_list[idx] for idx in indices[:, i]] ...]`,
// the (1 + 2k) x n unicode ndarray, the 3-decimal rounding (:102 / :143) and the `Similarity < 0.001 -> 0, To -> None`
// rule (:119-123).  The strings must be ASCII (bytes == code points; the host checks while packing); other lists take
// the host Arrow path.
#include <cub/device/device_scan.cuh>
#include "pfz_common.cuh"

namespace pfz {

// entry e = r * n + i (column-major).  sims[e] = round(val, 3) or 0; lens[e] = byte length of the matched string or 0 (int64:
// their prefix sum, the byte positions, reaches 2^31 once a frame's matched strings total 2 GiB);
// bitmap bit i of column r = 1 iff the slot holds a match with a rounded score >= 0.001.
__global__ void __launch_bounds__(256) tail_count_kernel(const int32_t *__restrict__ idx, const double *__restrict__ val, int n, int k,
                                                         const int64_t *__restrict__ to_off, double *__restrict__ sims, int64_t *__restrict__ lens,
                                                         uint32_t *__restrict__ bitmap, int words_per_col) {
    const int lane = lane_id();
    const int64_t total = (int64_t)k * (((int64_t)n + 31) / 32) * 32;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int n32 = ((n + 31) / 32) * 32;
        const int r = (int)(t / n32), i = (int)(t - (int64_t)r * n32);
        bool ok = false; double s = 0.0; int64_t len = 0;
        if (i < n) {
            const int j = idx[(int64_t)i * k + r];
            s = __ddiv_rn(rint(__dmul_rn(val[(int64_t)i * k + r], 1000.0)), 1000.0);      // np.round(x, 3)
            ok = j >= 0 && !(s < 0.001);
            if (ok) len = to_off[j + 1] - to_off[j]; else s = 0.0;
            sims[(int64_t)r * n + i] = s;
            lens[(int64_t)r * n + i] = len;
        }
        const unsigned m = __ballot_sync(FULL, ok);
        if (lane == 0) bitmap[(int64_t)r * words_per_col + (i >> 5)] = m;
    }
}

// one warp per entry: copy the matched string's code points (ASCII) as bytes; offsets relative to the column start
__global__ void __launch_bounds__(256) tail_copy_kernel(const int32_t *__restrict__ idx, int n, int k, const int32_t *__restrict__ to_blob,
                                                        const int64_t *__restrict__ to_off, const int64_t *__restrict__ pos,
                                                        int64_t *__restrict__ offsets, uint8_t *__restrict__ data) {
    const int lane = lane_id();
    const int64_t n_ent = (int64_t)n * k;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t e = gw; e < n_ent; e += nw) {
        const int r = (int)(e / n), i = (int)(e - (int64_t)r * n);
        const int64_t p0 = pos[e], len = pos[e + 1] - p0;
        const int64_t col0 = pos[(int64_t)r * n];
        if (lane == 0) {
            offsets[(int64_t)r * (n + 1) + i] = p0 - col0;
            if (i == n - 1) offsets[(int64_t)r * (n + 1) + n] = pos[e + 1] - col0;
        }
        if (len > 0) {
            const int j = idx[(int64_t)i * k + r];
            const int64_t src = to_off[j];
            for (int64_t c = lane; c < len; c += 32) data[p0 + c] = (uint8_t)to_blob[src + c];
        }
    }
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int64_t pfz_frame_tail_ws_bytes(int64_t n_entries) {
    size_t bytes = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int64_t *)nullptr, n_entries + 1) != cudaSuccess) return -1;
    return (int64_t)bytes;
}

int pfz_frame_tail_count(const int32_t *top_idx, const double *top_val, int32_t n, int32_t k, const int64_t *to_offsets, double *sims,
                         int64_t *lens_pos, uint32_t *bitmap, void *ws, int64_t ws_bytes, void *stream) {
    if (n <= 0 || k <= 0) return 0;
    cudaStream_t st = as_stream(stream);
    const int words_per_col = (n + 31) / 32;
    const int64_t total = (int64_t)k * words_per_col * 32;
    int grid = (int)((total + 255) / 256); if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    PFZ_CUDA_OK(cudaMemsetAsync(lens_pos + (int64_t)n * k, 0, sizeof(int64_t), st));
    tail_count_kernel<<<grid, 256, 0, st>>>(top_idx, top_val, n, k, to_offsets, sims, lens_pos, bitmap, words_per_col);
    PFZ_LAUNCH_OK();
    size_t bytes = (size_t)ws_bytes;
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(ws, bytes, lens_pos, (int64_t)n * k + 1, st));
    return 0;
}

int pfz_frame_tail_copy(const int32_t *top_idx, int32_t n, int32_t k, const int32_t *to_blob, const int64_t *to_offsets, const int64_t *pos,
                        int64_t *offsets, uint8_t *data, void *stream) {
    if (n <= 0 || k <= 0) return 0;
    const int64_t n_ent = (int64_t)n * k;
    int grid = (int)((n_ent * 32 + 255) / 256); if (grid > SM_COUNT * 16) grid = SM_COUNT * 16;
    tail_copy_kernel<<<grid, 256, 0, as_stream(stream)>>>(top_idx, n, k, to_blob, to_offsets, pos, offsets, data);
    PFZ_LAUNCH_OK();
    return 0;
}
}
