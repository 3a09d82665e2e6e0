// tav_compact.cu — order-preserving compaction of the rows after a removal (tav_remove_rows).
//
// The removed rows are given as keys[i] = rem[i] - i over the sorted, distinct removed ordinals rem[0..m).
// keys is non-decreasing (rem[i + 1] >= rem[i] + 1), and surviving row s lands on row d = s - #{rem < s}, so
// the source of destination d is s = d + #{i : keys[i] <= d}: one upper bound per warp, then a galloping
// walk over its run of consecutive destinations (a run of removed rows is a run of equal keys, which the walk
// crosses in a logarithmic number of loads, wherever in the warp's destinations it begins).
//
// Rows move only downwards, so a destination can be the source of a lower destination that has not been read
// yet: the gather never writes the buffer it reads.  The caller gathers either into a fresh allocation (out
// of place) or into a scratch window that is then copied back (in place, ascending windows: the sources of a
// window all lie at or above its first row, and rows above the window are written only by later windows).
//
// Every copy moves whole rows with vector loads and stores of V bytes, V the largest of 16 / 8 / 4 / 2 that
// divides the row width in bytes (rows of a multiple of 16 bytes take 16-byte accesses).

#include <algorithm>

#include "tav_internal.h"

namespace tav {
namespace {

constexpr int kCompactThreads = 256;
constexpr int kRowsPerWarp = 16;  // consecutive destinations per warp: one binary search for all of them
constexpr int kUnroll = 4;        // vectors per lane loaded before any is stored (a 2 KB row in one batch)

template <int V>
struct Vec;
template <>
struct Vec<16> { using T = uint4; };
template <>
struct Vec<8> { using T = uint2; };
template <>
struct Vec<4> { using T = uint32_t; };
template <>
struct Vec<2> { using T = uint16_t; };

// #{i : keys[i] <= d} given j = #{i : keys[i] <= d'} for some d' <= d: the next key decides in one load
// when no key lies in (d', d] (the common case); otherwise an exponential then a binary search from j
__device__ __forceinline__ int64_t upper_bound_from(const int64_t* __restrict__ keys, int64_t j, int64_t m, int64_t d) {
    if (j >= m || __ldg(keys + j) > d) return j;
    int64_t lo = j, step = 1, hi = j + 1;  // keys[lo] <= d
    while (hi < m && __ldg(keys + hi) <= d) {
        lo = hi;
        step <<= 1;
        hi = lo + step;
    }
    hi = min(hi, m);  // keys[hi] > d, or hi == m
    ++lo;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) <= d) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// destinations [d_begin, d_end) of the compacted rows: dst row (d - d_base) = src row (d + #{keys <= d})
template <int V>
__global__ void __launch_bounds__(kCompactThreads) compact_gather_kernel(
    const char* __restrict__ src, char* __restrict__ dst, const int64_t* __restrict__ keys, int64_t m,
    int64_t d_begin, int64_t d_end, int64_t d_base, int64_t row_vecs) {
    using T = typename Vec<V>::T;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * kCompactThreads + threadIdx.x) >> 5;
    const int64_t d0 = d_begin + warp * kRowsPerWarp;
    if (d0 >= d_end) return;
    const int64_t d1 = min(d0 + kRowsPerWarp, d_end);
    int64_t j = upper_bound_from(keys, 0, m, d0);  // #{i : keys[i] <= d0}
    for (int64_t d = d0; d < d1; ++d) {
        j = upper_bound_from(keys, j, m, d);
        const T* s = reinterpret_cast<const T*>(src) + (d + j) * row_vecs;
        T* t = reinterpret_cast<T*>(dst) + (d - d_base) * row_vecs;
        for (int64_t v0 = lane; v0 < row_vecs; v0 += 32 * kUnroll) {
            T r[kUnroll];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u)
                if (v0 + 32 * u < row_vecs) r[u] = s[v0 + 32 * u];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u)
                if (v0 + 32 * u < row_vecs) t[v0 + 32 * u] = r[u];
        }
    }
}

// n contiguous vectors src -> dst (the copy back of a scratch window)
template <int V>
__global__ void __launch_bounds__(kCompactThreads) compact_copy_kernel(const char* __restrict__ src,
                                                                      char* __restrict__ dst, int64_t n) {
    using T = typename Vec<V>::T;
    const T* s = reinterpret_cast<const T*>(src);
    T* t = reinterpret_cast<T*>(dst);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kCompactThreads;
    for (int64_t i0 = static_cast<int64_t>(blockIdx.x) * kCompactThreads + threadIdx.x; i0 < n; i0 += stride * kUnroll) {
        T r[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
            if (i0 + stride * u < n) r[u] = s[i0 + stride * u];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
            if (i0 + stride * u < n) t[i0 + stride * u] = r[u];
    }
}

int vec_bytes(size_t row_bytes) {
    for (int v : {16, 8, 4}) if (row_bytes % v == 0) return v;
    return 2;  // rows are a whole number of 16-bit elements
}

template <int V>
cudaError_t gather_v(const void* src, void* dst, const int64_t* keys, int64_t m, int64_t d_begin, int64_t d_end,
                     int64_t d_base, size_t row_bytes, cudaStream_t s) {
    const int64_t warps = (d_end - d_begin + kRowsPerWarp - 1) / kRowsPerWarp;
    const int64_t blocks = (warps * 32 + kCompactThreads - 1) / kCompactThreads;
    compact_gather_kernel<V><<<static_cast<unsigned>(blocks), kCompactThreads, 0, s>>>(
        static_cast<const char*>(src), static_cast<char*>(dst), keys, m, d_begin, d_end, d_base,
        static_cast<int64_t>(row_bytes / V));
    return cudaGetLastError();
}

template <int V>
cudaError_t copy_v(const void* src, void* dst, size_t bytes, int sms, cudaStream_t s) {
    const int64_t n = static_cast<int64_t>(bytes / V);
    const int64_t blocks = std::min<int64_t>((n + kCompactThreads - 1) / kCompactThreads, int64_t(sms) * 16);
    compact_copy_kernel<V><<<static_cast<unsigned>(blocks), kCompactThreads, 0, s>>>(
        static_cast<const char*>(src), static_cast<char*>(dst), n);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_compact_gather(const void* src, void* dst, const int64_t* keys, int64_t m, int64_t d_begin,
                                  int64_t d_end, int64_t d_base, size_t row_bytes, cudaStream_t s) {
    if (d_end <= d_begin) return cudaSuccess;
    switch (vec_bytes(row_bytes)) {
        case 16: return gather_v<16>(src, dst, keys, m, d_begin, d_end, d_base, row_bytes, s);
        case 8: return gather_v<8>(src, dst, keys, m, d_begin, d_end, d_base, row_bytes, s);
        case 4: return gather_v<4>(src, dst, keys, m, d_begin, d_end, d_base, row_bytes, s);
        default: return gather_v<2>(src, dst, keys, m, d_begin, d_end, d_base, row_bytes, s);
    }
}

cudaError_t launch_compact_copy(int device, const void* src, void* dst, int64_t n_rows, size_t row_bytes,
                                cudaStream_t s) {
    if (n_rows <= 0) return cudaSuccess;
    int sms = 0;
    cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (e != cudaSuccess) return e;
    const size_t bytes = static_cast<size_t>(n_rows) * row_bytes;
    switch (vec_bytes(row_bytes)) {  // a grid-stride copy: 16 CTAs per SM
        case 16: return copy_v<16>(src, dst, bytes, sms, s);
        case 8: return copy_v<8>(src, dst, bytes, sms, s);
        case 4: return copy_v<4>(src, dst, bytes, sms, s);
        default: return copy_v<2>(src, dst, bytes, sms, s);
    }
}

}  // namespace tav
