// gsr_binning.cu — (gaussian, tile) pair generation, depth sort and tile ranges, and the
// per-gaussian record packing of the reference-surface renderers.
//
// Replaces the reference's src/tile_culling.cu:124-340: instead of an fp64 key
// z + (max_z+1)*tile sorted by torch::sort plus an index_select, each pair gets
// the 64-bit key (tile << 32 | order-preserving bits of z) and is sorted together
// with its gaussian id by one cub::DeviceRadixSort over only the significant bits.
// Order is identical: (tile, z) ascending, ties by gaussian index (radix sort is
// stable and pairs are emitted in gaussian order) — SURVEY.md Q12.
#include <cub/cub.cuh>

#include "gsr_common.cuh"
#include "gsr_math.cuh"
#include "gsr_record.cuh"

namespace gsr {

constexpr int BIN_THREADS = 256;

// tiles overlapped by one gaussian.  Reference: src/tile_culling.cu:139-176.
// When keys != nullptr also emits the pairs at keys[base...].
// id_bits > 0: the gaussian id is packed into the low id_bits of the key, (tile | depth | id), and no ids
// array is written (keys-only sort); id_bits == 0: key = (tile | depth), ids[] holds the gaussian id.
__device__ __forceinline__ int walk_tiles(const Obb& o, float u, float v, int ntx, int nty,
                                          uint32_t zkey, uint32_t id, uint64_t* __restrict__ keys,
                                          uint32_t* __restrict__ ids, int64_t base, int depth_bits = 32,
                                          int id_bits = 0, int64_t cap = INT64_MAX) {
    int x0, x1, y0, y1;
    tile_window(u, v, o.radius_tiles, ntx, nty, x0, x1, y0, y1);
    int n = 0;
    for (int tx = x0; tx < x1; ++tx) {
        const float left = __fmul_rn(__int2float_rn(tx), 16.0f);
        const float right = __fmul_rn(__int2float_rn(tx + 1), 16.0f);
        for (int ty = y0; ty < y1; ++ty) {
            const float top = __fmul_rn(__int2float_rn(ty), 16.0f);
            const float bottom = __fmul_rn(__int2float_rn(ty + 1), 16.0f);
            if (obb_hits_tile(o, left, right, top, bottom)) {
                if (keys && base + n < cap) {  // cap: capacity of a speculatively sized pair buffer
                    const uint32_t tile = (uint32_t)(ty * ntx + tx);
                    const uint64_t k = ((uint64_t)tile << depth_bits) | zkey;
                    if (id_bits > 0) {
                        keys[base + n] = (k << id_bits) | id;
                    } else {
                        keys[base + n] = k;
                        ids[base + n] = id;
                    }
                }
                ++n;
            }
        }
    }
    return n;
}

__global__ void __launch_bounds__(BIN_THREADS)
    k_count_tiles(int N, const float* __restrict__ uvs, const float* __restrict__ conic, int ntx, int nty,
                  float mh, int32_t* __restrict__ counts) {
    const int i = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (i >= N) return;
    const float u = uvs[i * 2], v = uvs[i * 2 + 1];
    Obb o;
    compute_obb(u, v, __fadd_rn(conic[i * 3], 0.25f), __fmul_rn(conic[i * 3 + 1], 0.5f),
                __fadd_rn(conic[i * 3 + 2], 0.25f), mh, o);
    counts[i] = walk_tiles(o, u, v, ntx, nty, 0u, 0u, nullptr, nullptr, 0);
}

__global__ void __launch_bounds__(BIN_THREADS)
    k_emit_pairs_api(int N, const float* __restrict__ uvs, const float* __restrict__ xyz_cam,
                     const float* __restrict__ conic, int ntx, int nty, float mh,
                     const int32_t* __restrict__ offsets, uint64_t* __restrict__ keys,
                     uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (i >= N) return;
    if (offsets[i + 1] == offsets[i]) return;
    const float u = uvs[i * 2], v = uvs[i * 2 + 1];
    Obb o;
    compute_obb(u, v, __fadd_rn(conic[i * 3], 0.25f), __fmul_rn(conic[i * 3 + 1], 0.5f),
                __fadd_rn(conic[i * 3 + 2], 0.25f), mh, o);
    walk_tiles(o, u, v, ntx, nty, depth_key(xyz_cam[i * 3 + 2]), (uint32_t)i, keys, ids, offsets[i]);
}

// fused path: the record already holds a, 2b, c (b = 0.5 * 2b is exact)
__global__ void __launch_bounds__(BIN_THREADS)
    k_emit_pairs_fused(int N, const float* __restrict__ records,
                       const uint32_t* __restrict__ zkey, const uint8_t* __restrict__ visible,
                       const uint64_t* __restrict__ scan, int ntx, int nty, float mh, int depth_bits,
                       int id_bits, uint64_t* __restrict__ keys, uint32_t* __restrict__ ids,
                       int32_t* __restrict__ vis_idx, float* __restrict__ uv_compact, int64_t cap,
                       const uint64_t* __restrict__ tile_mask, const uint32_t* __restrict__ tile_win) {
    const int i = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (cap > 0) {
        // Speculatively sized buffers (the host has not read P yet): positions [P, cap) get the all-ones key, which
        // sorts behind every real pair (tile field >= n_tiles) and is ignored by the range kernel
        const int64_t P = (int64_t)(scan[N - 1] & 0xffffffffu);
        for (int64_t p = P + (int64_t)blockIdx.x * BIN_THREADS + threadIdx.x; p < cap;
             p += (int64_t)gridDim.x * BIN_THREADS) {
            keys[p] = ~0ull;
            if (ids != nullptr) ids[p] = 0u;
        }
    }
    if (i >= N) return;
    if (!visible[i]) return;
    const uint64_t incl = scan[i];
    const uint64_t prev = (i > 0) ? scan[i - 1] : 0ull;
    const uint32_t rank = (uint32_t)(prev >> 32);
    const uint32_t cnt = (uint32_t)(incl & 0xffffffffu) - (uint32_t)(prev & 0xffffffffu);
    const float u = records[(size_t)i * REC + R_U], v = records[(size_t)i * REC + R_V];
    vis_idx[rank] = i;
    uv_compact[rank * 2 + 0] = u;
    uv_compact[rank * 2 + 1] = v;
    if (cnt == 0) return;
    const uint32_t win = (tile_win != nullptr) ? tile_win[i] : 0xffffffffu;
    if (win != 0xffffffffu) {
        // the per-gaussian stage already tested this gaussian's tile window: expand its hit mask (ascending bit =
        // the enumeration order of walk_tiles: x-major, then y)
        uint64_t m = tile_mask[i];
        const int x0 = (int)(win & 0xffu), y0 = (int)((win >> 8) & 0xffu), wy = (int)(win >> 24);
        const int64_t base = (int64_t)(prev & 0xffffffffu);
        const int64_t lim = cap > 0 ? cap : INT64_MAX;
        // key = tile << (depth_bits + id_bits) | low; everything below the tile field is the same for all pairs
        const int tile_shift = depth_bits + id_bits;
        const uint64_t low = (id_bits > 0) ? (((uint64_t)zkey[i] << id_bits) | (uint32_t)i) : (uint64_t)zkey[i];
        // bit b = x * wy + y, ascending: the column is tracked incrementally — no division per pair
        int n = 0, col0 = 0, tx = x0;
        while (m) {
            const int b = __ffsll((long long)m) - 1;
            m &= m - 1;
            while (b - col0 >= wy) {
                col0 += wy;
                ++tx;
            }
            if (base + n < lim) {
                keys[base + n] = ((uint64_t)(uint32_t)((y0 + b - col0) * ntx + tx) << tile_shift) | low;
                if (id_bits == 0) ids[base + n] = (uint32_t)i;
            }
            ++n;
        }
        return;
    }
    Obb o;
    const float* r = records + (size_t)i * REC;
    compute_obb(u, v, r[R_A], __fmul_rn(r[R_B2], 0.5f), r[R_C], mh, o);
    walk_tiles(o, u, v, ntx, nty, zkey[i], (uint32_t)i, keys, ids, (int64_t)(prev & 0xffffffffu), depth_bits,
               id_bits, cap > 0 ? cap : INT64_MAX);
}

// tile_ranges[t] = first sorted position whose tile id >= t  (ranges[n_tiles] = P).
// One block stages BIN_THREADS+1 tile ids through shared memory; each position closes the
// ranges of every tile id in (tile[p-1], tile[p]].
__global__ void __launch_bounds__(BIN_THREADS)
    k_tile_ranges(int P, int n_tiles, int depth_bits, const uint64_t* __restrict__ keys,
                  int32_t* __restrict__ ranges) {
    __shared__ int32_t s_tile[BIN_THREADS + 1];
    const int p0 = blockIdx.x * BIN_THREADS;
    const int p = p0 + threadIdx.x;
    // padding keys (all ones, speculatively sized buffers) carry a tile field >= n_tiles: clamp it, so that the
    // first padding position closes every remaining range and the others close nothing
    if (p < P) s_tile[threadIdx.x + 1] = (int32_t)min((uint64_t)n_tiles, keys[p] >> depth_bits);
    if (threadIdx.x == 0) s_tile[0] = (p0 > 0) ? (int32_t)min((uint64_t)n_tiles, keys[p0 - 1] >> depth_bits) : -1;
    __syncthreads();
    if (p >= P) return;
    const int cur = s_tile[threadIdx.x + 1];
    const int prev = s_tile[threadIdx.x];
    for (int t = prev + 1; t <= cur; ++t) ranges[t] = p;  // cur <= n_tiles: ranges has n_tiles + 1 entries
    if (p == P - 1)
        for (int t = cur + 1; t <= n_tiles; ++t) ranges[t] = P;
}

__global__ void k_fill_i32(int n, int32_t* __restrict__ out, int32_t value) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = value;
}

__global__ void __launch_bounds__(BIN_THREADS) k_ids_to_i32(int P, const uint32_t* __restrict__ in,
                                                            int32_t* __restrict__ out) {
    const int p = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (p < P) out[p] = (int32_t)in[p];
}

__global__ void __launch_bounds__(BIN_THREADS)
    k_pack_records(int N, const float* __restrict__ uvs, const float* __restrict__ opacity,
                   const float* __restrict__ rgb, const float* __restrict__ conic, float* __restrict__ out) {
    const int g = blockIdx.x * BIN_THREADS + threadIdx.x;
    if (g >= N) return;
    float rec[REC];
    make_record(uvs[g * 2], uvs[g * 2 + 1], conic[g * 3], conic[g * 3 + 1], conic[g * 3 + 2], opacity[g],
                rgb[g * 3], rgb[g * 3 + 1], rgb[g * 3 + 2], rec);
    float4* o = reinterpret_cast<float4*>(out + (size_t)g * REC);
    o[0] = make_float4(rec[0], rec[1], rec[2], rec[3]);
    o[1] = make_float4(rec[4], rec[5], rec[6], rec[7]);
    o[2] = make_float4(rec[8], rec[9], rec[10], rec[11]);
}

// tile field width: 2^bits > n_tiles (strictly), so that the all-ones tile id never names a real tile — it is the
// padding key of speculatively sized pair buffers and must sort behind every real pair
static inline int sort_end_bit(int n_tiles, int depth_bits) {
    int bits = 1;
    while ((1 << bits) <= n_tiles) ++bits;
    return depth_bits + bits;
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace gsr

using namespace gsr;

#define BGRID(n) dim3((unsigned)(((int64_t)(n) + BIN_THREADS - 1) / BIN_THREADS)), dim3(BIN_THREADS), 0, st

extern "C" {

size_t gsr_binning_count_temp_bytes(int N) {
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_bytes, (int32_t*)nullptr, (int32_t*)nullptr, N + 1);
    return align256(scan_bytes) + align256(sizeof(int32_t) * (size_t)(N + 1));
}

int gsr_binning_count(int N, const float* uvs, const float* conic, int ntx, int nty, float mh,
                      int32_t* offsets, void* temp, size_t temp_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || temp_bytes < gsr_binning_count_temp_bytes(N)) return GSR_ERR_BAD_ARG;
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_bytes, (int32_t*)nullptr, (int32_t*)nullptr, N + 1);
    int32_t* counts = reinterpret_cast<int32_t*>((char*)temp + align256(scan_bytes));
    // counts has N+1 entries, the last one 0, so the exclusive scan yields offsets[N] == P
    k_fill_i32<<<1, 1, 0, st>>>(1, counts + N, 0);
    if (N > 0) k_count_tiles<<<BGRID(N)>>>(N, uvs, conic, ntx, nty, mh, counts);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(temp, scan_bytes, counts, offsets, N + 1, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

size_t gsr_sort_pairs_temp_bytes(int P) {
    size_t b = 0;
    cub::DeviceRadixSort::SortPairs((void*)nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr,
                                    (uint32_t*)nullptr, (uint32_t*)nullptr, P > 0 ? P : 1, 0, 64);
    return align256(b);
}

int gsr_sort_pairs(int P, int n_tiles, int depth_bits, const uint64_t* keys_in, const uint32_t* ids_in,
                   uint64_t* keys_out, uint32_t* ids_out, void* temp, size_t temp_bytes, void* stream) {
    if (P <= 0) return GSR_OK;
    if (depth_bits < 1 || depth_bits > 32) return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    size_t b = temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, b, keys_in, keys_out, ids_in, ids_out, P, 0,
                                                    sort_end_bit(n_tiles, depth_bits), st);
    return (int)e;
}

int gsr_tile_ranges(int P, int n_tiles, int depth_bits, const uint64_t* keys_sorted, int32_t* ranges,
                    void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0) {
        k_fill_i32<<<BGRID(n_tiles + 1)>>>(n_tiles + 1, ranges, 0);
    } else {
        k_tile_ranges<<<BGRID(P)>>>(P, n_tiles, depth_bits, keys_sorted, ranges);
    }
    return (int)cudaGetLastError();
}

size_t gsr_binning_sort_temp_bytes(int P) {
    const size_t p = (size_t)(P > 0 ? P : 1);
    return gsr_sort_pairs_temp_bytes(P) + 2 * align256(8 * p) + 2 * align256(4 * p);
}

int gsr_binning_emit_sort(int N, int P, const float* uvs, const float* xyz_cam, const float* conic,
                          int ntx, int nty, float mh, const int32_t* offsets, int32_t* sorted_idx,
                          int32_t* ranges, void* temp, size_t temp_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int n_tiles = ntx * nty;
    if (temp_bytes < gsr_binning_sort_temp_bytes(P)) return GSR_ERR_BAD_ARG;
    if (P <= 0) return gsr_tile_ranges(0, n_tiles, 32, nullptr, ranges, stream);
    const size_t p = (size_t)P;
    char* base = (char*)temp;
    const size_t sort_bytes = gsr_sort_pairs_temp_bytes(P);
    uint64_t* keys_a = (uint64_t*)(base + sort_bytes);
    uint64_t* keys_b = (uint64_t*)((char*)keys_a + align256(8 * p));
    uint32_t* ids_a = (uint32_t*)((char*)keys_b + align256(8 * p));
    uint32_t* ids_b = (uint32_t*)((char*)ids_a + align256(4 * p));
    k_emit_pairs_api<<<BGRID(N)>>>(N, uvs, xyz_cam, conic, ntx, nty, mh, offsets, keys_a, ids_a);
    int rc = gsr_sort_pairs(P, n_tiles, 32, keys_a, ids_a, keys_b, ids_b, temp, sort_bytes, stream);
    if (rc) return rc;
    k_ids_to_i32<<<BGRID(P)>>>(P, ids_b, sorted_idx);
    return gsr_tile_ranges(P, n_tiles, 32, keys_b, ranges, stream);
}

int gsr_emit_pairs(int N, const float* records, const uint32_t* depth_key,
                   const uint8_t* visible, const uint64_t* scan, int ntx, int nty, float mh, int depth_bits,
                   uint64_t* keys, uint32_t* ids, int32_t* vis_idx, float* uv_compact, int64_t capacity,
                   const uint64_t* tile_mask, const uint32_t* tile_win, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (N <= 0) return GSR_OK;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    k_emit_pairs_fused<<<BGRID(N)>>>(N, records, depth_key, visible, scan, ntx, nty, mh, depth_bits, 0, keys,
                                     ids, vis_idx, uv_compact, capacity, tile_mask, tile_win);
    return (int)cudaGetLastError();
}

// ---- keys-only variant: (tile | depth | gaussian id) in one 64-bit key -------------------------------
int gsr_packed_id_bits(int N, int n_tiles, int depth_bits) {
    int id_bits = 1;
    while (((int64_t)1 << id_bits) < (int64_t)N) ++id_bits;
    return (sort_end_bit(n_tiles, depth_bits) + id_bits <= 64) ? id_bits : 0;
}

int gsr_emit_keys(int N, const float* records, const uint32_t* depth_key, const uint8_t* visible,
                  const uint64_t* scan, int ntx, int nty, float mh, int depth_bits, int id_bits, uint64_t* keys,
                  int32_t* vis_idx, float* uv_compact, int64_t capacity, const uint64_t* tile_mask,
                  const uint32_t* tile_win, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (N <= 0) return GSR_OK;
    if (id_bits < 1 || id_bits != gsr_packed_id_bits(N, ntx * nty, depth_bits)) return GSR_ERR_BAD_ARG;
    if ((tile_mask == nullptr) != (tile_win == nullptr)) return GSR_ERR_BAD_ARG;
    k_emit_pairs_fused<<<BGRID(N)>>>(N, records, depth_key, visible, scan, ntx, nty, mh, depth_bits, id_bits, keys,
                                     nullptr, vis_idx, uv_compact, capacity, tile_mask, tile_win);
    return (int)cudaGetLastError();
}

size_t gsr_sort_keys_temp_bytes(int P) {
    size_t b = 0;
    cub::DeviceRadixSort::SortKeys((void*)nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, P > 0 ? P : 1, 0, 64);
    return align256(b);
}

int gsr_sort_keys(int P, int n_tiles, int depth_bits, int id_bits, const uint64_t* keys_in, uint64_t* keys_out,
                  void* temp, size_t temp_bytes, void* stream) {
    if (P <= 0) return GSR_OK;
    if (depth_bits < 1 || depth_bits > 32 || id_bits < 1) return GSR_ERR_BAD_ARG;
    size_t b = temp_bytes;
    // the id bits are NOT sorted: the sort is stable and pairs are emitted in gaussian order
    cudaError_t e = cub::DeviceRadixSort::SortKeys(temp, b, keys_in, keys_out, P, id_bits,
                                                   id_bits + sort_end_bit(n_tiles, depth_bits), (cudaStream_t)stream);
    return (int)e;
}

int gsr_pack_gaussian_records(int N, const float* uvs, const float* opacity, const float* rgb, const float* conic,
                              float* records, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (N <= 0) return GSR_OK;
    k_pack_records<<<BGRID(N)>>>(N, uvs, opacity, rgb, conic, records);
    return (int)cudaGetLastError();
}

}  // extern "C"
