// sm_90a kernels of the multi-version Confluent decode (rv_decode_*_versions, DESIGN.md §7 "Several writer schemas").
//
//   vp_count_kernel    one lane per message: the Confluent or single-object header, the writer of its schema id or
//                      fingerprint (binary search in the registered keys, staged in shared memory), per tile the
//                      messages and bytes of every writer
//   vp_scan_kernel     one CTA per (output chunk, writer): the tiles' counts scanned into bases, the group's totals
//   vp_scatter_kernel  one lane per message: its rank in its group (warp shuffles + per-warp totals in shared memory),
//                      the group's i64 offsets, the space-0 row map; each warp copies its messages' bytes together
//   take_rows_kernel   one lane per output row of one (chunk, row space): bits by __ballot_sync, fixed-width values by
//                      gather, and per block the summed lengths of every offsets slot
//   take_scan_kernel   one CTA per offsets slot: the block sums scanned into block bases
//   take_offsets_kernel  one lane per output row: offsets, Utf8 / Binary bytes, the child row space's row map
//   vp_report_kernel   permissive registries: one lane per bad message, its message index and its header
//
// Permissive registries (rv_versions_permissive) run the *_perm instances of the same bodies: a message that fails its
// header check joins the chunk's bad group instead of setting the error word, the scatter records the inverse of the row
// map, and the take writes a null row for a kNoRow entry.  The strict kernels keep their code.
#include "kernels.cuh"

#include "plan.hpp"
#include "take.cuh"

namespace rv {
namespace {

constexpr int kVpWarps = kTakeBlock / 32;

struct TileRange { int chunk; int64_t r0, end; };

__device__ __forceinline__ TileRange tile_range(const VersionsParams& p, int t) {
    const int j = min(t / p.tiles_per_chunk, p.k - 1);
    const int64_t cs = int64_t(j) * p.chunk_rows;
    TileRange tr;
    tr.chunk = j;
    tr.r0 = cs + int64_t(t - j * p.tiles_per_chunk) * kTakeBlock;
    tr.end = (j == p.k - 1) ? p.n : cs + p.chunk_rows;
    return tr;
}

// Key: uint32_t (Confluent schema ids, p.ids) or unsigned long long (single-object fingerprints, p.fps).
template <class Key>
__device__ __forceinline__ const Key* vp_keys(const VersionsParams& p);
template <>
__device__ __forceinline__ const uint32_t* vp_keys<uint32_t>(const VersionsParams& p) { return p.ids; }
template <>
__device__ __forceinline__ const unsigned long long* vp_keys<unsigned long long>(const VersionsParams& p) { return p.fps; }

// PERM: the tables have a last column, the bad group, which counts the messages that fail their header check.
template <class Key, bool PERM>
__device__ __forceinline__ void vp_count_body(const VersionsParams& p) {
    __shared__ Key s_ids[kMaxVersions];
    __shared__ uint32_t s_cnt[kMaxVersions + (PERM ? 1 : 0)];
    __shared__ unsigned long long s_bytes[kMaxVersions + (PERM ? 1 : 0)];
    const int W = PERM ? p.n_ids - 1 : p.n_ids;  // registered keys
    const int WT = p.n_ids;                       // table columns
    for (int w = threadIdx.x; w < WT; w += kTakeBlock) {
        if (!PERM || w < W) s_ids[w] = vp_keys<Key>(p)[w];
        s_cnt[w] = 0;
        s_bytes[w] = 0;
    }
    __syncthreads();
    const TileRange tr = tile_range(p, int(blockIdx.x));
    const int64_t row = tr.r0 + threadIdx.x;
    if (row < tr.end) {
        const int64_t a = p.offsets[row], len = p.offsets[row + 1] - a;
        int w = -1;
        const uint32_t code = vp_header(p.data + a, len, s_ids, W, &w);
        if (code != E_OK) {
            if (PERM) {
                atomicAdd(&s_cnt[W], 1u);
                p.bad[atomicAdd(p.n_bad, 1ull)] = (static_cast<unsigned long long>(row) << 8) | code;
            } else {
                atomicMin(p.err, (static_cast<unsigned long long>(row) << 8) | code);
            }
            w = -1;
        } else {
            atomicAdd(&s_cnt[w], 1u);
            atomicAdd(&s_bytes[w], static_cast<unsigned long long>(len));
        }
        p.msg_w[row] = uint16_t(w < 0 ? 0xFFFF : w);
    }
    __syncthreads();
    for (int w = threadIdx.x; w < WT; w += kTakeBlock) {
        p.tile_cnt[size_t(blockIdx.x) * WT + w] = s_cnt[w];
        p.tile_bytes[size_t(blockIdx.x) * WT + w] = s_bytes[w];
    }
}

template <class Key>
__global__ void __launch_bounds__(kTakeBlock) vp_count_kernel(const VersionsParams p) { vp_count_body<Key, false>(p); }
template <class Key>
__global__ void __launch_bounds__(kTakeBlock) vp_count_perm_kernel(const VersionsParams p) { vp_count_body<Key, true>(p); }

// Exclusive scan of a chunk's tile counts and bytes of writer blockIdx.y (in place), in the manner of encode_scan_kernel.
__global__ void __launch_bounds__(kTakeBlock) vp_scan_kernel(const VersionsParams p) {
    __shared__ unsigned long long s_c[kVpWarps], s_b[kVpWarps];
    const int j = blockIdx.x, w = blockIdx.y, W = p.n_ids;
    const int t_begin = j * p.tiles_per_chunk, t_end = (j == p.k - 1) ? p.n_tiles : t_begin + p.tiles_per_chunk;
    const int T = t_end - t_begin, per = (T + kTakeBlock - 1) / kTakeBlock;
    const int a = t_begin + min(T, int(threadIdx.x) * per), b = t_begin + min(T, (int(threadIdx.x) + 1) * per);
    unsigned long long lc = 0, lb = 0;
    for (int i = a; i < b; ++i) { lc += p.tile_cnt[size_t(i) * W + w]; lb += p.tile_bytes[size_t(i) * W + w]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long ic = lc, ib = lb;
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long vc = __shfl_up_sync(0xFFFFFFFFu, ic, d), vb = __shfl_up_sync(0xFFFFFFFFu, ib, d);
        if (lane >= d) { ic += vc; ib += vb; }
    }
    if (lane == 31) { s_c[warp] = ic; s_b[warp] = ib; }
    __syncthreads();
    if (warp == 0) {
        const unsigned long long vc = lane < kVpWarps ? s_c[lane] : 0ull, vb = lane < kVpWarps ? s_b[lane] : 0ull;
        unsigned long long xc = vc, xb = vb;
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long uc = __shfl_up_sync(0xFFFFFFFFu, xc, d), ub = __shfl_up_sync(0xFFFFFFFFu, xb, d);
            if (lane >= d) { xc += uc; xb += ub; }
        }
        if (lane < kVpWarps) { s_c[lane] = xc - vc; s_b[lane] = xb - vb; }
        if (lane == 31) { p.group_tot[(size_t(j) * W + w) * 2] = xc; p.group_tot[(size_t(j) * W + w) * 2 + 1] = xb; }
    }
    __syncthreads();
    unsigned long long rc = s_c[warp] + (ic - lc), rb = s_b[warp] + (ib - lb);
    for (int i = a; i < b; ++i) {
        const uint32_t c = p.tile_cnt[size_t(i) * W + w];
        const unsigned long long by = p.tile_bytes[size_t(i) * W + w];
        p.tile_cnt[size_t(i) * W + w] = uint32_t(rc);
        p.tile_bytes[size_t(i) * W + w] = rb;
        rc += c;
        rb += by;
    }
}

// PERM: the bad group (the tables' last column) takes no rank, bytes or offsets; every group row's message goes to p.inv.
template <bool PERM>
__device__ __forceinline__ void vp_scatter_body(const VersionsParams& p) {
    __shared__ uint32_t s_wc[kVpWarps][kMaxVersions];
    __shared__ unsigned long long s_wb[kVpWarps][kMaxVersions];
    const int W = p.n_ids;
    const int WK = PERM ? W - 1 : W;
    for (int i = threadIdx.x; i < kVpWarps * WK; i += kTakeBlock) { s_wc[i / WK][i % WK] = 0; s_wb[i / WK][i % WK] = 0; }
    __syncthreads();
    const TileRange tr = tile_range(p, int(blockIdx.x));
    const int64_t row = tr.r0 + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int w = -1;
    int64_t a = 0, len = 0;
    if (row < tr.end) {
        const uint16_t m = p.msg_w[row];
        if (m != 0xFFFF) { w = m; a = p.offsets[row]; len = p.offsets[row + 1] - a; }
    }
    // rank and byte position among the warp's messages of the same writer
    uint32_t pc = 0, tc = 0;
    unsigned long long pb = 0, tb = 0;
    for (int i = 0; i < 32; ++i) {
        const int wi = __shfl_sync(0xFFFFFFFFu, w, i);
        const long long li = __shfl_sync(0xFFFFFFFFu, len, i);
        if (wi == w) { tc += 1; tb += (unsigned long long)li; if (i < lane) { pc += 1; pb += (unsigned long long)li; } }
    }
    if (w >= 0 && pc + 1 == tc) { s_wc[warp][w] = tc; s_wb[warp][w] = tb; }
    __syncthreads();
    unsigned long long pos = 0;
    if (w >= 0) {
        unsigned long long rank = p.tile_cnt[size_t(blockIdx.x) * W + w] + pc;
        pos = p.tile_bytes[size_t(blockIdx.x) * W + w] + pb;
        for (int q = 0; q < warp; ++q) { rank += s_wc[q][w]; pos += s_wb[q][w]; }
        const size_t g = size_t(tr.chunk) * W + w;
        int64_t* go = p.goffs + p.goff_base[g];
        go[rank] = int64_t(pos);
        if (rank + 1 == p.group_tot[g * 2]) go[rank + 1] = int64_t(pos + (unsigned long long)len);
        p.map0[row] = take_pack(uint32_t(w), rank);
        if (PERM) p.inv[p.goff_base[g] + rank] = row;
        pos += p.gdata_off[g];
    } else if (row < tr.end) {
        p.map0[row] = kNoRow;
    }
    // the warp copies its messages one after another, 32 bytes a step
    for (int i = 0; i < 32; ++i) {
        const int wi = __shfl_sync(0xFFFFFFFFu, w, i);
        const long long li = __shfl_sync(0xFFFFFFFFu, len, i), ai = __shfl_sync(0xFFFFFFFFu, a, i);
        const unsigned long long di = __shfl_sync(0xFFFFFFFFu, pos, i);
        if (wi < 0) continue;
        const uint8_t* src = p.data + ai;
        uint8_t* dst = p.gdata + di;
        for (long long b = lane; b < li; b += 32) dst[b] = src[b];
    }
}

__global__ void __launch_bounds__(kTakeBlock) vp_scatter_kernel(const VersionsParams p) { vp_scatter_body<false>(p); }
__global__ void __launch_bounds__(kTakeBlock) vp_scatter_perm_kernel(const VersionsParams p) { vp_scatter_body<true>(p); }

__device__ __forceinline__ long long block_sum(long long v, long long* s_part) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
    if (lane == 0) s_part[warp] = v;
    __syncthreads();
    long long t = 0;
    for (int q = 0; q < kVpWarps; ++q) t += s_part[q];
    __syncthreads();
    return t;
}

// exclusive prefix of v over the block's threads
__device__ __forceinline__ long long block_excl(long long v, long long* s_part) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long incl = v;
    for (int d = 1; d < 32; d <<= 1) { const long long u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += u; }
    if (lane == 31) s_part[warp] = incl;
    __syncthreads();
    long long base = 0;
    for (int q = 0; q < warp; ++q) base += s_part[q];
    __syncthreads();
    return base + incl - v;
}

// PERM: a kNoRow entry is a null row (take_null_value, take_null_offsets_row).
template <bool PERM>
__device__ __forceinline__ void take_rows_body(const TakeSpace* spaces, const TakeJob* jobs) {
    __shared__ long long s_part[kVpWarps];
    const TakeSpace sp = spaces[blockIdx.y];
    if (int64_t(blockIdx.x) * kTakeBlock >= max(sp.rows, 1ll)) return;
    const int64_t r = int64_t(blockIdx.x) * kTakeBlock + threadIdx.x;
    const bool valid = r < sp.rows;
    const unsigned long long e = valid ? sp.map[r] : 0ull;
    const bool null_row = PERM && e == kNoRow;
    const uint32_t w = take_writer(e);
    const int64_t s = take_row(e);
    for (int q = sp.first_job; q < sp.first_job + sp.n_jobs; ++q) {
        const TakeJob jb = jobs[q];
        switch (SlotRole(jb.role)) {
            case SlotRole::Validity: case SlotRole::Bits: {
                const uint32_t word = __ballot_sync(0xFFFFFFFFu, valid && !null_row && take_bit(jb, w, s));
                if ((threadIdx.x & 31) == 0 && valid) reinterpret_cast<uint32_t*>(jb.dst)[r >> 5] = word;
                break;
            }
            case SlotRole::Offsets: {
                const long long t = block_sum(valid && !null_row ? take_len(jb, w, s) : 0, s_part);
                if (threadIdx.x == 0) jb.block_base[blockIdx.x] = t;
                break;
            }
            default:
                if (null_row) take_null_value(jb, r);
                else if (valid) take_value(jb, w, s, r);
        }
    }
}

__global__ void __launch_bounds__(kTakeBlock) take_rows_kernel(const TakeSpace* spaces, const TakeJob* jobs) { take_rows_body<false>(spaces, jobs); }
__global__ void __launch_bounds__(kTakeBlock) take_rows_perm_kernel(const TakeSpace* spaces, const TakeJob* jobs) { take_rows_body<true>(spaces, jobs); }

__global__ void __launch_bounds__(kTakeBlock) take_scan_kernel(const TakeScan* scans) {
    __shared__ long long s_part[kVpWarps];
    const TakeScan sc = scans[blockIdx.x];
    long long carry = 0;
    for (long long i0 = 0; i0 < sc.n; i0 += kTakeBlock) {
        const long long i = i0 + threadIdx.x;
        const long long v = i < sc.n ? sc.base[i] : 0;
        const long long ex = block_excl(v, s_part);
        if (i < sc.n) sc.base[i] = carry + ex;
        carry += block_sum(v, s_part);
    }
}

template <bool PERM>
__device__ __forceinline__ void take_offsets_body(const TakeSpace* spaces, const TakeJob* jobs) {
    __shared__ long long s_part[kVpWarps];
    const TakeSpace sp = spaces[blockIdx.y];
    if (int64_t(blockIdx.x) * kTakeBlock >= max(sp.rows, 1ll)) return;
    const int64_t r = int64_t(blockIdx.x) * kTakeBlock + threadIdx.x;
    const bool valid = r < sp.rows;
    const unsigned long long e = valid ? sp.map[r] : 0ull;
    const bool null_row = PERM && e == kNoRow;
    const uint32_t w = take_writer(e);
    const int64_t s = take_row(e);
    for (int q = sp.first_job; q < sp.first_job + sp.n_jobs; ++q) {
        const TakeJob jb = jobs[q];
        if (SlotRole(jb.role) != SlotRole::Offsets) continue;
        const int32_t len = valid && !null_row ? take_len(jb, w, s) : 0;
        const long long pos = jb.block_base[blockIdx.x] + block_excl(len, s_part);
        if (r == 0) reinterpret_cast<int32_t*>(jb.dst)[0] = 0;
        if (!valid) continue;
        if (null_row) { take_null_offsets_row(jb, r, int32_t(pos)); continue; }
        take_offsets_row(jb, w, s, r, int32_t(pos), len);
        if (jb.dst_data) take_copy(jb.dst_data + pos, jb.src_data[w] + take_start(jb, w, s), len);
    }
}

__global__ void __launch_bounds__(kTakeBlock) take_offsets_kernel(const TakeSpace* spaces, const TakeJob* jobs) { take_offsets_body<false>(spaces, jobs); }
__global__ void __launch_bounds__(kTakeBlock) take_offsets_perm_kernel(const TakeSpace* spaces, const TakeJob* jobs) {
    take_offsets_body<true>(spaces, jobs);
}

// list[0, n_part): the partition's (message << 8 | code); list[n_part, n): the sub-decodes' (index into inv << 8 | code),
// rewritten in place to (message << 8 | code).  An E_FRAME_ID message's first header_bytes bytes go to hdr[i * 16].
__global__ void __launch_bounds__(kTakeBlock) vp_report_kernel(unsigned long long* list, int64_t n_part, int64_t n, const int64_t* inv,
                                                               const uint8_t* data, const int64_t* offsets, int header_bytes, uint8_t* hdr) {
    const int64_t i = int64_t(blockIdx.x) * kTakeBlock + threadIdx.x;
    if (i >= n) return;
    unsigned long long e = list[i];
    if (i >= n_part) {
        e = (static_cast<unsigned long long>(inv[e >> 8]) << 8) | (e & 0xFF);
        list[i] = e;
    }
    if ((e & 0xFF) != E_FRAME_ID) return;
    const uint8_t* m = data + offsets[e >> 8];
    for (int b = 0; b < header_bytes; ++b) hdr[i * 16 + b] = m[b];
}

}  // namespace

void launch_versions_partition(const VersionsParams& p, bool single_object, bool permissive, cudaStream_t s) {
    const unsigned tiles = unsigned(p.n_tiles);
    if (permissive) {
        if (single_object) vp_count_perm_kernel<unsigned long long><<<tiles, kTakeBlock, 0, s>>>(p);
        else vp_count_perm_kernel<uint32_t><<<tiles, kTakeBlock, 0, s>>>(p);
    } else {
        if (single_object) vp_count_kernel<unsigned long long><<<tiles, kTakeBlock, 0, s>>>(p);
        else vp_count_kernel<uint32_t><<<tiles, kTakeBlock, 0, s>>>(p);
    }
    vp_scan_kernel<<<dim3(static_cast<unsigned>(p.k), static_cast<unsigned>(p.n_ids)), kTakeBlock, 0, s>>>(p);
}

void launch_versions_scatter(const VersionsParams& p, bool permissive, cudaStream_t s) {
    if (permissive) vp_scatter_perm_kernel<<<unsigned(p.n_tiles), kTakeBlock, 0, s>>>(p);
    else vp_scatter_kernel<<<unsigned(p.n_tiles), kTakeBlock, 0, s>>>(p);
}

void launch_take_level(const TakeSpace* spaces, int n_spaces, long long blocks, const TakeJob* jobs, const TakeScan* scans, int n_scans,
                       bool permissive, cudaStream_t s) {
    constexpr int kMaxY = 65535;  // gridDim.y
    for (int e = 0; e < n_spaces; e += kMaxY) {
        const dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(min(kMaxY, n_spaces - e)));
        if (permissive) take_rows_perm_kernel<<<grid, kTakeBlock, 0, s>>>(spaces + e, jobs);
        else take_rows_kernel<<<grid, kTakeBlock, 0, s>>>(spaces + e, jobs);
    }
    if (n_scans <= 0) return;
    take_scan_kernel<<<static_cast<unsigned>(n_scans), kTakeBlock, 0, s>>>(scans);
    for (int e = 0; e < n_spaces; e += kMaxY) {
        const dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(min(kMaxY, n_spaces - e)));
        if (permissive) take_offsets_perm_kernel<<<grid, kTakeBlock, 0, s>>>(spaces + e, jobs);
        else take_offsets_kernel<<<grid, kTakeBlock, 0, s>>>(spaces + e, jobs);
    }
}

void launch_versions_report(unsigned long long* list, int64_t n_part, int64_t n, const int64_t* inv, const uint8_t* data, const int64_t* offsets,
                            int header_bytes, uint8_t* hdr, cudaStream_t s) {
    if (n <= 0) return;
    vp_report_kernel<<<static_cast<unsigned>((n + kTakeBlock - 1) / kTakeBlock), kTakeBlock, 0, s>>>(list, n_part, n, inv, data, offsets, header_bytes, hdr);
}

}  // namespace rv
