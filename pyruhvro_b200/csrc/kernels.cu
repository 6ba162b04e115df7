// sm_90a kernels of the Avro -> Arrow direct decode (statically compiled part).
//
//   fused_kernel       the generic (interpreter) instance of the fused decode pass (dev_kernels.cuh): one CTA per
//                      256-record tile; TMA-staged window, COUNT walk, in-tile scan, decoupled look-back across
//                      tiles, EMIT walk, bulk-store write-out.  The schema-specialised instance (rvj_fused) is
//                      generated and compiled at run time by jit.cpp from the same body.
//   null_count_kernel  popcount of validity bitmaps (decides lazy validity export).
//   rebase / concat    fix-ups for gathering shard-local batches into one (multi-GPU).
//
// Integer/byte work bounded by HBM bandwidth; no tensor-core use.
#include "kernels.cuh"

#include <algorithm>

#include "dev_kernels.cuh"
#include "interp.cuh"
#include "ocf_walk.cuh"

namespace rv {
namespace {

__global__ void __launch_bounds__(kBlock) fused_kernel(const DecodeParams p) { fused_body<InterpWalker>(p, int(blockIdx.x)); }

// One bitmap per blockIdx.x, 16 parts per bitmap.  The bit count of bitmaps of deeper row spaces is only known on
// the device (the chunk's stream total in the control block), so jobs carry a pointer to it.
__global__ void null_count_kernel(const NullCountJob* jobs, long long* ones_out) {
    const NullCountJob job = jobs[blockIdx.x];
    const int64_t n_bits = job.n_bits_dev ? int64_t(*job.n_bits_dev) : job.n_bits;
    const int64_t n_words = (n_bits + 31) >> 5;
    long long ones = 0;
    for (int64_t w = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; w < n_words; w += int64_t(gridDim.y) * blockDim.x) {
        uint32_t v = __ldg(job.bitmap + w);
        const int64_t rem = n_bits - (w << 5);
        if (rem < 32) v &= (1u << rem) - 1u;
        ones += __popc(v);
    }
    for (int d = 16; d; d >>= 1) ones += __shfl_xor_sync(0xFFFFFFFFu, ones, d);
    __shared__ long long s_w[32];
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = ones;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long tot = 0;
        for (int i = 0; i < int(blockDim.x >> 5); ++i) tot += s_w[i];
        if (tot) atomicAdd(reinterpret_cast<unsigned long long*>(ones_out + blockIdx.x), static_cast<unsigned long long>(tot));
    }
}

// Packs the scattered slots of a capacity-planned arena into an exact-size one (device -> device), so that the
// device -> host copy that follows moves no slack: one CTA column per copy job, 16 bytes per thread and step.
__global__ void compact_kernel(const CompactJob* jobs) {
    const CompactJob job = jobs[blockIdx.x];
    const int64_t nvec = job.bytes >> 4;
    const uint4* s = reinterpret_cast<const uint4*>(job.src);
    uint4* d = reinterpret_cast<uint4*>(job.dst);
    for (int64_t i = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < nvec; i += int64_t(gridDim.y) * blockDim.x) d[i] = s[i];
    if (blockIdx.y == 0)
        for (int64_t i = (nvec << 4) + threadIdx.x; i < job.bytes; i += blockDim.x) job.dst[i] = job.src[i];
}

// ---- object container files: record offsets -------------------------------------------------------------------------
// One LANE per block walks the block's datums (ocf_walk.cuh).  Blocks are independent, so a file of thousands of blocks
// keeps the device busy; the decode kernel then runs on the offsets like on any packed input.
__global__ void ocf_offsets_kernel(const OcfParams q) {
    const int b = int(blockIdx.x * blockDim.x + threadIdx.x);
    if (b >= q.n_blocks) return;
    ocf_walk_block(q, b);
}

// ---- multi-GPU gather: every rank pushes its Arrow buffers into the gathered arena on the leader GPU ----------------
// One launch per rank, blockIdx.x = job, blockIdx.y = part of the job.  The destination is written in aligned 32-bit
// words, consecutive lanes -> consecutive words (whole 128-byte lines per warp store over NVLink); the fix-up of each
// buffer kind is fused into the copy:
//   RAW      bytes at any destination alignment: each destination word is cut out of two source words (funnel shift);
//   OFFSETS  dst[1 + i] = src[1 + i] + add   (Arrow offsets rebased by what the earlier ranks hold);
//   BITS     the bitmap shifted to its bit position; words that other ranks share are merged with atomic OR (the arena
//            starts zeroed), fully covered words are plain stores.
__global__ void gather_push_kernel(const PushJob* jobs) {
    const PushJob job = jobs[blockIdx.x];
    const int64_t tid = int64_t(blockIdx.y) * blockDim.x + threadIdx.x, nthr = int64_t(gridDim.y) * blockDim.x;
    if (job.kind == 1) {  // GK_OFFSETS
        const int32_t* s = reinterpret_cast<const int32_t*>(job.src);
        int32_t* d = reinterpret_cast<int32_t*>(job.dst);
        const int32_t add = int32_t(job.param);
        for (int64_t i = tid; i < job.count; i += nthr) d[1 + i] = s[1 + i] + add;
    } else if (job.kind == 2) {  // GK_BITS
        const uint32_t* src = reinterpret_cast<const uint32_t*>(job.src);
        uint32_t* dst = reinterpret_cast<uint32_t*>(job.dst);
        const int64_t nbits = job.count, dst_bit = job.param;
        const int64_t w0 = dst_bit >> 5, w1 = (dst_bit + nbits + 31) >> 5;
        const unsigned sh = unsigned(dst_bit & 31);
        const int64_t n_src_words = (nbits + 31) >> 5;
        for (int64_t w = w0 + tid; w < w1; w += nthr) {
            const int64_t k = w - w0;  // source word whose low bits land at bit `sh` of this word
            uint32_t lo = 0, hi = 0;
            if (k < n_src_words) {
                hi = src[k];
                const int64_t rem = nbits - (k << 5);
                if (rem < 32) hi &= (1u << rem) - 1u;
            }
            if (k >= 1 && sh) {
                lo = src[k - 1];
                const int64_t rem = nbits - ((k - 1) << 5);
                if (rem < 32) lo &= (1u << rem) - 1u;
            }
            const uint32_t v = sh ? ((hi << sh) | (lo >> (32u - sh))) : hi;
            const bool whole = (w << 5) >= dst_bit && ((w + 1) << 5) <= dst_bit + nbits;  // no other rank writes this word
            if (whole) dst[w] = v;
            else if (v) atomicOr(dst + w, v);
        }
    } else {  // GK_RAW
        const uintptr_t da = reinterpret_cast<uintptr_t>(job.dst);
        const int64_t to_word = int64_t((4u - unsigned(da & 3u)) & 3u);
        const int64_t head = job.count < to_word ? job.count : to_word;  // bytes up to the first aligned word
        const int64_t nwords = (job.count - head) >> 2;
        uint32_t* dw = reinterpret_cast<uint32_t*>(job.dst + head);
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(job.src + (head & ~int64_t(3)));  // (src is 64-byte aligned, head < 4: this is src)
        const unsigned sh = unsigned(head & 3) * 8u;
        for (int64_t i = tid; i < nwords; i += nthr) dw[i] = sh ? __funnelshift_r(sw[i], sw[i + 1], sh) : sw[i];
        if (blockIdx.y == 0) {
            if (int64_t(threadIdx.x) < head) job.dst[threadIdx.x] = job.src[threadIdx.x];
            const int64_t done = head + (nwords << 2);
            if (done + int64_t(threadIdx.x) < job.count) job.dst[done + threadIdx.x] = job.src[done + threadIdx.x];
        }
    }
}

// ---- fix-ups for gathering shard-local Arrow buffers into one batch (multi-GPU, SURVEY.md 8(e)) ----
// dst[i] = src[i] + add: rebases a shard's i32 offsets by the total of the shards before it.
__global__ void rebase_i32_kernel(int32_t* dst, const int32_t* src, long long n, int32_t add) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] + add;
}

// ORs `nbits` bits of `src` (bit 0 first) into `dst` starting at bit `dst_bit`; dst must be zero where
// nothing was written yet.  One thread per destination word; seam words are shared between shards, hence atomicOr.
__global__ void concat_bits_kernel(uint32_t* dst, long long dst_bit, const uint32_t* src, long long nbits) {
    const long long w0 = dst_bit >> 5, w1 = (dst_bit + nbits + 31) >> 5;
    const unsigned sh = unsigned(dst_bit & 31);
    const long long n_src_words = (nbits + 31) >> 5;
    for (long long w = w0 + blockIdx.x * (long long)blockDim.x + threadIdx.x; w < w1; w += (long long)gridDim.x * blockDim.x) {
        const long long k = w - w0;  // source word whose low bits land at bit `sh` of this word
        uint32_t lo = 0, hi = 0;
        if (k < n_src_words) {
            hi = src[k];
            const long long rem = nbits - (k << 5);
            if (rem < 32) hi &= (1u << rem) - 1u;
        }
        if (k >= 1 && sh) {
            lo = src[k - 1];
            const long long rem = nbits - ((k - 1) << 5);
            if (rem < 32) lo &= (1u << rem) - 1u;
        }
        const uint32_t v = sh ? ((hi << sh) | (lo >> (32u - sh))) : hi;
        if (v) atomicOr(dst + w, v);
    }
}

}  // namespace

void launch_rebase_i32(int32_t* dst, const int32_t* src, long long n, int32_t add, cudaStream_t s) {
    if (n <= 0) return;
    const int blocks = int(std::min<long long>((n + 255) / 256, 132 * 8));
    rebase_i32_kernel<<<blocks, 256, 0, s>>>(dst, src, n, add);
}

void launch_concat_bits(uint32_t* dst, long long dst_bit, const uint32_t* src, long long nbits, cudaStream_t s) {
    if (nbits <= 0) return;
    const long long words = ((dst_bit + nbits + 31) >> 5) - (dst_bit >> 5);
    const int blocks = int(std::min<long long>((words + 255) / 256, 132 * 8));
    concat_bits_kernel<<<blocks, 256, 0, s>>>(dst, dst_bit, src, nbits);
}

cudaError_t prepare_kernels() {
    cudaError_t e = cudaFuncSetAttribute(fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fused_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (e == cudaSuccess) e = prepare_kernels_permissive();
    return e;
}

void launch_fused(const DecodeParams& p, size_t smem, cudaStream_t s, bool permissive) {
    if (permissive) launch_fused_permissive(p, smem, s);
    else fused_kernel<<<unsigned(p.n_tiles), kBlock, smem, s>>>(p);
}

void launch_null_count(const NullCountJob* jobs, int n_jobs, long long* out, cudaStream_t s) {
    if (n_jobs <= 0) return;
    null_count_kernel<<<dim3(n_jobs, 16), 256, 0, s>>>(jobs, out);
}

void launch_ocf_offsets(const OcfParams& q, cudaStream_t s) {
    if (q.n_blocks <= 0) return;
    ocf_offsets_kernel<<<unsigned((q.n_blocks + 63) / 64), 64, 0, s>>>(q);
}

void launch_gather_push(const PushJob* jobs, int n_jobs, int parts, cudaStream_t s) {
    if (n_jobs <= 0) return;
    gather_push_kernel<<<dim3(n_jobs, parts), 256, 0, s>>>(jobs);
}

void launch_compact(const CompactJob* jobs, int n_jobs, int parts, cudaStream_t s) {
    if (n_jobs <= 0) return;
    compact_kernel<<<dim3(n_jobs, parts), 256, 0, s>>>(jobs);
}

}  // namespace rv
