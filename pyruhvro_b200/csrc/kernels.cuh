// Launch wrappers of the statically compiled kernels (sm_90a).  See kernels.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "dev_types.h"
#include "take.cuh"

namespace rv {

struct NullCountJob {
    const uint32_t* bitmap;
    int64_t n_bits;                            // used when n_bits_dev is null
    const unsigned long long* n_bits_dev;      // device word holding the bit count (rows of a deeper row space)
};

struct CompactJob {
    const uint8_t* src;
    uint8_t* dst;      // both 16-byte aligned
    int64_t bytes;
};

// One push of the multi-GPU gather (gather.hpp): `dst` may be peer memory (NVLink).
struct PushJob {
    const uint8_t* src;   // this rank's buffer (64-byte aligned)
    uint8_t* dst;         // where it lands in the gathered arena (RAW: any alignment; OFFSETS: element `row_base`; BITS: the bitmap's first word)
    int64_t count;        // RAW: bytes; OFFSETS: rows; BITS: bits
    int64_t param;        // OFFSETS: add; BITS: destination bit
    int32_t kind;         // GatherKind
    int32_t pad;
};

cudaError_t prepare_kernels();  // opt in to large dynamic shared memory (once per device)

void launch_fused(const DecodeParams& p, size_t smem, cudaStream_t s, bool permissive = false);  // interpreter walker, one CTA per tile
// the permissive instance (kernels_perm.cu, a translation unit of its own so that the two compile side by side)
cudaError_t prepare_kernels_permissive();
void launch_fused_permissive(const DecodeParams& p, size_t smem, cudaStream_t s);
void launch_rebase_i32(int32_t* dst, const int32_t* src, long long n, int32_t add, cudaStream_t s);
void launch_concat_bits(uint32_t* dst, long long dst_bit, const uint32_t* src, long long nbits, cudaStream_t s);
void launch_null_count(const NullCountJob* jobs, int n_jobs, long long* out, cudaStream_t s);
void launch_compact(const CompactJob* jobs, int n_jobs, int parts, cudaStream_t s);
void launch_ocf_offsets(const OcfParams& q, cudaStream_t s);
void launch_gather_push(const PushJob* jobs, int n_jobs, int parts, cudaStream_t s);
// multi-version Confluent decode (versions.cu): count + scan of the partition, then (after the host placed the groups)
// the scatter; one level of row spaces of the take
// keys: p.ids, or p.fps; permissive: the *_perm instances (a bad group per chunk, a null row per kNoRow entry)
void launch_versions_partition(const VersionsParams& p, bool single_object, bool permissive, cudaStream_t s);
void launch_versions_scatter(const VersionsParams& p, bool permissive, cudaStream_t s);
void launch_take_level(const TakeSpace* spaces, int n_spaces, long long blocks, const TakeJob* jobs, const TakeScan* scans, int n_scans,
                       bool permissive, cudaStream_t s);
// permissive registries: the call's bad list in message terms, and the headers of its E_FRAME_ID messages (16 bytes each)
void launch_versions_report(unsigned long long* list, int64_t n_part, int64_t n, const int64_t* inv, const uint8_t* data, const int64_t* offsets,
                            int header_bytes, uint8_t* hdr, cudaStream_t s);

}  // namespace rv
