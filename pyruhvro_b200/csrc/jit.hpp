// Plan compiler: turns a decode plan into a schema-specialised walker (CUDA C++ source built from
// the hand-written ops of dev_core.cuh), compiles it with NVRTC for sm_90a and caches the cubin.
//
// Why: the generic interpreter spends ~30 instructions per input byte on dispatch (DNode fetch,
// presence masks, a 12-way switch) and both kernels are issue-bound.  The generated
// walker is straight-line code per field with every slot / stream / flag a literal; it is the GPU
// analogue of the reference inlining its Nullable* variants to avoid "Box indirection + double
// match dispatch" (ruhvro/src/fast_decode.rs:69-72).  The interpreter remains the generic path
// when NVRTC is unavailable (RV_JIT=0 forces it).
#pragma once
#include <string>
#include <vector>

#include "plan.hpp"

namespace rv {

// Source of `struct rv::gen::Walker` (includes only dev_core.cuh; also compiled for the host by tests/emu), for tiles of
// `tile` records: the walker's item table (kItemBytes) is sized for them.
std::string generate_walker_source(const Plan& plan, int tile = kBlock);

// Lists/maps whose items the generated walker emits item-parallel (one item per lane): those of the top-level
// record whose items are walked.  Their item positions take item_table_bytes(n) of the CTA's shared memory.
int item_parallel_lists(const Plan& plan);

// Full NVRTC translation unit: walker + the `rvj_fused` kernel, for tiles of `tile` records (kBlock or kWideTile).
std::string generate_kernel_source(const Plan& plan, int tile);

// Compiles (or fetches from the on-disk cache) the cubin for `arch` (e.g. "sm_90a").
// Needs no GPU.  Returns false and fills `log` when NVRTC cannot be loaded or compilation fails.
// ignore_cache: recompile even if the on-disk cache holds an entry (it is replaced).
bool jit_cubin(const std::string& source, const std::string& arch, std::vector<char>* cubin, std::string* log, bool ignore_cache = false);

}  // namespace rv
