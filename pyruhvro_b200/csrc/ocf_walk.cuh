// Object container files: the record offsets of one block (ocf.hpp).  The body of ocf_offsets_kernel (kernels.cu), one
// lane per block; the host emulation (tests/emu) runs the same function for every block, so the CPU suite checks the walk
// the device runs.
#pragma once
#include "interp.cuh"

namespace rv {

// *err = min(*err, v): atomic on the device, where the lanes of all blocks share the word.
RV_HD void ocf_err_min(unsigned long long* err, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    atomicMin(err, v);
#else
    if (v < *err) *err = v;
#endif
}

// The datums of a block carry no lengths, so the lane walks them one after the other with the precise COUNT walk (full
// validation) straight from global memory and notes where each one starts.  A failing record reports (record << 8 | code)
// and ends the block's walk; a block whose records end before its size reports E_FRAME at its last record.  The bytes
// between blocks (count, size, sync marker) trail a block's last record and are ignored like any trailing bytes
// (fast_decode.rs:825-828).
RV_HD void ocf_walk_block(const OcfParams& q, int b) {
    const OcfBlockDev blk = q.blocks[b];
    uint32_t cur[kMaxStreams];  // the walk's per-stream counters (unused here): local memory
    long long pos = blk.data_off;
    const long long end = blk.data_off + blk.size;
    for (long long i = 0; i < blk.count; ++i) {
        q.offsets[blk.rec_base + i] = pos;
        // every record's counters start at zero: they are overflow-checked, and Arrow's i32 limit is per output batch,
        // not per block (the decode pass checks the batches)
        for (int s = 0; s < q.n_streams; ++s) cur[s] = 0;
        WalkCtx<false> c;
        c.nodes = q.nodes;
        c.cur = cur;
        c.cur_stride = 1;
        c.sym_off = q.sym_off;
        c.sym_bytes = q.sym_bytes;
        c.bufs = nullptr;
        c.ptrs_saddr = 0;
        c.err = 0;
        c.stage_on = false;
        c.in_range = true;
        c.row0 = 0;
        c.store_word = false;
        c.base = q.data + pos;
        c.pos = 0;
        const long long left = end - pos;
        c.end = uint32_t(left > 0xFFFFFFF0ll ? 0xFFFFFFF0ll : left);
        InterpWalker::Cur none;
        InterpWalker::walk<WM_COUNT>(c, q.n_nodes, none);
        if (c.err) { ocf_err_min(q.err, (static_cast<unsigned long long>(blk.rec_base + i) << 8) | c.err); return; }
        pos += c.pos;
    }
    if (pos != end) ocf_err_min(q.err, (static_cast<unsigned long long>(blk.rec_base + (blk.count ? blk.count - 1 : 0)) << 8) | E_FRAME);  // the block's size disagrees with its records
    if (b == q.n_blocks - 1) q.offsets[q.n_records] = q.end_off;
}

}  // namespace rv
