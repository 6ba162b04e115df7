// Device core of the record walk: byte access, wire primitives and per-type decode ops.
//
// These are the hand-written building blocks of BOTH walkers:
//   * interp.cuh        — the generic lock-step interpreter over DNodes (statically compiled);
//   * generated walkers — straight-line code emitted per schema by jit.cpp and compiled with
//                         NVRTC for sm_90a (same ops, constants folded, no dispatch).
// Each op restates one arm of the reference's FieldDecoder::decode / append_null
// (ruhvro/src/fast_decode.rs:420-534) for a lane that either consumes bytes (`valid`) or appends
// the null slot.  MODE: WM_COUNT accumulates per-stream contributions into cur[stream];
// WM_EMIT writes Arrow buffers at the cursors the scans produced.
//
// Two contexts, two flavours of every primitive:
//   * WalkCtx<true>  FAST.  The record lies in the CTA's shared-memory window.  The readers are written for the
//     encodings every Avro writer produces (one-byte branch / union / enum indices, one- or two-byte varints with a
//     rolled loop behind them, non-negative block counts) and do no per-byte bounds checks: end-of-buffer is
//     checked where a length is applied, once per list item and at a few points of the straight line (eof_check),
//     which bounds how far a reader can run past the record (kWindowPad).  Anything else — non-canonical or
//     over-long varints, negative lengths / block counts, bad booleans, indices out of range, running past the
//     end — only raises c.err ("not plain": no category, no recovery).  The kernel then repeats that record with
//     the PRECISE flavour, which decides whether it is an error and which one.
//   * WalkCtx<false> PRECISE.  Reads the record where the caller put it (global memory / host memory) byte by byte
//     with the reference's checks in the reference's order, so the first error of a record and its category are
//     the reference's (fast_decode.rs:845-922).
//
// Compiles for: nvcc (device), NVRTC (device), g++ (tests/emu host emulation of both flavours; test infra only).
#pragma once
#include "dev_types.h"

#if defined(__CUDACC__)
#define RV_HD __host__ __device__ __forceinline__
#else
#define RV_HD inline
#endif

#if defined(__CUDACC__)
extern __shared__ __align__(16) uint8_t rv_smem[];  // the CTA's dynamic shared memory (all regions)
#endif

namespace rv {

enum WalkMode : int { WM_COUNT = 0, WM_EMIT = 1 };

// ---- shared-memory access by 32-bit shared-space address --------------------------------------------------
// (indexing rv_smem through generic pointers makes the compiler rebuild the shared-window base — S2R + LEA —
// next to most loads; a plain 32-bit address register + immediate offset is what the LSU wants)
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) { uint32_t v; asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t v; asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint64_t lds_u64(uint32_t a) { uint64_t v; asm("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void reds_or_u32(uint32_t a, uint32_t v) { asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t lds_u8v(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts_u8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
#endif

// ---- warp collectives of the item-parallel list emit (generated walkers) ----------------------------------------
// On the host, the item-parallel emit runs only under a lock-step warp emulation (tests/emu/warp_emu.cpp) that installs
// itself here: it holds the item-position table and runs the 32 lanes of a warp as coroutines that meet at every
// collective, where each lane hands in one value and gets the whole warp's 32.  Without it (the per-lane host emulation)
// the generated walkers keep their per-lane item loops.
#if !defined(__CUDA_ARCH__)
struct HostWarpEmu {
    uint8_t* items;                                       // the tile's item-position table
    const uint32_t* (*exchange)(uint32_t lane, uint32_t v);
};
// (internal linkage: an inline function's static would be one object across every emulation library in the process)
static inline HostWarpEmu*& host_warp_emu() { static HostWarpEmu* e = nullptr; return e; }
#endif
// Whether the item-parallel emit (and the count walk's item positions) are in use: always on the device.
RV_HD bool item_parallel_on() {
#if defined(__CUDA_ARCH__)
    return true;
#else
    return host_warp_emu() != nullptr;
#endif
}
RV_HD uint32_t warp_shfl(uint32_t v, uint32_t src, uint32_t lane) {
#if defined(__CUDA_ARCH__)
    (void)lane;
    return __shfl_sync(0xFFFFFFFFu, v, int(src));
#else
    return host_warp_emu()->exchange(lane, v)[src];
#endif
}
RV_HD bool warp_any(bool pred, uint32_t lane) {
#if defined(__CUDA_ARCH__)
    (void)lane;
    return __any_sync(0xFFFFFFFFu, pred);
#else
    const uint32_t* a = host_warp_emu()->exchange(lane, pred ? 1u : 0u);
    for (int i = 0; i < 32; ++i) if (a[i]) return true;
    return false;
#endif
}
// inclusive prefix sum over the warp's lanes
RV_HD uint32_t warp_scan_incl(uint32_t v, uint32_t lane) {
#if defined(__CUDA_ARCH__)
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (int(lane) >= d) v += u;
    }
    return v;
#else
    const uint32_t* a = host_warp_emu()->exchange(lane, v);
    uint32_t s = 0;
    for (uint32_t i = 0; i <= lane; ++i) s += a[i];
    return s;
#endif
}

// SM = the record's bytes were staged into shared memory (device) — the FAST flavour.
template <bool SM>
struct WalkCtx {
    static constexpr bool kShared = SM;
    const uint8_t* base;   // precise: global / host window holding this record.  fast on the host (emulation): the window
    uint32_t sbase;        // fast (device): shared-space address of the staged window's first byte
    uint32_t pos, end;     // cursor / record end, relative to the window
    uint32_t err;          // precise: first error of this record.  fast: != 0 "not plain", repeat with the precise flavour
    uint32_t pm;           // interpreter: presence by tree level
    uint64_t usel;         // interpreter: selected variant per union nesting level (8 bits each)
    const DNode* nodes;    // interpreter: the plan
    uint32_t* cur;         // interpreter: per-lane cursors, cur[stream * cur_stride]
    uint32_t cur_stride;   //   (generated walkers keep their cursors in registers)
    void* const* bufs;     // slot -> buffer of this chunk (global memory table)
    uint32_t ptrs_saddr;   // device emit: shared-space address of the CTA's copy of that table (0: none)
    const int32_t* sym_off;
    const uint8_t* sym_bytes;
    bool stage_on;         // precise (device emit): Utf8 bytes go to the shared-memory staging area like the fast lanes'
    uint32_t stage_saddr;  // shared-space address of the Utf8 staging area
    uint32_t adj_saddr;    // shared-space address of adj[stream]: staging offset of the stream's region minus the tile base
    uint32_t row0;         // chunk-local row of this record
    bool in_range;         // the lane owns a record
    bool store_word;       // space-0 bitmaps: this lane stores the warp's ballot word
    uint32_t items_saddr;  // fast (device): shared-space address of the item-position table (dev_types.h kItemSlots)
};

// Entry `i` of the item-position table, written by the FAST count walk and read by the item-parallel emit.
template <class C>
RV_HD void itab_put(C& c, uint32_t i, uint32_t v) {
#if defined(__CUDA_ARCH__)
    sts_u8(c.items_saddr + i, v);
#else
    host_warp_emu()->items[i] = uint8_t(v);
#endif
}
template <class C>
RV_HD uint32_t itab_get(const C& c, uint32_t i) {
#if defined(__CUDA_ARCH__)
    return lds_u8v(c.items_saddr + i);
#else
    (void)c;
    return host_warp_emu()->items[i];
#endif
}

// PRECISE: records the first error of the record and parks the cursor at the record's end, so every later
// read of this lane fails on its own (EOF) without the walkers re-checking c.err at each node.
// FAST: only notes that the record is not plain.
template <class C>
RV_HD void fail(C& c, uint32_t code) {
    if (C::kShared) { c.err |= code; return; }
    if (!c.err) c.err = code;
    c.pos = c.end;
}

template <class C>
RV_HD uint32_t ld_u8(const C& c, uint32_t pos) {
#if defined(__CUDA_ARCH__)
    if (C::kShared) return lds_u8(c.sbase + pos);
#endif
    return c.base[pos];
}

// Arrow buffer of `slot`.  The emit CTAs keep this chunk's pointer table in shared memory: a record walk
// dereferences ~30 of them and a global (L1) load each time is a long-scoreboard stall on the lane's
// critical path.
template <class C>
RV_HD void* buf_ptr(const C& c, int slot) {
#if defined(__CUDA_ARCH__)
    if (c.ptrs_saddr) return reinterpret_cast<void*>(lds_u64(c.ptrs_saddr + uint32_t(slot) * 8u));
#endif
    return c.bufs[slot];
}

RV_HD int64_t zz32(uint32_t r) { return int64_t(int32_t((r >> 1) ^ (0u - (r & 1u)))); }
RV_HD int64_t zz64(uint64_t r) { return int64_t(r >> 1) ^ -int64_t(r & 1); }

// FAST: deferred end-of-buffer check.  The walkers place one wherever a straight line of readers could otherwise
// have consumed more than kWindowPad bytes unchecked, and one at the end of the record.
template <int MODE, class C>
RV_HD void eof_check(C& c) {
    if (C::kShared && MODE == WM_COUNT) {
        if (c.pos > c.end) { c.err |= E_EOF; c.pos = c.end; }
    }
}

// The 7-bit groups of four varint bytes (continuation bits already dropped by the caller's mask) packed into 28 bits.
RV_HD uint32_t pack7x4(uint32_t w) {
    return (w & 0x7Fu) | ((w & 0x7F00u) >> 1) | ((w & 0x7F0000u) >> 2) | ((w & 0x7F000000u) >> 3);
}

// Bytes 3.. of a varint whose first two bytes both had the continuation bit.  FAST flavour on the device: the (at most
// eight) remaining bytes are taken as ONE 64-bit window — three aligned shared loads — the terminating byte is found
// with a bit scan and the 7-bit groups are packed without a loop; a byte-at-a-time loop cost ~12 instructions per byte
// with 64-bit shifts (random longs: ~100 per value).  Elsewhere (precise flavour, host): the reference's loop.
template <bool CHECK, class C>
RV_HD uint64_t varint_tail(C& c, uint64_t r) {
#if defined(__CUDA_ARCH__)
    if (C::kShared) {
        const uint32_t a = c.sbase + c.pos, al = a & ~3u, sh = (a & 3u) * 8u;
        const uint32_t w0 = lds_u32(al), w1 = lds_u32(al + 4u);
        uint32_t lo = __funnelshift_r(w0, w1, sh);
        const uint32_t t_lo = ~lo & 0x80808080u;                          // bytes whose continuation bit is clear
        if (t_lo) {                                                       // ends within four more bytes (values below 2^42)
            const uint32_t n = uint32_t(__ffs(int(t_lo))) >> 3;
            c.pos += n;
            lo &= 0xFFFFFFFFu >> (32u - 8u * n);
            return r | (uint64_t(pack7x4(lo & 0x7F7F7F7Fu)) << 14);
        }
        uint32_t hi = __funnelshift_r(w1, lds_u32(al + 8u), sh);
        const uint32_t t_hi = ~hi & 0x80808080u;
        uint32_t n = 8u;
        if (t_hi) { n = 4u + (uint32_t(__ffs(int(t_hi))) >> 3); hi &= 0xFFFFFFFFu >> (64u - 8u * n); }
        else if (CHECK) c.err |= E_VARINT;                                // an 11th byte would follow: too long
        c.pos += n;
        const uint64_t v56 = uint64_t(pack7x4(lo & 0x7F7F7F7Fu)) | (uint64_t(pack7x4(hi & 0x7F7F7F7Fu)) << 28);
        return r | (v56 << 14);   // (bits beyond 64 fall off, as in the reference's `<< shift`)
    }
#endif
    uint32_t shift = 14;
    for (;;) {
        const uint32_t b = ld_u8(c, c.pos++);
        r |= uint64_t(b & 0x7Fu) << shift;
        if (!(b & 0x80u)) break;
        shift += 7;
        if (shift >= 70) { if (CHECK) c.err |= E_VARINT; break; }  // (emit: unreachable on validated input; bounds the loop regardless)
    }
    return r;
}

// read_zigzag_long (fast_decode.rs:854-869).
//
// CHECK = false is used by the EMIT walk only: it runs after the count walk went over the very same bytes
// with CHECK = true (and the tile was abandoned on any error), so bounds / range checks would only re-prove
// what is known.  (Inputs are borrowed for the duration of the call and must not be mutated meanwhile.)
template <bool CHECK = true, class C>
RV_HD int64_t rd_varint(C& c) {
    if (C::kShared) {  // FAST: one / two bytes inline, no bounds checks (see eof_check)
        const uint32_t b0 = ld_u8(c, c.pos);
        if (b0 < 0x80u) { c.pos += 1; return zz32(b0); }
        const uint32_t b1 = ld_u8(c, c.pos + 1);
        c.pos += 2;
        const uint32_t lo = (b0 & 0x7Fu) | ((b1 & 0x7Fu) << 7);
        if (b1 < 0x80u) return zz32(lo);
        return zz64(varint_tail<CHECK>(c, lo));
    }
    if (!CHECK || c.pos < c.end) {
        const uint32_t b = ld_u8(c, c.pos);
        if (b < 0x80u) { c.pos += 1; return zz32(b); }
    }
    uint64_t r = 0;
    uint32_t shift = 0;
    for (;;) {
        if (CHECK && c.pos >= c.end) { fail(c, E_EOF); return 0; }
        const uint32_t b = ld_u8(c, c.pos++);
        r |= uint64_t(b & 0x7Fu) << shift;
        if (!(b & 0x80u)) break;
        shift += 7;
        if (CHECK && shift >= 64) { fail(c, E_VARINT); return 0; }
        if (!CHECK && shift >= 70) break;  // unreachable on validated input; bounds the loop regardless
    }
    return zz64(r);
}

// FAST only: a varint the schema expects to be a small non-negative number in ONE byte (union / enum index).
// Anything else (continuation bit, negative) is "not plain".
template <bool CHECK, class C>
RV_HD uint32_t rd_small(C& c) {
    const uint32_t b = ld_u8(c, c.pos);
    c.pos += 1;
    if (CHECK) c.err |= b & 0x81u;
    return b >> 1;
}

// Length prefix of a string (read_string, fast_decode.rs:902-911): false on error.
template <bool CHECK = true, class C>
RV_HD bool rd_len(C& c, uint32_t& len) {
    if (C::kShared) {  // FAST
        const uint32_t b0 = ld_u8(c, c.pos);
        uint32_t z;
        if (b0 < 0x80u) { c.pos += 1; z = b0; }
        else {
            const uint32_t b1 = ld_u8(c, c.pos + 1);
            c.pos += 2;
            z = (b0 & 0x7Fu) | ((b1 & 0x7Fu) << 7);
            if (b1 >= 0x80u) {
                const uint64_t r = varint_tail<CHECK>(c, z);
                if (CHECK && r > 0xFFFFFFFFull) { c.err |= E_EOF; len = 0; return true; }
                z = uint32_t(r);
            }
        }
        len = z >> 1;
        // negative, or longer than what is left of the record (pos may already be past the end; len < 2^31)
        // (32-bit sum: pos stays within the window + pad, far below 2^31)
        if (CHECK && ((z & 1u) || c.pos + len > c.end)) { c.err |= E_EOF; len = 0; }
        return true;
    }
    bool have = false;
    if (!CHECK || c.pos < c.end) {
        const uint32_t b = ld_u8(c, c.pos);
        if (b < 0x80u) {  // one byte: zigzag(len) < 128, odd = negative
            c.pos += 1;
            if (CHECK && (b & 1u)) { fail(c, E_NEG_LEN); return false; }
            len = b >> 1;
            have = true;
        }
    }
    if (!have) {
        const int64_t l = rd_varint<CHECK>(c);
        if (CHECK) {
            if (c.err) return false;
            if (l < 0) { fail(c, E_NEG_LEN); return false; }
            if (l > int64_t(0xFFFFFFFFu)) { fail(c, E_EOF); return false; }
        }
        len = uint32_t(l);
    }
    if (CHECK && len > c.end - c.pos) { fail(c, E_EOF); return false; }
    return true;
}

// union_branch (fast_decode.rs:585-593): true = Value, false = Null (or error).
template <bool CHECK = true, class C>
RV_HD bool rd_branch(C& c, bool null_first) {
    if (C::kShared) {  // FAST: the canonical one-byte encodings of branch 0 / 1
        const uint32_t b = ld_u8(c, c.pos);
        c.pos += 1;
        if (CHECK) c.err |= b & 0xFDu;
        return (b == 2u) == null_first;
    }
    if (!CHECK || c.pos < c.end) {
        const uint32_t b = ld_u8(c, c.pos);
        if (b == 0u || b == 2u) {  // canonical one-byte encodings of branch 0 / 1
            c.pos += 1;
            return (b == 2u) == null_first;
        }
    }
    const int64_t idx = rd_varint<CHECK>(c);
    if (CHECK && c.err) return false;
    if (!CHECK || idx == 0 || idx == 1) return (idx == 1) == null_first;
    fail(c, E_BRANCH);
    return false;
}

// Bit `row` of a validity / boolean buffer.  Space 0: rows are lane-aligned, so the warp ballots
// and one lane stores a whole 32-bit word.  Deeper spaces: rows are lane-private cursors, so set
// bits go through atomicOr into a zero-initialised buffer.
template <int D, class C>
RV_HD void put_bit(C& c, int slot, uint32_t row, bool bit) {
#if defined(RV_ABL_NOBITS)
    return;
#endif
#if defined(__CUDA_ARCH__)
    if (D == 0) {
        const unsigned w = __ballot_sync(0xFFFFFFFFu, bit);
        if (c.store_word) static_cast<uint32_t*>(buf_ptr(c, slot))[row >> 5] = w;
    } else {
        if (bit) atomicOr(static_cast<unsigned int*>(buf_ptr(c, slot)) + (row >> 5), 1u << (row & 31));
    }
#else
    if (bit && (D > 0 || c.in_range)) static_cast<uint8_t*>(buf_ptr(c, slot))[row >> 3] |= uint8_t(1u << (row & 7));
#endif
}

template <int D, class C>
RV_HD bool may_store(const C& c) {
#if defined(RV_ABL_NOSTORE)
    return false;
#else
    return (D > 0) || c.in_range;
#endif
}

// 4 / 8 raw little-endian bytes at the cursor (EMIT).  FAST: two / three aligned words + funnel shifts instead of a
// byte at a time.
template <class C>
RV_HD uint32_t ld_le32(const C& c, uint32_t p) {
#if defined(__CUDA_ARCH__)
    if (C::kShared) {
        const uint32_t a = c.sbase + p;
        return __funnelshift_r(lds_u32(a & ~3u), lds_u32((a & ~3u) + 4u), (a & 3u) * 8u);
    }
#endif
    return ld_u8(c, p) | (ld_u8(c, p + 1) << 8) | (ld_u8(c, p + 2) << 16) | (ld_u8(c, p + 3) << 24);
}
template <class C>
RV_HD uint64_t ld_le64(const C& c, uint32_t p) {
#if defined(__CUDA_ARCH__)
    if (C::kShared) {
        const uint32_t a = c.sbase + p, al = a & ~3u, sh = (a & 3u) * 8u;
        const uint32_t w0 = lds_u32(al), w1 = lds_u32(al + 4u), w2 = lds_u32(al + 8u);
        return uint64_t(__funnelshift_r(w0, w1, sh)) | (uint64_t(__funnelshift_r(w1, w2, sh)) << 32);
    }
#endif
    return uint64_t(ld_le32(c, p)) | (uint64_t(ld_le32(c, p + 4)) << 32);
}

// ---- fixed-width leaves -------------------------------------------------------------------
template <int MODE, int D, class C>
RV_HD void op_i32(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {
    int32_t v = 0;
    if (valid) {
        const int64_t x = rd_varint<MODE == WM_COUNT>(c);
        if (C::kShared || MODE == WM_EMIT || !c.err) v = int32_t(x); else valid = false;
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) static_cast<int32_t*>(buf_ptr(c, slot_a))[row] = v;
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

template <int MODE, int D, class C>
RV_HD void op_i64(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {
    int64_t v = 0;
    if (valid) {
        const int64_t x = rd_varint<MODE == WM_COUNT>(c);
        if (C::kShared || MODE == WM_EMIT || !c.err) v = x; else valid = false;
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) static_cast<int64_t*>(buf_ptr(c, slot_a))[row] = v;
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

template <int MODE, int D, class C>
RV_HD void op_f32(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {  // read_f32 :871-879
    uint32_t v = 0;
    if (valid) {
        if (!C::kShared && MODE == WM_COUNT && c.end - c.pos < 4u) { fail(c, E_EOF); valid = false; }
        else {
            if (MODE == WM_EMIT) v = ld_le32(c, c.pos);
            c.pos += 4;
        }
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) static_cast<uint32_t*>(buf_ptr(c, slot_a))[row] = v;
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

template <int MODE, int D, class C>
RV_HD void op_f64(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {  // read_f64 :881-891
    uint64_t v = 0;
    if (valid) {
        if (!C::kShared && MODE == WM_COUNT && c.end - c.pos < 8u) { fail(c, E_EOF); valid = false; }
        else {
            if (MODE == WM_EMIT) v = ld_le64(c, c.pos);
            c.pos += 8;
        }
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) static_cast<uint64_t*>(buf_ptr(c, slot_a))[row] = v;
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

template <int MODE, int D, class C>
RV_HD void op_bool(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {  // read_bool :893-900
    bool v = false;
    if (valid) {
        if (!C::kShared && MODE == WM_COUNT && c.pos >= c.end) { fail(c, E_EOF); valid = false; }
        else {
            const uint32_t b = ld_u8(c, c.pos++);
            if (MODE == WM_COUNT && b > 1u) { fail(c, E_BOOL); if (!C::kShared) valid = false; } else v = b != 0u;
        }
    }
    if (MODE == WM_EMIT) {
        put_bit<D>(c, slot_a, row, v);
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

#if defined(__CUDA_ARCH__)
// shared -> shared copy of `len` (> 0) bytes between two shared-space addresses.  Destination word j takes 4 source
// bytes at an arbitrary alignment: two aligned source words + a funnel shift.  The first and last words are
// shared with the neighbouring strings (written by other lanes), so they are merged with an atomic OR into the
// zero-initialised staging area; interior words are plain stores.  Source reads may touch up to 3 bytes
// before / 4 bytes after the string: still inside the CTA's shared memory.
// The warp's cost is its longest string, and a word-at-a-time loop makes every word wait for its own load.  So the
// last word's loads are issued next to the first word's, and the interior words go four per trip with all of a trip's
// loads issued together.  A string of up to 6 destination words (most real strings) then
// waits for three rounds of loads at most.  The loop stays rolled because a generated walker has a dozen call sites.
__device__ __forceinline__ void copy_smem_words(const uint32_t d, const uint32_t src, const uint32_t len) {
    const uint32_t a = d & 3u;
    const uint32_t nwords = (a + len + 3u) >> 2;
    const uint32_t sp = src - a;  // source byte that lands in byte 0 of destination word 0
    const uint32_t sh = (sp & 3u) * 8u;
    const uint32_t sw = sp & ~3u;
    const uint32_t dw = d & ~3u;
    const uint32_t m_first = 0xFFFFFFFFu << (a * 8u);
    const uint32_t e = (a + len) & 3u;
    const uint32_t m_last = e ? (0xFFFFFFFFu >> ((4u - e) * 8u)) : 0xFFFFFFFFu;
    const uint32_t v = __funnelshift_r(lds_u32(sw), lds_u32(sw + 4u), sh);
    if (nwords == 1u) {
        reds_or_u32(dw, v & m_first & m_last);
        return;
    }
    const uint32_t last = (nwords - 1u) * 4u;  // byte offset of the last destination word
    const uint32_t vl = __funnelshift_r(lds_u32(sw + last), lds_u32(sw + last + 4u), sh);
    reds_or_u32(dw, v & m_first);
    reds_or_u32(dw + last, vl & m_last);
#pragma unroll 1
    for (uint32_t j = 4u; j < last; j += 16u) {  // up to four interior words per trip
        const uint32_t n = last - j;             // bytes of interior words from j on (>= 4)
        const uint32_t w0 = lds_u32(sw + j), w1 = lds_u32(sw + j + 4u);
        const uint32_t w2 = n > 4u ? lds_u32(sw + j + 8u) : 0u;
        const uint32_t w3 = n > 8u ? lds_u32(sw + j + 12u) : 0u;
        const uint32_t w4 = n > 12u ? lds_u32(sw + j + 16u) : 0u;
        sts_u32(dw + j, __funnelshift_r(w0, w1, sh));
        if (n > 4u) sts_u32(dw + j + 4u, __funnelshift_r(w1, w2, sh));
        if (n > 8u) sts_u32(dw + j + 8u, __funnelshift_r(w2, w3, sh));
        if (n > 12u) sts_u32(dw + j + 12u, __funnelshift_r(w3, w4, sh));
    }
}
#endif

// ---- Utf8 leaves ----------------------------------------------------------------------------
// Destination of string bytes: the CTA's shared-memory staging area (written out by the kernel afterwards through
// bulk stores) for records walked in shared memory; precise lanes inside such a tile stage their bytes too
// (stage_on; one atomic OR per byte, they are rare), and a tile that does not fit shared memory at all writes its
// strings straight to the Arrow data buffers.
template <class C>
RV_HD void copy_from_record(C& c, int slot_b, int stream, uint32_t o, uint32_t s, uint32_t len) {
#if defined(__CUDA_ARCH__)
    if (C::kShared) {
#if !defined(RV_ABL_NOCOPY)  // (RV_ABL_*: timing ablations for tools/sweep_jit.py — they produce wrong output)
        copy_smem_words(c.stage_saddr + lds_u32(c.adj_saddr + uint32_t(stream) * 4u) + o, c.sbase + s, len);
#endif
        return;
    }
    if (c.stage_on) {
        const uint32_t d = c.stage_saddr + lds_u32(c.adj_saddr + uint32_t(stream) * 4u) + o;
        for (uint32_t i = 0; i < len; ++i) reds_or_u32((d + i) & ~3u, uint32_t(c.base[s + i]) << (((d + i) & 3u) * 8u));
        return;
    }
#endif
    (void)stream;
    uint8_t* dst = static_cast<uint8_t*>(buf_ptr(c, slot_b)) + o;
    for (uint32_t i = 0; i < len; ++i) dst[i] = uint8_t(ld_u8(c, s + i));
}

template <class C>
RV_HD void copy_from_symbols(C& c, int slot_b, int stream, uint32_t o, const uint8_t* src, uint32_t len) {
#if defined(__CUDA_ARCH__)
    if (C::kShared || c.stage_on) {
        const uint32_t d = c.stage_saddr + lds_u32(c.adj_saddr + uint32_t(stream) * 4u) + o;
        for (uint32_t i = 0; i < len; ++i) reds_or_u32((d + i) & ~3u, uint32_t(src[i]) << (((d + i) & 3u) * 8u));
        return;
    }
#endif
    (void)stream;
    uint8_t* dst = static_cast<uint8_t*>(buf_ptr(c, slot_b)) + o;
    for (uint32_t i = 0; i < len; ++i) dst[i] = src[i];
}

template <int MODE, int D, class C>
RV_HD void utf8_finish(C& c, bool valid, uint32_t len, int slot_a, int slot_v, uint32_t& cur, uint32_t row) {
    if (MODE == WM_COUNT) {
        const uint32_t nxt = cur + len;
        if (nxt < cur) fail(c, E_OVERFLOW);
        cur = nxt;
    } else {
        const uint32_t o = cur + len;
        if (may_store<D>(c)) static_cast<int32_t*>(buf_ptr(c, slot_a))[row + 1] = int32_t(o);
        cur = o;
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

template <int MODE, int D, class C>
RV_HD void op_str(C& c, bool valid, int slot_a, int slot_b, int slot_v, int stream, uint32_t row, uint32_t& cur) {  // read_string :902-922
    uint32_t len = 0;
    if (valid) {
        if (!rd_len<MODE == WM_COUNT>(c, len)) { valid = false; len = 0; }
        else {
            if (MODE == WM_EMIT && len) copy_from_record(c, slot_b, stream, cur, c.pos, len);
            c.pos += len;
        }
    }
    utf8_finish<MODE, D>(c, valid, len, slot_a, slot_v, cur, row);
}

template <int MODE, int D, class C>
// `remap` (NF_ENUM_MAP, resolved plans): a writer symbol whose entry after the table's n + 1 offsets is non-zero has no
// reader symbol, and its record fails with E_ENUM_MAP.
RV_HD void op_enum(C& c, bool valid, int slot_a, int slot_b, int slot_v, int stream, uint32_t row, int sym_base, int n_sym, uint32_t& cur,
                   bool remap = false) {  // append_enum :570-578
    uint32_t len = 0;
    if (valid) {
        if (C::kShared) {  // FAST
            uint32_t l = rd_small<MODE == WM_COUNT>(c);
            if (MODE == WM_COUNT && l >= uint32_t(n_sym)) { c.err |= E_ENUM; l = 0; }
            if (MODE == WM_COUNT && remap && c.sym_off[sym_base + n_sym + 1 + int32_t(l)]) c.err |= E_ENUM_MAP;
            const int32_t b0 = c.sym_off[sym_base + int32_t(l)];
            len = uint32_t(c.sym_off[sym_base + int32_t(l) + 1] - b0);
            if (MODE == WM_EMIT) copy_from_symbols(c, slot_b, stream, cur, c.sym_bytes + b0, len);
        } else {
            const int64_t l = rd_varint<MODE == WM_COUNT>(c);
            if (MODE == WM_COUNT && c.err) valid = false;
            else if (MODE == WM_COUNT && uint64_t(l) >= uint64_t(uint32_t(n_sym))) { fail(c, E_ENUM); valid = false; }
            else if (MODE == WM_COUNT && remap && c.sym_off[sym_base + n_sym + 1 + int32_t(l)]) { fail(c, E_ENUM_MAP); valid = false; }
            else {
                const int32_t b0 = c.sym_off[sym_base + int32_t(l)];
                len = uint32_t(c.sym_off[sym_base + int32_t(l) + 1] - b0);
                if (MODE == WM_EMIT) copy_from_symbols(c, slot_b, stream, cur, c.sym_bytes + b0, len);
            }
        }
    }
    utf8_finish<MODE, D>(c, valid, len, slot_a, slot_v, cur, row);
}

// ---- schema resolution (rv_schema_resolve) ----------------------------------------------------------------------
// Bit patterns of a converted value.  One rounding step, to nearest even (__ll2float_rn / __ll2double_rn; on the host the
// default rounding mode of the conversion does the same).
RV_HD uint32_t f32_bits_of_i64(int64_t v) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(__ll2float_rn(v));
#else
    const float f = float(v);
    uint32_t u;
    __builtin_memcpy(&u, &f, 4);
    return u;
#endif
}
RV_HD uint64_t f64_bits_of_i64(int64_t v) {
#if defined(__CUDA_ARCH__)
    return uint64_t(__double_as_longlong(__ll2double_rn(v)));
#else
    const double d = double(v);
    uint64_t u;
    __builtin_memcpy(&u, &d, 8);
    return u;
#endif
}
RV_HD uint64_t f64_bits_of_f32(uint32_t w) {  // exact
#if defined(__CUDA_ARCH__)
    return uint64_t(__double_as_longlong(double(__uint_as_float(w))));
#else
    float f;
    __builtin_memcpy(&f, &w, 4);
    const double d = f;
    uint64_t u;
    __builtin_memcpy(&u, &d, 8);
    return u;
#endif
}

// NK_PROMOTE: the writer's value as op_i32 / op_i64 / op_f32 read it (with their checks), stored as the reader's type.
template <int MODE, int D, class C>
RV_HD void op_promote(C& c, bool valid, int from, int to, int slot_a, int slot_v, uint32_t row) {
    uint64_t bits = 0;
    if (valid) {
        if (from == NK_F32) {
            if (!C::kShared && MODE == WM_COUNT && c.end - c.pos < 4u) { fail(c, E_EOF); valid = false; }
            else {
                if (MODE == WM_EMIT) bits = f64_bits_of_f32(ld_le32(c, c.pos));
                c.pos += 4;
            }
        } else {
            const int64_t x = rd_varint<MODE == WM_COUNT>(c);
            if (C::kShared || MODE == WM_EMIT || !c.err) {
                const int64_t v = from == NK_I32 ? int64_t(int32_t(x)) : x;  // an int is the `as i32` of its varint
                if (MODE == WM_EMIT) bits = to == NK_I64 ? uint64_t(v) : (to == NK_F32 ? uint64_t(f32_bits_of_i64(v)) : f64_bits_of_i64(v));
            } else {
                valid = false;
            }
        }
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) {
            if (to == NK_F32) static_cast<uint32_t*>(buf_ptr(c, slot_a))[row] = uint32_t(bits);
            else static_cast<uint64_t*>(buf_ptr(c, slot_a))[row] = bits;
        }
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

// NK_DEFAULT: reads nothing.  `valid` is false where the parent is absent.  A Utf8 default counts its bytes into the
// node's stream like any string and copies them from the symbol table.
template <int MODE, int D, class C>
RV_HD void op_default(C& c, bool valid, int out, int lo, int hi, int slot_a, int slot_b, int slot_v, int stream, uint32_t row, uint32_t& cur) {
    if (out == NK_STR) {
        uint32_t len = 0;
        if (valid) {
            const int32_t b0 = c.sym_off[lo];
            len = uint32_t(c.sym_off[lo + 1] - b0);
            if (MODE == WM_EMIT && len) copy_from_symbols(c, slot_b, stream, cur, c.sym_bytes + b0, len);
        }
        utf8_finish<MODE, D>(c, valid, len, slot_a, slot_v, cur, row);
        return;
    }
    if (MODE != WM_EMIT) return;
    if (out == NK_BOOL) {
        put_bit<D>(c, slot_a, row, valid && lo != 0);
    } else if (may_store<D>(c)) {
        if (out == NK_I32 || out == NK_F32) static_cast<uint32_t*>(buf_ptr(c, slot_a))[row] = valid ? uint32_t(lo) : 0u;
        else static_cast<uint64_t*>(buf_ptr(c, slot_a))[row] = valid ? ((uint64_t(uint32_t(hi)) << 32) | uint32_t(lo)) : 0ull;
    }
    if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
}

// ---- the wider subset (SURVEY.md 8(f) rank 3): bytes, fixed, uuid, decimal -------------------------------------
// (time-millis / time-micros are op_i32 / op_i64; bytes is op_str.)  The reference has no code for these — its fast
// path rejects the schemas (fast_decode.rs:16-17) and its fallback cannot build the columns (complex.rs:431) — so the
// values follow the Avro specification and the Arrow types schema_translate.rs:58,133-143 assigns.

// `n` bytes at window offset p0 -> dst (global), or zeros for a null slot.
template <class C>
RV_HD void store_raw(C& c, uint8_t* dst, uint32_t p0, uint32_t n, bool valid) {
    for (uint32_t i = 0; i < n; ++i) dst[i] = valid ? uint8_t(ld_u8(c, p0 + i)) : uint8_t(0);
}

// fixed(N) -> FixedSizeBinary(N): N raw bytes.
template <int MODE, int D, class C>
RV_HD void op_fixed(C& c, bool valid, int n_, int slot_a, int slot_v, uint32_t row) {
    const uint32_t n = uint32_t(n_), p0 = c.pos;
    if (valid) {
        if (MODE == WM_COUNT && (C::kShared ? c.pos + n > c.end : c.end - c.pos < n)) { fail(c, E_EOF); valid = false; }
        else c.pos += n;
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) store_raw(c, static_cast<uint8_t*>(buf_ptr(c, slot_a)) + size_t(row) * n, p0, n, valid);
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

RV_HD int hex_val(uint32_t ch) {
    if (ch >= '0' && ch <= '9') return int(ch - '0');
    ch |= 0x20u;
    if (ch >= 'a' && ch <= 'f') return int(ch - 'a' + 10);
    return -1;
}

// uuid (a string on the wire) -> FixedSizeBinary(16), RFC 4122 byte order.  Accepted texts: the hyphenated form
// (8-4-4-4-12, 36 characters) and the plain 32 hex digits.
template <int MODE, int D, class C>
RV_HD void op_uuid(C& c, bool valid, int slot_a, int slot_v, uint32_t row) {
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (valid) {
        uint32_t len = 0;
        if (!rd_len<MODE == WM_COUNT>(c, len)) { valid = false; }
        else if (MODE == WM_COUNT && (C::kShared ? c.err != 0 : false)) { /* not plain: the precise flavour decides */ }
        else if (len != 36u && len != 32u) { if (MODE == WM_COUNT) { fail(c, E_VALUE); if (!C::kShared) valid = false; } }
        else {
            const bool hyph = len == 36u;
            uint32_t p = c.pos;
            bool ok = true;
            for (int i = 0; i < 16; ++i) {
                if (hyph && (i == 4 || i == 6 || i == 8 || i == 10)) { ok = ok && ld_u8(c, p) == uint32_t('-'); ++p; }
                const int hi = hex_val(ld_u8(c, p)), lo = hex_val(ld_u8(c, p + 1));
                p += 2;
                ok = ok && hi >= 0 && lo >= 0;
                w[i >> 2] |= uint32_t(((hi & 15) << 4) | (lo & 15)) << ((i & 3) * 8);
            }
            if (MODE == WM_COUNT && !ok) { fail(c, E_VALUE); if (!C::kShared) valid = false; }
            else c.pos += len;
        }
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) {
            uint32_t* dst = static_cast<uint32_t*>(buf_ptr(c, slot_a)) + size_t(row) * 4;
            for (int i = 0; i < 4; ++i) dst[i] = valid ? w[i] : 0u;
        }
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

// decimal -> Decimal128: `fixed_n` < 0: bytes (varint length first), else fixed(N).  The payload is the unscaled value,
// big-endian two's complement; it is sign-extended into the 16-byte little-endian Arrow value.  More than 16 bytes
// cannot be represented: E_VALUE.
template <int MODE, int D, class C>
RV_HD void op_decimal(C& c, bool valid, int fixed_n, int slot_a, int slot_v, uint32_t row) {
    uint64_t lo = 0, hi = 0;
    if (valid) {
        uint32_t len = 0;
        bool ok = true;
        if (fixed_n < 0) {
            ok = rd_len<MODE == WM_COUNT>(c, len);
            if (ok && MODE == WM_COUNT && len > 16u) { fail(c, E_VALUE); ok = C::kShared; len = 0; }
        } else {
            len = uint32_t(fixed_n);
            if (MODE == WM_COUNT && (C::kShared ? c.pos + len > c.end : c.end - c.pos < len)) { fail(c, E_EOF); ok = false; }
        }
        if (!ok) valid = false;
        else {
            if (MODE == WM_EMIT && len > 0) {
                lo = hi = (ld_u8(c, c.pos) & 0x80u) ? ~0ull : 0ull;
                for (uint32_t i = 0; i < len; ++i) {
                    hi = (hi << 8) | (lo >> 56);
                    lo = (lo << 8) | uint64_t(ld_u8(c, c.pos + i));
                }
            }
            c.pos += len;
        }
    }
    if (MODE == WM_EMIT) {
        if (may_store<D>(c)) {
            uint64_t* dst = static_cast<uint64_t*>(buf_ptr(c, slot_a)) + size_t(row) * 2;
            dst[0] = lo;
            dst[1] = hi;
        }
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

// ---- containers -------------------------------------------------------------------------------
// N-variant union head (UnionDecoder::decode / append_null :643-668): returns the selected variant
// (-1: the union itself is absent -> every child appends null, type_id 0).
template <int MODE, int D, class C>
RV_HD int op_union(C& c, bool valid, int n_variants, int slot_a, uint32_t row) {
    int sel = -1;
    if (valid) {
        if (C::kShared) {  // FAST
            uint32_t idx = rd_small<MODE == WM_COUNT>(c);
            if (MODE == WM_COUNT && idx >= uint32_t(n_variants)) { c.err |= E_BRANCH; idx = 0; }
            sel = int(idx);
        } else {
            const int64_t idx = rd_varint<MODE == WM_COUNT>(c);
            if (MODE == WM_EMIT) sel = int(idx);
            else if (!c.err) {
                if (idx < 0 || idx >= int64_t(n_variants)) fail(c, E_BRANCH);
                else sel = int(idx);
            }
        }
    }
    if (MODE == WM_EMIT && may_store<D>(c)) static_cast<int8_t*>(buf_ptr(c, slot_a))[row] = int8_t(sel < 0 ? 0 : sel);
    return sel;
}

// read_block_count (:689-700) inside the item loop of ListDecoder / MapDecoder (:703-719,745-762).
// Returns 0: list ended or error (leave the loop); 1: `rem` items follow; 2: a zero-width block was
// folded into `total` (read the next block header).
template <bool CHECK = true, class C>
RV_HD int rd_block(C& c, int64_t& rem, uint32_t& total, bool zero_items) {
    int64_t n = rd_varint<CHECK>(c);
    if (C::kShared) {  // FAST: writers emit positive counts; a negative one (with its byte size) is left to the precise flavour
        if (CHECK && (n < 0 || c.err)) { c.err |= E_EOF; return 0; }
        if (n == 0) return 0;
        if (zero_items) {
            if (CHECK && n > int64_t(0x7FFFFFFF) - int64_t(total)) { c.err |= E_OVERFLOW; return 0; }
            total += uint32_t(n);
            return 2;
        }
        rem = n;
        return 1;
    }
    if (CHECK && c.err) return 0;
    if (n < 0) {
        (void)rd_varint<CHECK>(c);  // block byte size: ignored, the items are always walked
        if (CHECK && c.err) return 0;
        n = int64_t(0 - uint64_t(n));
        if (n < 0) return 2;  // i64::MIN: `0..n` is an empty range in the reference
    }
    if (n == 0) return 0;
    if (zero_items) {  // items are zero bytes wide and own no buffers: no need to iterate
        if (CHECK && n > int64_t(0x7FFFFFFF) - int64_t(total)) { fail(c, E_OVERFLOW); return 0; }
        total += uint32_t(n);
        return 2;
    }
    rem = n;
    return 1;
}

// After every item of a list / map in COUNT mode: true = leave the loop.  PRECISE: the first error parked the
// cursor.  FAST: the deferred end-of-buffer check — and ANY "not plain" flag: the lane's fast result is thrown away
// then, and this is what bounds a garbage block count.  (The end-of-buffer test alone does not: an item whose last
// node reads nothing — an unselected union variant, a nested list that just stopped — leaves the cursor parked AT
// the end by eof_check / the inner item_stop, and a forged count of 2^63 would be walked in full.)
template <int MODE, class C>
RV_HD bool item_stop(C& c) {
    if (MODE != WM_COUNT) return false;
    if (C::kShared) {
        if (c.pos > c.end) { c.err |= E_EOF; c.pos = c.end; return true; }
        return c.err != 0;
    }
    return c.err != 0;
}

// ---- skip ops: nodes of a top-level field outside a column projection (NF_SKIP) --------------------------------
// In either walk mode they read and check exactly what the decoding op's COUNT path reads and checks (so the FAST
// flavour raises the same "not plain" flags and the PRECISE flavour the same first error), and store and count nothing.
// One exception, by design: nothing of a skipped field is an Arrow offset, so it cannot overflow one (E_OVERFLOW).
// Leaves: `kind` is a literal in the generated walkers, so the switch folds away.
template <class C>
RV_HD void skip_leaf(C& c, bool valid, int kind, int aux) {
    uint32_t none = 0;  // a length summed for one value only: cannot wrap
    switch (kind) {
        case NK_I32: case NK_I64: op_i64<WM_COUNT, 0>(c, valid, -1, -1, 0u); break;
        case NK_F32: op_f32<WM_COUNT, 0>(c, valid, -1, -1, 0u); break;
        case NK_F64: op_f64<WM_COUNT, 0>(c, valid, -1, -1, 0u); break;
        case NK_BOOL: op_bool<WM_COUNT, 0>(c, valid, -1, -1, 0u); break;
        case NK_STR: case NK_BYTES: op_str<WM_COUNT, 0>(c, valid, -1, -1, -1, -1, 0u, none); break;
        case NK_ENUM:  // op_enum's COUNT checks without the symbol lookup (aux = symbol count)
            if (!valid) break;
            if (C::kShared) {
                if (rd_small<true>(c) >= uint32_t(aux)) c.err |= E_ENUM;
            } else {
                const int64_t l = rd_varint<true>(c);
                if (!c.err && uint64_t(l) >= uint64_t(uint32_t(aux))) fail(c, E_ENUM);
            }
            break;
        case NK_FIXED: op_fixed<WM_COUNT, 0>(c, valid, aux, -1, -1, 0u); break;
        case NK_UUID: op_uuid<WM_COUNT, 0>(c, valid, -1, -1, 0u); break;
        case NK_DEC_BYTES: op_decimal<WM_COUNT, 0>(c, valid, -1, -1, -1, 0u); break;
        case NK_DEC_FIXED: op_decimal<WM_COUNT, 0>(c, valid, aux, -1, -1, 0u); break;
        default: break;  // NK_NULL reads nothing
    }
}

// Block header of a skipped list / map: rd_block's reads and checks without a row count.  0: the list ended (or an
// error); 1: `rem` items follow; 2: read the next header (a block of zero-width items is not iterated).
template <class C>
RV_HD int skip_block(C& c, int64_t& rem, bool zero_items) {
    int64_t n = rd_varint<true>(c);
    if (C::kShared) {
        if (n < 0 || c.err) { c.err |= E_EOF; return 0; }
    } else {
        if (c.err) return 0;
        if (n < 0) {
            (void)rd_varint<true>(c);  // block byte size: ignored, the items are always walked
            if (c.err) return 0;
            n = int64_t(0 - uint64_t(n));
            if (n < 0) return 2;  // i64::MIN: an empty range
        }
    }
    if (n == 0) return 0;
    if (zero_items) return 2;
    rem = n;
    return 1;
}

template <int MODE, int D, class C>
RV_HD void list_finish(C& c, bool valid, uint32_t first_row, uint32_t total, int slot_a, int slot_v, uint32_t& cur, uint32_t row) {
    if (MODE == WM_COUNT) {
        const uint32_t nxt = cur + total;
        if (nxt < cur || nxt > 0x7FFFFFFFu) fail(c, E_OVERFLOW);
        cur = nxt;
    } else {
        cur = first_row + total;
        if (may_store<D>(c)) static_cast<int32_t*>(buf_ptr(c, slot_a))[row + 1] = int32_t(first_row + total);
        if (slot_v >= 0) put_bit<D>(c, slot_v, row, valid);
    }
}

}  // namespace rv
