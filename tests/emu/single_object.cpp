// TEST INFRASTRUCTURE ONLY — host emulation of the single-object partition (rv_decode_*_versions on a registry from
// rv_versions_create_single_object): the product's 64-bit header check (take.cuh vp_header over fingerprints), one lane
// per message.  The device's vp_count_kernel runs tiles of kTakeBlock messages inside each output chunk and keeps the
// lowest failing message with atomicMin; the tiles run here last chunk first, last tile first, so that only the minimum,
// not the order, can decide which message is reported.
#include <algorithm>
#include <cstdint>

#include "../../pyruhvro_b200/csrc/take.cuh"

using namespace rv;

// writer[i]: the index into fps (ascending) of message i's fingerprint, -1 for a message that failed its header check.
// Returns 0, or the code of the lowest failing message (E_FRAME 12, E_FRAME_ID 14) with *err_record its index.
extern "C" int emu_partition_single_object(const uint8_t* data, const int64_t* off, int64_t n, int64_t k, const unsigned long long* fps,
                                           int n_fps, int32_t* writer, int64_t* err_record) {
    k = std::max<int64_t>(1, std::min<int64_t>(k, std::max<int64_t>(n, 1)));
    const int64_t cr = n / k;
    unsigned long long best = ~0ull;
    for (int64_t j = k - 1; j >= 0; --j) {
        const int64_t cs = j * cr, ce = j == k - 1 ? n : cs + cr;
        for (int64_t t0 = cs + ((ce - cs - 1) / kTakeBlock) * kTakeBlock; t0 >= cs; t0 -= kTakeBlock)
            for (int64_t i = t0; i < std::min(ce, t0 + kTakeBlock); ++i) {
                int w = -1;
                const uint32_t code = vp_header(data + off[i], off[i + 1] - off[i], fps, n_fps, &w);
                if (code != E_OK) best = std::min(best, (static_cast<unsigned long long>(i) << 8) | code);
                writer[i] = code == E_OK ? w : -1;
            }
    }
    if (best == ~0ull) return 0;
    *err_record = int64_t(best >> 8);
    return int(best & 0xFF);
}
