// kj_emu_long.cpp -- TEST INFRASTRUCTURE ONLY: the CPU warp emulator (kj_emu.cpp, same translation unit) on the long-read instances
// (kj_classify_item<..., LONG = true>, the wide fields of kj_core.h KjW<true>), as the library runs them for mates longer than KJ_MAX_READ_LEN:
// every read goes through the long instance (of the compact layout where the descriptor says compact), with the long work-space layout and
// Greedy ring, and reads of up to KJ_MAX_LONG_READ_LEN bases are admitted.  Compiled by tests/emu_long.py.
#include <type_traits>
#define KJ_EMU 1
#include "../../kaiju_b200/csrc/kj_warp.h"
struct KjEmuStats;
#include "../../kaiju_b200/csrc/kj_core.h"
#include "../../kaiju_b200/csrc/kj_core_greedy.h"
#include "../../kaiju_b200/csrc/kj_host.h"

template <int MODE, class IdxT, int ROLE = 0>
static uint32_t kj_emu_item_long(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* = nullptr) {
    if (ROLE == 1) return KJ_TAX_BAD;          // the long instances have no front-end / search pair: under KJ_EMU_SPLIT the search runs the whole item
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT) return kj_classify_item<MODE, KjCompactIdx, 0, true>(cx, s1, n1, s2, n2, paired, best_out);
    return kj_classify_item<MODE, IdxT, 0, true>(cx, s1, n1, s2, n2, paired, best_out);
}
#undef KJ_MAX_READ_LEN
#define KJ_MAX_READ_LEN KJ_MAX_LONG_READ_LEN
#undef KJ_MAX_PROTEIN_LEN
#define KJ_MAX_PROTEIN_LEN (KJ_MAX_LONG_READ_LEN / 3)
#define kj_classify_item kj_emu_item_long
#define kj_smem_layout kj_smem_layout<true>
#define kj_greedy_scratch_bytes kj_greedy_scratch_bytes<true>
#include "kj_emu.cpp"
