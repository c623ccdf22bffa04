// kj_emu_tiered.cpp -- TEST INFRASTRUCTURE ONLY: the CPU warp emulator (kj_emu.cpp, same translation unit) on the compact tiered layout
// (kj_layout.h, layout 3), as kj_select_kernel picks it on the device: the transcoded compact records are split at record nb_dev
// (KJ_TIER_DEVICE_RECORDS, clamped to [0, nb]) into two separately allocated arrays, the "device" part [0, nb_dev) and the "host" part
// [nb_dev, nb), and every read runs kj_classify_item<..., KjTieredIdx, ...>.  Each array ends at an inaccessible page and starts behind poisoned
// bytes, so a record address computed from the wrong base or with the wrong offset faults or reads garbage instead of a neighbouring record.
// Compiled twice by tests/emu_tiered.py: the short-read instances, and with -DKJ_EMU_TIERED_LONG the long-read instances (as kj_emu_long.cpp).
#include <sys/mman.h>
#include <unistd.h>
#include <map>
#include <mutex>
#include <type_traits>
#define KJ_EMU 1
#include "../../kaiju_b200/csrc/kj_warp.h"
struct KjEmuStats;
#include "../../kaiju_b200/csrc/kj_core.h"
#include "../../kaiju_b200/csrc/kj_core_greedy.h"
#include "../../kaiju_b200/csrc/kj_host.h"

#if defined(KJ_EMU_TIERED_LONG)
template <int MODE, class IdxT, int ROLE = 0>
static uint32_t kj_emu_item_tiered(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* = nullptr) {
    if (ROLE == 1) return KJ_TAX_BAD;          // the long instances have no front-end / search pair: under KJ_EMU_SPLIT the search runs the whole item
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT_TIERED) return kj_classify_item<MODE, KjTieredIdx, 0, true>(cx, s1, n1, s2, n2, paired, best_out);
    return kj_classify_item<MODE, IdxT, 0, true>(cx, s1, n1, s2, n2, paired, best_out);
}
#undef KJ_MAX_READ_LEN
#define KJ_MAX_READ_LEN KJ_MAX_LONG_READ_LEN
#undef KJ_MAX_PROTEIN_LEN
#define KJ_MAX_PROTEIN_LEN (KJ_MAX_LONG_READ_LEN / 3)
#define kj_smem_layout kj_smem_layout<true>
#define kj_greedy_scratch_bytes kj_greedy_scratch_bytes<true>
#else
template <int MODE, class IdxT, int ROLE = 0>
static uint32_t kj_emu_item_tiered(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* rec = nullptr) {
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT_TIERED) return kj_classify_item<MODE, KjTieredIdx, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
    return kj_classify_item<MODE, IdxT, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
}
#endif
#define kj_classify_item kj_emu_item_tiered
#define kjemu_create kjemu_create_untiered
#define kjemu_destroy kjemu_destroy_untiered
#include "kj_emu.cpp"
#undef kjemu_create
#undef kjemu_destroy

namespace {
// `bytes` of records in a mapping of their own: the array ends where an inaccessible page begins, the bytes between the leading inaccessible
// page and the array hold 0xA5
struct Guarded { void* map = nullptr; size_t len = 0; uint64_t* arr = nullptr; };
Guarded guarded_copy(const uint64_t* src, size_t bytes) {
    const size_t pg = (size_t)sysconf(_SC_PAGESIZE), body = (bytes + pg - 1) / pg * pg;
    Guarded g; g.len = body + 2 * pg;
    g.map = mmap(nullptr, g.len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (g.map == MAP_FAILED) { perror("kjemu: mmap"); abort(); }
    char* b = (char*)g.map;
    memset(b + pg, 0xA5, body);
    g.arr = (uint64_t*)(b + pg + body - bytes);
    if (bytes) memcpy(g.arr, src, bytes);
    if (mprotect(b, pg, PROT_NONE) || mprotect(b + pg + body, pg, PROT_NONE) || mprotect(b + pg, body, PROT_READ)) { perror("kjemu: mprotect"); abort(); }
    return g;
}
struct Split { Guarded dev, host; };
std::mutex g_split_mu; std::map<void*, Split> g_splits;
}

extern "C" {
// the emulator context of kj_emu.cpp; a compact index (KJ_FORCE_COMPACT) is split into the tiered layout when KJ_TIER_DEVICE_RECORDS is set
void* kjemu_create(const char* fmi_path, const char* nodes_path, const kj_params* p) {
    void* h = kjemu_create_untiered(fmi_path, nodes_path, p);
    const char* e = getenv("KJ_TIER_DEVICE_RECORDS");
    if (!h || !e) return h;
    EmuCtx* c = (EmuCtx*)h; KjDevIndex& D = c->D;
    if (D.wide != KJ_LAYOUT_COMPACT) return h;
    const uint64_t nb = c->H.nb, nd = std::min<uint64_t>((uint64_t)atoll(e), nb), W = KJ_RANK_WORDS_COMPACT;
    Split s; s.dev = guarded_copy(c->H.rank.data(), (size_t)(nd * W * 8)); s.host = guarded_copy(c->H.rank.data() + nd * W, (size_t)((nb - nd) * W * 8));
    D.rank = s.dev.arr; D.tier.host = s.host.arr; D.tier.nb_dev = nd; D.wide = KJ_LAYOUT_COMPACT_TIERED;
    std::vector<uint64_t>().swap(c->H.rank);          // only the two split arrays are left to read
    std::lock_guard<std::mutex> lk(g_split_mu); g_splits[h] = s;
    return h;
}
void kjemu_destroy(void* h) {
    {
        std::lock_guard<std::mutex> lk(g_split_mu);
        auto it = g_splits.find(h);
        if (it != g_splits.end()) { munmap(it->second.dev.map, it->second.dev.len); munmap(it->second.host.map, it->second.host.len); g_splits.erase(it); }
    }
    kjemu_destroy_untiered(h);
}
// layout of the emulator context (3 = compact tiered) and its split record
int kjemu_layout(void* h, unsigned long long* nb_dev, unsigned long long* nb) {
    const EmuCtx* c = (const EmuCtx*)h;
    if (nb_dev) *nb_dev = c->D.wide == KJ_LAYOUT_COMPACT_TIERED ? c->D.tier.nb_dev : c->D.nb;
    if (nb) *nb = c->D.nb;
    return c->D.wide;
}
}
