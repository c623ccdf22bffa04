// kj_emu_spread.cpp -- TEST INFRASTRUCTURE ONLY: the CPU warp emulator (kj_emu.cpp, same translation unit) on the compact spread layout
// (kj_layout.h, layout 4), as kj_select_kernel picks it on the device: the transcoded compact records are cut into G contiguous segments
// (KJ_SPREAD_RECORDS=n0,n1,...: the record counts of every segment but the last, which takes the rest, as in kj_plan_group), each copied into
// an array of its own, and every read runs kj_classify_item<..., KjSpreadIdx, ...>.  Each array ends at an inaccessible page and starts behind
// poisoned bytes, so a record address computed from the wrong segment or with the wrong offset faults or reads garbage instead of a
// neighbouring record.  Compiled twice by tests/emu_spread.py: the short-read instances, and with -DKJ_EMU_SPREAD_LONG the long-read instances.
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

#if defined(KJ_EMU_SPREAD_LONG)
template <int MODE, class IdxT, int ROLE = 0>
static uint32_t kj_emu_item_spread(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* = nullptr) {
    if (ROLE == 1) return KJ_TAX_BAD;          // the long instances have no front-end / search pair: under KJ_EMU_SPLIT the search runs the whole item
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT_SPREAD) return kj_classify_item<MODE, KjSpreadIdx, 0, true>(cx, s1, n1, s2, n2, paired, best_out);
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
static uint32_t kj_emu_item_spread(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* rec = nullptr) {
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT_SPREAD) return kj_classify_item<MODE, KjSpreadIdx, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
    return kj_classify_item<MODE, IdxT, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
}
#endif
#define kj_classify_item kj_emu_item_spread
#define kjemu_create kjemu_create_unspread
#define kjemu_destroy kjemu_destroy_unspread
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
std::mutex g_split_mu; std::map<void*, std::vector<Guarded>> g_splits;
}

extern "C" {
// the emulator context of kj_emu.cpp; a compact index (KJ_FORCE_COMPACT) is cut into the spread layout when KJ_SPREAD_RECORDS is set
void* kjemu_create(const char* fmi_path, const char* nodes_path, const kj_params* p) {
    void* h = kjemu_create_unspread(fmi_path, nodes_path, p);
    const char* e = getenv("KJ_SPREAD_RECORDS");
    if (!h || !e) return h;
    EmuCtx* c = (EmuCtx*)h; KjDevIndex& D = c->D;
    if (D.wide != KJ_LAYOUT_COMPACT) return h;
    const uint64_t nb = c->H.nb, W = KJ_RANK_WORDS_COMPACT;
    std::vector<uint64_t> first{0};
    for (const char* q = e; *q;) {
        const uint64_t n = strtoull(q, (char**)&q, 10); if (*q == ',') q++;
        if (first.size() < KJ_MAX_GROUP) first.push_back(std::min(nb, first.back() + n));
    }
    const size_t G = first.size(); first.push_back(nb);
    std::vector<Guarded> segs;
    memset(&D.spread, 0, sizeof D.spread);
    for (int g = 0; g < KJ_MAX_GROUP; g++) D.spread.first[g] = ~0ull;
    for (size_t g = 0; g < G; g++) {
        segs.push_back(guarded_copy(c->H.rank.data() + first[g] * W, (size_t)((first[g + 1] - first[g]) * W * 8)));
        D.spread.base[g] = segs.back().arr; D.spread.first[g] = first[g];
    }
    D.spread.n = (uint32_t)G; D.rank = D.spread.base[0]; D.wide = KJ_LAYOUT_COMPACT_SPREAD;
    std::vector<uint64_t>().swap(c->H.rank);          // only the segments are left to read
    std::lock_guard<std::mutex> lk(g_split_mu); g_splits[h] = segs;
    return h;
}
void kjemu_destroy(void* h) {
    {
        std::lock_guard<std::mutex> lk(g_split_mu);
        auto it = g_splits.find(h);
        if (it != g_splits.end()) { for (Guarded& g : it->second) munmap(g.map, g.len); g_splits.erase(it); }
    }
    kjemu_destroy_unspread(h);
}
// layout of the emulator context (4 = compact spread), its segment count and starts (first[0..n], first[n] = nb)
int kjemu_layout(void* h, unsigned int* n_seg, unsigned long long* first) {
    const EmuCtx* c = (const EmuCtx*)h;
    const bool sp = c->D.wide == KJ_LAYOUT_COMPACT_SPREAD; const uint32_t n = sp ? c->D.spread.n : 1;
    if (n_seg) *n_seg = n;
    if (first) { for (uint32_t g = 0; g < n; g++) first[g] = sp ? c->D.spread.first[g] : 0; first[n] = c->D.nb; }
    return c->D.wide;
}
}
