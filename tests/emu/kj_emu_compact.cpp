// kj_emu_compact.cpp -- TEST INFRASTRUCTURE ONLY: the CPU warp emulator (kj_emu.cpp, same translation unit) with the compact rank layout
// (kj_layout.h) running on its own instantiation, as kj_select_kernel picks it on the device: an index whose descriptor says layout 2
// (KJ_FORCE_COMPACT) runs kj_classify_item<..., KjCompactIdx, ...> where kj_emu.cpp asks for the 64-bit one.  Also the rank check of the
// layouts against naive counting.  Compiled by tests/emu_compact.py.
#include <type_traits>
#define KJ_EMU 1
#include "../../kaiju_b200/csrc/kj_warp.h"
struct KjEmuStats;
#include "../../kaiju_b200/csrc/kj_core.h"
#include "../../kaiju_b200/csrc/kj_core_greedy.h"

template <int MODE, class IdxT, int ROLE = 0>
static uint32_t kj_emu_item_by_layout(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* rec = nullptr) {
    if constexpr (std::is_same<IdxT, uint64_t>::value)
        if (cx.ix->wide == KJ_LAYOUT_COMPACT) return kj_classify_item<MODE, KjCompactIdx, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
    return kj_classify_item<MODE, IdxT, ROLE>(cx, s1, n1, s2, n2, paired, best_out, rec);
}
#define kj_classify_item kj_emu_item_by_layout
#include "kj_emu.cpp"
#undef kj_classify_item

extern "C" {
// Rank queries of the layout the transcoder picks (KJ_FORCE_COMPACT / KJ_FORCE_WIDE) on a BWT of n letters (codes < alen), against naive counting:
// host_rank and the kernels' kj_rank / LF step for every letter c < alen and every k in [0, n].  The checkpoint quirk is switched off (it is
// checked against the oracle elsewhere).  Returns the number of mismatches (or -1 if the index cannot be built), *layout = the layout.
long long kjemu_rank_check(const uint8_t* bwt, uint64_t n, int alen, int* layout) {
    static const char* kAlpha = "*ACDEFGHIKLMNPQRSTVWYXBZ";
    std::vector<int32_t> start((size_t)alen + 1); for (int a = 0; a <= alen; a++) start[(size_t)a] = a;
    uint8_t sa[8] = {0}; uint64_t st = 1, node = 1, parent = 1;
    kj_index_view v; memset(&v, 0, sizeof v);
    v.alen = alen; v.alphabet = kAlpha; v.bwtlen = (int64_t)n; v.bwt = bwt; v.startLcode = start.data(); v.db_len = (int64_t)n; v.nseq = 1; v.ncheck = 1;
    v.chpt_exp = 0; v.nbytes = 1; v.pbits = 8; v.sa = sa; v.seq_taxon = &st;
    kj_taxonomy_view t; t.n = 1; t.node = &node; t.parent = &parent;
    KjHostIndex H; if (kj_build_host_index(v, t, H) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); return -1; }
    *layout = H.wide; H.quirk_lo = ~0ull;
    KjDevIndex D; memset(&D, 0, sizeof D);
    D.rank = H.rank.data(); D.nb = H.nb; D.letters = H.letters.data(); D.bwtlen = n; D.alen = alen; D.wide = H.wide; D.quirk_lo = ~0ull; D.quirk_d = H.quirk_d; D.sa_check = ~0ull;
    if (H.wide != KJ_LAYOUT_COMPACT) for (int a = 0; a < alen; a++) D.rank_base[a] = D.rank + (uint64_t)a * H.nb * kj_rank_words(H.wide);
    for (int a = 0; a <= alen; a++) D.C[a] = H.C[a];
    long long bad = 0; std::vector<uint64_t> cnt((size_t)alen, 0);
    for (uint64_t k = 0; k <= n; k++) {
        for (int c = 0; c < alen; c++) {
            const uint64_t want = H.C[c] + cnt[(size_t)c];
            const uint64_t dev = H.wide == KJ_LAYOUT_COMPACT ? (uint64_t)kj_rank<KjCompactIdx>(D, (uint32_t)c, (KjCompactIdx)k)
                               : H.wide ? (uint64_t)kj_rank<uint64_t>(D, (uint32_t)c, (uint64_t)k) : (uint64_t)kj_rank<uint32_t>(D, (uint32_t)c, (uint32_t)k);
            bad += (kj_host_rank(H, (uint32_t)c, k) != want) + (dev != want);
        }
        if (k < n) {
            const uint32_t l = bwt[k];
            if (H.wide == KJ_LAYOUT_COMPACT) { uint32_t c = 99; const uint64_t r = kj_clf(D, k, c); bad += (c != l) + (r != H.C[l] + cnt[l]); }
            else bad += kj_letter(D, k) != l;
            cnt[l]++;
        }
    }
    return bad;
}
}
