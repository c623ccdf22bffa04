// kj_emu_seg.cpp -- TEST INFRASTRUCTURE ONLY: the product's SEG filter (kj_seg<LONG> of kaiju_b200/csrc/kj_core.h, compiled with -DKJ_EMU) on the
// CPU warp emulator (kj_emu.cpp, same translation unit), one fragment at a time, in the work space the kernels carve for a given max_len.
// The SEG constants come from the product's own host code (build_tables, kj_lnfact_table of kj_host.cpp, included here for its file-local
// table builder).  Besides the regions, the harness re-walks the region search of kj_seg_level with counters, so a test can tell which
// branches its inputs reach.  Compiled by tests/emu_seg.py.
#include "kj_emu.cpp"
#include "../../kaiju_b200/csrc/kj_host.cpp"

namespace {
// which parts of the region search a fragment reached (summed over the calls of one kjemu_seg)
enum { COV_TRIM_MIN1, COV_TRIM_MAXTRIM, COV_TRIM_LONG, COV_STIRLING, COV_LEVEL1, COV_MERGE, COV_RAW, COV_N };

struct SegState {
    KjTables tb; std::vector<double> lnf; KjDevIndex D; kjemu::Sched* sched;
    SegState() {
        if (build_tables("*ACDEFGHIKLMNPQRSTVWYX", tb) != KJ_OK) { fprintf(stderr, "kjemu_seg: %s\n", kj_last_error()); abort(); }
        kj_lnfact_table(lnf); memset(&D, 0, sizeof D); D.lnfact = lnf.data(); D.n_lnfact = (int)lnf.size(); D.tables = &tb;
        sched = new kjemu::Sched();
    }
};
SegState& state() { static SegState* s = new SegState(); return *s; }

// The harness's copy of kj_seg_level's control flow (same trigger loop, same trims from the product), without a region cap: it records every
// raw region in creation order and counts the branches.  Only the coverage word comes from here; the regions a test compares are kj_seg's.
template <bool LONG>
int cov_level(const KjSegArgs& A, int level, int s0, int n, std::vector<KjSeg>& segs, uint64_t* cov) {
    const uint8_t* frag = A.frag; const uint8_t* hf = A.hf;
    if (KJ_SEG_WINDOW > n) return 0;
    const int first = KJ_SEG_DOWNSET, last = n - KJ_SEG_UPSET; int lowlim = first, made = 0;
    for (int i = first; i <= last; i++) {
        if (!(hf[s0 + i - KJ_SEG_DOWNSET] & 1)) continue;
        int j = i;
        while (j >= lowlim && (hf[s0 + j - KJ_SEG_DOWNSET] & 2)) j--;
        const int loi = j + 1;
        j = i;
        while (j <= last && (hf[s0 + j - KJ_SEG_DOWNSET] & 2)) j++;
        const int hii = j - 1;
        int leftend = loi - KJ_SEG_DOWNSET, rightend = hii + KJ_SEG_UPSET - 1;
        const int n2 = rightend - leftend + 1;
        if (A.w.lane == 0) {
            cov[n2 > 127 ? COV_TRIM_LONG : n2 - KJ_SEG_MAXTRIM > 1 ? COV_TRIM_MAXTRIM : COV_TRIM_MIN1]++;
            if (n2 >= KJ_LNFACT_REF) cov[COV_STIRLING]++;                  // ln(n!) of the window length n2 > 10,000: Stirling's formula
        }
        if constexpr (LONG) { const uint64_t tr = kj_seg_trim_wide(A.w, A.scratch, frag + s0 + leftend, n2, A.lnf); leftend += (int)(tr >> 32); rightend -= n2 - (int)(uint32_t)tr - 1; }
        else { const uint32_t tr = kj_seg_trim(A.w, A.scratch, frag + s0 + leftend, n2, A.lnf); leftend += (int)(tr >> 16); rightend -= n2 - (int)(tr & 0xffffu) - 1; }
        if (level == 0 && i + KJ_SEG_UPSET - 1 < leftend) {
            const int lend = loi - KJ_SEG_DOWNSET, rend = leftend - 1;
            std::vector<KjSeg> sub;
            if (cov_level<LONG>(A, 1, s0 + lend, rend - lend + 1, sub, cov) > 0) { segs.push_back(sub.back()); if (A.w.lane == 0) cov[COV_LEVEL1]++; }
        }
        KjSeg r; r.begin = leftend + s0; r.end = rightend + s0; segs.push_back(r); made++;
        i = hii < rightend + KJ_SEG_DOWNSET ? hii : rightend + KJ_SEG_DOWNSET;
        lowlim = i + 1;
    }
    return made;
}

struct SegArg {
    const uint8_t* res; int n; bool is_long, compact; KjRunParams* rp; KjSmemLayout L; uint8_t* smem; uint32_t err;
    int ns[32]; uint64_t cov[COV_N];
};
void seg_body(kjemu::Sched* s, int lane, void* a) {
    SegArg* A = (SegArg*)a; SegState& S = state();
    KjWarpCtx cx; memset(&cx, 0, sizeof cx);
    cx.w.lane = lane; cx.w.s = s; cx.ix = &S.D; cx.rp = A->rp; cx.tb = &S.tb; cx.smem = A->smem; cx.L = A->L; cx.err = &A->err;
    uint8_t* frag = cx.smem + cx.L.frag_off;
    for (int t = lane; t < A->n; t += 32) frag[t] = A->res[t];
    cx.w.sync();
    A->ns[lane] = A->is_long ? kj_seg<true>(cx, A->n, A->compact) : kj_seg<false>(cx, A->n, A->compact);
    cx.w.sync();
    // coverage: the window flags kj_seg left behind are still in place (the trim scratch lies elsewhere); the product's regions are not touched.
    // No region <=> no window at or below locut (every window can trigger), and then there is nothing to walk.
    if (A->ns[lane] == 0) return;
    KjSegArgs G; G.w = cx.w; G.frag = frag; G.hf = cx.smem + cx.L.hflag_off; G.segs = nullptr; G.scratch = cx.smem + cx.L.segcnt_off; G.lnf = S.lnf.data(); G.cap = 0; G.err = nullptr;
    std::vector<KjSeg> raw; uint64_t cov[COV_N] = {0};
    if (A->is_long) cov_level<true>(G, 0, 0, A->n, raw, cov); else cov_level<false>(G, 0, 0, A->n, raw, cov);
    if (lane == 0) {
        cov[COV_RAW] = raw.size();
        // s_MergeSegs over the reversed creation order, as kj_seg_regions_t walks it: count the merges
        for (int cur = (int)raw.size() - 1, nx = cur - 1; nx >= 0; nx--) {
            if (raw[cur].begin - raw[nx].end - 1 < 0) { cov[COV_MERGE]++; if (raw[cur].begin > raw[nx].begin) raw[cur].begin = raw[nx].begin; }
            else cur = nx;
        }
        for (int k = 0; k < COV_N; k++) A->cov[k] = cov[k];
    }
}
}  // namespace

extern "C" {
// SEG of one fragment (residues = alphabet indices 1..20) in the work space of a batch whose longest mate is max_len bases (kj_fill_run_params).
// Returns the number of merged regions (their [begin, end] pairs in regions[0 .. 2 * min(count, cap))), or -1 when the fragment does not fit
// the work space.  err: the kernel's error flags (8 = region array full).  cov[0..6]: trims of n2 <= 51 (minlen 1), trims of 52..127
// (minlen n2 - 50), trims above 127 residues, trims over more than 10,000 residues, level-1 regions kept, merges, raw regions.
int kjemu_seg(const uint8_t* res, int n, uint32_t max_len, int is_long, int compact, int* regions, int cap, uint32_t* err, uint64_t* cov) {
    kj_params p; memset(&p, 0, sizeof p); p.mode = 0; p.min_fragment_length = 11; p.seg = 1;
    KjRunParams rp; kj_fill_run_params(p, max_len, rp);
    if (n < 0 || (uint32_t)n > rp.max_frag) return -1;
    SegArg A; memset(&A, 0, sizeof A);
    A.res = res; A.n = n; A.is_long = is_long != 0; A.compact = compact != 0; A.rp = &rp;
    A.L = A.is_long ? kj_smem_layout<true>(rp) : kj_smem_layout<false>(rp);
    std::vector<uint8_t> smem(A.L.total + 64, 0xA5);                  // poison: SEG must not rely on zeroed work space
    A.smem = smem.data();
    kjemu::run_warp(state().sched, seg_body, &A);
    for (int l = 1; l < 32; l++) if (A.ns[l] != A.ns[0]) { fprintf(stderr, "kjemu_seg: non-uniform region count\n"); abort(); }
    for (uint32_t g = 0; g < A.L.nguard; g++) for (uint32_t b = 0; b < 64; b++) if (smem[A.L.guard[g] + b] != 0xA5) {
        fprintf(stderr, "kjemu_seg: work-space red zone %u (offset %u) overwritten\n", g, A.L.guard[g]); abort(); }
    for (size_t b = A.L.total; b < smem.size(); b++) if (smem[b] != 0xA5) { fprintf(stderr, "kjemu_seg: store past the work space\n"); abort(); }
    const KjSeg* segs = (const KjSeg*)(smem.data() + A.L.segs_off);
    for (int k = 0; k < A.ns[0] && k < cap; k++) { regions[2 * k] = segs[k].begin; regions[2 * k + 1] = segs[k].end; }
    *err = A.err;
    for (int k = 0; k < COV_N; k++) cov[k] = A.cov[k];
    return A.ns[0];
}
// the region capacity of the work space for max_len (KJ_SEG_CAP of its longest fragment) and that fragment length
int kjemu_seg_cap(uint32_t max_len, uint32_t* max_frag) {
    kj_params p; memset(&p, 0, sizeof p); p.mode = 0; p.min_fragment_length = 11; p.seg = 1;
    KjRunParams rp; kj_fill_run_params(p, max_len, rp); *max_frag = rp.max_frag; return (int)KJ_SEG_CAP(rp.max_frag);
}
}
