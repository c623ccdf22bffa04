// kj_core.h -- the per-read classification path as warp-cooperative device code (one warp = one read item).
//
// Replaces, behind the C ABI of include/kaiju_b200.h, the reference's
//   ConsumerThread::doWork / getAllFragmentsBits / getNextFragment / classify_length / classify_greedyblosum /
//   addAllMismatchVariantsAtPosSI / eval_match_scores / ids_from_SI   (src/ConsumerThread.cpp:190-845)
//   greedyExact / maxMatches / maxMatches_withStart / UpdateSI / InitialSI / get_suffix (src/bwt/bwt.c:105-380)
//   FMindex / FMindexCurrent (src/bwt/compactfmi.c:267-336), SeqBufferSeg (blast_seg.c:2278-2332),
//   lca_from_ids (src/util.cpp:194-263).
// It is not a translation: lanes run independent backward-search chains (one per match end position j),
// the fragment priority queue is a shared-memory key array popped by warp arg-max, SEG's window entropies
// are integer class look-ups and its trim search is lane-parallel, ids are resolved 32 SA rows at a time.
// The sequential semantics that decide ties (SURVEY.md 8a "exactness notes") are replayed exactly.
//
// Conventions: every warp collective is called from warp-uniform control flow with the full mask;
// variables commented "uniform" hold the same value in all 32 lanes.
#pragma once
#include "kj_warp.h"
#include "kj_layout.h"

// ---------------------------------------------------------------------------------------------
// per-warp shared-memory carve-up
// ---------------------------------------------------------------------------------------------
#define KJ_SEG_CAP(max_frag) ((max_frag) / 4u + 8u)
struct KjKept { uint64_t lo; uint32_t len; uint32_t aux; };     // one suffix interval (an SI of bwt.h:25-34)

// Field width is a compile-time property of an instantiation.  LONG = false: the kernels of mates up to KJ_MAX_READ_LEN bases (15-bit array
// positions and 14-bit lengths in 32-bit queue payloads, 16-bit match positions, prefix sums and SEG counts).  LONG = true: the long-read
// kernels (mates up to KJ_MAX_LONG_READ_LEN = 2^20 - 1 bases): 64-bit payloads, 32-bit positions, prefix sums and counts, unclamped scores.
template <bool LONG> struct KjW { typedef uint32_t pay; typedef uint16_t pos; };
template <> struct KjW<true> { typedef uint64_t pay; typedef uint32_t pos; };
#define KJ_LONG_LO_BITS 40      // long kernels: suffix-array rows stay below 2^40, so a match start rides in the bits above (Greedy's result list)

// (member order: the kernels read these from the parameter bank in 8-byte pairs; accs_off and total are read together)
struct KjSmemLayout {
    uint32_t qkey_off, qpay_off, kept_off, res_off, res2_off, pre_off, ids_off, qord_off, aa_off, aa_stride, frag_off, hflag_off,
             segcnt_off, seghist_off, accs_off, total, segs_off;
#if defined(KJ_EMU)
    uint32_t guard[16], nguard;         // emulator only: 64-byte red zones between the sub-arrays, checked after every read item
#endif
};
#if defined(KJ_EMU)
#define KJ_GUARD(L, o) { (L).guard[(L).nguard++] = (o); (o) += 64u; }
#else
#define KJ_GUARD(L, o)
#endif
static KJ_HD uint32_t kj_align(uint32_t x, uint32_t a) { return (x + a - 1) / a * a; }
template <bool LONG = false>
static KJ_HD KjSmemLayout kj_smem_layout(const KjRunParams& p) {
    constexpr uint32_t pay_bytes = sizeof(typename KjW<LONG>::pay), match_bytes = LONG ? 24u : 16u, pre_bytes = sizeof(typename KjW<LONG>::pos);
    KjSmemLayout L; uint32_t o = 0;
#if defined(KJ_EMU)
    L.nguard = 0;
#endif
    L.qkey_off = o; o += 8u * p.item_cap; KJ_GUARD(L, o)
    L.kept_off = o; o += 16u * p.kept_cap_smem; KJ_GUARD(L, o)
    L.segs_off = o; o += 8u * KJ_SEG_CAP(p.max_frag); KJ_GUARD(L, o)          // {int begin,end}
    L.qpay_off = o; o += pay_bytes * kj_align(p.item_cap, 2); KJ_GUARD(L, o)
    L.qord_off = o; o += kj_align(p.item_cap, 8); KJ_GUARD(L, o)           // slots in pop order (valid while no SEG piece was pushed)
    L.ids_off = o; o += 4u * 24u; KJ_GUARD(L, o)
    L.accs_off = o; o += 4u * 24u; KJ_GUARD(L, o)                            // accession ranks of the visited sequences (verbose output) + their count
    L.aa_stride = kj_align(p.max_len + 4, 8);
    L.aa_off = o; o += 4u * L.aa_stride; KJ_GUARD(L, o)
    L.frag_off = o; o += kj_align(p.max_frag + 8, 8); KJ_GUARD(L, o)
    L.hflag_off = o; o += kj_align(p.max_frag + 8, 8); KJ_GUARD(L, o)
    // union: SEG trim scratch (alive inside getNextFragment's SEG gate) | greedy search arrays (alive after the gate)
    const uint32_t u = o;
    L.segcnt_off = u; L.seghist_off = u + 20u * 32u;
    // count histograms of the lane-parallel trim search for regions <= 127 residues; longer regions use the sorted-composition
    // variant (kj_seg_trim_long), whose per-lane state (20 x {uint16 count, letter, position}; uint32 counts in the long kernels) fits in the same bytes
    const uint32_t seg_rows = p.max_frag + 2 < 130u ? p.max_frag + 2 : 130u;
    const uint32_t seg_bytes = 20u * 32u + kj_align(seg_rows * 32u, 8);
    uint32_t g_bytes = 0;
    L.res_off = u; L.res2_off = u; L.pre_off = u;
    if (p.mode == 1) {
        L.res_off = u; g_bytes += match_bytes * kj_align(p.max_frag + 1, 2);           // per-j chain results
        L.res2_off = u + g_bytes; g_bytes += match_bytes * kj_align(p.max_frag + 1, 2);  // recorded matches in class order
        L.pre_off = u + g_bytes; g_bytes += pre_bytes * kj_align(p.max_frag + 2, 4);    // prefix sums of the BLOSUM62 diagonal
    }
    o = u + (seg_bytes > g_bytes ? seg_bytes : g_bytes);
    KJ_GUARD(L, o)
    L.total = kj_align(o, 16);
    return L;
}

struct KjWarpCtx {
    Warp w;
    const KjDevIndex* ix;
    const KjRunParams* rp;
    const KjTables* tb;
    uint8_t* smem;                      // this warp's carve-up
    KjSmemLayout L;
    KjKept* spill;                      // global scratch of this warp: rp->scratch_entries entries
    void* gscratch;                     // global scratch of this warp for the greedy variant queue
    uint32_t nids;                      // size of the match-id set left in shared memory by the last item (uniform)
    uint32_t* err;                      // global error flags: 1 item-queue overflow, 2 spill overflow, 4 greedy queue overflow, 128 fragment text overflow
    char* text; uint32_t text_cap, text_len;   // verbose output: the read's fragment-string area (nullptr = not requested), bytes used (uniform)
    bool want_acc;                       // verbose output: collect accession ranks
};
static KJ_DEV void kj_flag_error(KjWarpCtx& cx, uint32_t bit) {
#if defined(KJ_EMU)
    *cx.err |= bit;
#else
    atomicOr(cx.err, bit);
#endif
}

// Chosen by A/B runs: one warp's time is dominated by chains of dependent short-latency instructions,
// so shorter dependence chains beat fewer instructions.  Tried and rejected as slower: two lanes per chain in phase B,
// compaction of low-diversity SEG windows, screening several queued fragments at once with two chains per lane.
// ---------------------------------------------------------------------------------------------
// FM index primitives.  IdxT = uint32_t for indexes with bwtlen < 2^32 (all interval arithmetic in 32 bit), uint64_t otherwise.
// ---------------------------------------------------------------------------------------------
static KJ_DEV uint64_t kj_ld64(const void* p) {
#if defined(KJ_EMU)
    return *(const uint64_t*)p;
#else
    uint64_t v; asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(v) : "l"(p)); return v;
#endif
}
static KJ_DEV void kj_ld128(const void* p, uint64_t& a, uint64_t& b) {
#if defined(KJ_EMU)
    a = ((const uint64_t*)p)[0]; b = ((const uint64_t*)p)[1];
#else
    asm volatile("ld.global.nc.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
#endif
}
// FMindex(f, c, k) = C[c] + rank_c(BWT[0..k))        (compactfmi.c:267-307) for one end of an interval.  `base` = records of letter c.
// 32-bit kernels (narrow layout): ONE 16-byte load (header + the bitmap word of k's 64-row block) and one popcount.
// 64-bit kernels (wide layout): header + the one bitmap word holding row k -- two 8-byte loads from the same 32-byte sector,
// one popcount, no data-dependent branches; k < 2^38 so k >> 6 fits 32 bits.
template <class IdxT>
static KJ_DEV IdxT kj_rank_at(const uint64_t* base, IdxT k) {
    if (sizeof(IdxT) == 4) {
        uint64_t h, wd; kj_ld128(base + 2u * (size_t)((uint32_t)k >> 6), h, wd);
        return (IdxT)((uint32_t)h + (uint32_t)kj_popcll(wd & ((1ull << ((uint32_t)k & 63u)) - 1ull)));
    }
    const uint32_t q = (uint32_t)((uint64_t)k >> 6), blk = q / 3u, wi = q - 3u * blk, bit = (uint32_t)k & 63u;
    const uint64_t* rec = base + 4u * (size_t)blk;
    const uint64_t hdr = kj_ld64(rec);
    const uint64_t ww = kj_ld64(rec + 1u + wi);
    const uint32_t pc = (uint32_t)kj_popcll(ww & ((1ull << bit) - 1ull));
    const uint32_t add = wi == 0 ? 0u : ((uint32_t)(hdr >> (32u + 8u * wi)) & 0xffu);
    return (IdxT)((hdr & KJ_CNT_MASK) + (uint64_t)(add + pc));
}
// The compact layout (kj_layout.h) runs the 64-bit kernels with IdxT = KjCompactIdx: a 64-bit unsigned type distinct from uint64_t (unsigned
// long), so that the layout is a compile-time property of the instantiation and the narrow and wide instantiations are untouched by it.
typedef unsigned long long KjCompactIdx;
template <class IdxT> struct KjIsCompact { static constexpr bool v = false; };
template <> struct KjIsCompact<KjCompactIdx> { static constexpr bool v = true; };
static_assert(sizeof(KjCompactIdx) == 8 && !KjIsCompact<uint64_t>::v, "KjCompactIdx must be a 64-bit type distinct from uint64_t");
// The compact tiered layout (records [nb_dev, nb) in mapped host memory) runs them with IdxT = KjTieredIdx: a third 64-bit type, a row index
// that converts to and from unsigned 64-bit integers, so the interval arithmetic of the kernels is that of the compact instantiation.
struct KjTieredIdx {
    unsigned long long v;
    KjTieredIdx() = default;
    KJ_HD constexpr KjTieredIdx(unsigned long long x) : v(x) {}
    KJ_HD constexpr operator unsigned long long() const { return v; }
    KJ_HD KjTieredIdx& operator-=(KjTieredIdx d) { v -= d.v; return *this; }
};
template <class IdxT> struct KjIsTiered { static constexpr bool v = false; };
template <> struct KjIsTiered<KjTieredIdx> { static constexpr bool v = true; };
static_assert(sizeof(KjTieredIdx) == 8 && !KjIsTiered<uint64_t>::v && !KjIsTiered<KjCompactIdx>::v && !KjIsCompact<KjTieredIdx>::v,
              "KjTieredIdx must be a 64-bit type distinct from uint64_t and KjCompactIdx");
// The compact spread layout (records in segments over the HBM of a group of GPUs) runs them with IdxT = KjSpreadIdx: a fourth 64-bit type, built
// like KjTieredIdx.
struct KjSpreadIdx {
    unsigned long long v;
    KjSpreadIdx() = default;
    KJ_HD constexpr KjSpreadIdx(unsigned long long x) : v(x) {}
    KJ_HD constexpr operator unsigned long long() const { return v; }
    KJ_HD KjSpreadIdx& operator-=(KjSpreadIdx d) { v -= d.v; return *this; }
};
template <class IdxT> struct KjIsSpread { static constexpr bool v = false; };
template <> struct KjIsSpread<KjSpreadIdx> { static constexpr bool v = true; };
static_assert(sizeof(KjSpreadIdx) == 8 && !KjIsSpread<uint64_t>::v && !KjIsSpread<KjCompactIdx>::v && !KjIsSpread<KjTieredIdx>::v &&
              !KjIsCompact<KjSpreadIdx>::v && !KjIsTiered<KjSpreadIdx>::v, "KjSpreadIdx must be a 64-bit type distinct from the other index types");
// where kj_crec finds a compact record: one array, two tiers, or the segments of a group
#define KJ_CREC_ONE 0
#define KJ_CREC_TIER 1
#define KJ_CREC_SPREAD 2
// compact layout: rank of letter c at row k from the plane words of k's half-record `pl` (5 independent loads, issued by the caller) plus the
// midpoint count and the superblock count -- every address a function of (c, k) only, and no branch on the data
static KJ_DEV uint64_t kj_crank_planes(const KjDevIndex& ix, const uint64_t* rec, const uint64_t pw[5], uint32_t c, uint64_t k) {
    const uint64_t cw = kj_ld64(rec + KJ_CPT_COUNT_WORD + (c >> 2));
    const uint64_t sb = kj_ld64(ix.csb + (size_t)(k >> KJ_CSB_SHIFT) * KJ_CSB_STRIDE + c);
    uint64_t m = ~0ull;
    #pragma unroll
    for (int b = 0; b < 5; b++) m &= pw[b] ^ ((uint64_t)((c >> b) & 1u) - 1ull);      // rows whose letter equals c
    const uint32_t h = (uint32_t)(k >> 6) & 1u;
    const uint64_t below = (1ull << ((uint32_t)k & 63u)) - 1ull;
    // second half: rows [midpoint, k) are added; first half: rows [k, midpoint) are subtracted
    const uint64_t pc = (uint64_t)kj_popcll(m & (h ? below : ~below));
    const uint64_t v = sb + ((cw >> (16u * (c & 3u))) & 0xffffull);
    return h ? v + pc : v - pc;
}
// WHERE = KJ_CREC_TIER (compact tiered layout): the record lies in HBM below the split, in mapped host memory above it -- the base and the index
// are selected, not branched on, so the load addresses still follow from (c, k) alone.  KJ_CREC_SPREAD (compact spread layout): the segment of
// b = k >> 7 is the number of segment starts first[1..7] at or below b (an unrolled compare, unused slots hold ~0), then its base and first
// record are selected by that number -- again no branch, and an empty segment is never chosen (the next one starts at the same record).
// the segment of record b: record numbers are below 2^32 - 1 (kj_plan_group), so the compares take the low words (unused slots: 0xffffffff)
static KJ_DEV uint32_t kj_spread_seg(const KjSpreadRef& s, uint64_t b) {
    const uint32_t r = (uint32_t)b; uint32_t g = 0;
    #pragma unroll
    for (int i = 1; i < KJ_MAX_GROUP; i++) g += r >= (uint32_t)s.first[i] ? 1u : 0u;
    return g;
}
template <int WHERE = KJ_CREC_ONE>
static KJ_DEV const uint64_t* kj_crec(const KjDevIndex& ix, uint64_t k) {
    if constexpr (WHERE == KJ_CREC_TIER) {
        const uint64_t b = k >> 7, nd = ix.tier.nb_dev; const bool dev = b < nd;
        const uint64_t* base = dev ? ix.rank : ix.tier.host;
        return base + (size_t)(dev ? b : b - nd) * KJ_RANK_WORDS_COMPACT;
    } else if constexpr (WHERE == KJ_CREC_SPREAD) {
        const uint64_t b = k >> 7; const uint32_t g = kj_spread_seg(ix.spread, b);
        return ix.spread.base[g] + (size_t)(b - ix.spread.first[g]) * KJ_RANK_WORDS_COMPACT;
    } else return ix.rank + (size_t)(k >> 7) * KJ_RANK_WORDS_COMPACT;
}
static KJ_DEV void kj_cplanes(const uint64_t* rec, uint64_t k, uint64_t pw[5]) {
    const uint64_t* pl = rec + 5u * ((uint32_t)(k >> 6) & 1u);
    #pragma unroll
    for (int b = 0; b < 5; b++) pw[b] = kj_ld64(pl + b);
}
template <int WHERE = KJ_CREC_ONE>
static KJ_DEV uint64_t kj_crank(const KjDevIndex& ix, uint32_t c, uint64_t k) {
    const uint64_t* rec = kj_crec<WHERE>(ix, k); uint64_t pw[5]; kj_cplanes(rec, k, pw);
    return kj_crank_planes(ix, rec, pw, c, k);
}
// one LF step of the compact layout: the letter of row k and its rank, from k's record
template <int WHERE = KJ_CREC_ONE>
static KJ_DEV uint64_t kj_clf(const KjDevIndex& ix, uint64_t k, uint32_t& c) {
    const uint64_t* rec = kj_crec<WHERE>(ix, k); uint64_t pw[5]; kj_cplanes(rec, k, pw);
    const uint32_t bit = (uint32_t)k & 63u; c = 0;
    #pragma unroll
    for (int b = 0; b < 5; b++) c |= (uint32_t)((pw[b] >> bit) & 1ull) << b;
    return kj_crank_planes(ix, rec, pw, c, k);
}
static KJ_DEV const uint64_t* kj_letter_base(const KjDevIndex& ix, uint32_t c) { return ix.rank_base[c]; }
template <class IdxT>
static KJ_DEV IdxT kj_rank(const KjDevIndex& ix, uint32_t c, IdxT k) {
    if constexpr (KjIsCompact<IdxT>::v) return (IdxT)kj_crank(ix, c, (uint64_t)k);
    else if constexpr (KjIsTiered<IdxT>::v) return (IdxT)kj_crank<KJ_CREC_TIER>(ix, c, (uint64_t)k);
    else if constexpr (KjIsSpread<IdxT>::v) return (IdxT)kj_crank<KJ_CREC_SPREAD>(ix, c, (uint64_t)k);
    else return kj_rank_at<IdxT>(kj_letter_base(ix, c), k);
}
// UpdateSI (bwt.c:160-173)
template <class IdxT>
static KJ_DEV bool kj_update_si(const KjDevIndex& ix, uint32_t c, IdxT& lo, IdxT& hi) {
    IdxT nlo, nhi;
    if constexpr (KjIsCompact<IdxT>::v) { nlo = (IdxT)kj_crank(ix, c, (uint64_t)lo); nhi = (IdxT)kj_crank(ix, c, (uint64_t)hi); }
    else if constexpr (KjIsTiered<IdxT>::v) { nlo = (IdxT)kj_crank<KJ_CREC_TIER>(ix, c, (uint64_t)lo); nhi = (IdxT)kj_crank<KJ_CREC_TIER>(ix, c, (uint64_t)hi); }
    else if constexpr (KjIsSpread<IdxT>::v) { nlo = (IdxT)kj_crank<KJ_CREC_SPREAD>(ix, c, (uint64_t)lo); nhi = (IdxT)kj_crank<KJ_CREC_SPREAD>(ix, c, (uint64_t)hi); }
    else { const uint64_t* base = kj_letter_base(ix, c); nlo = kj_rank_at<IdxT>(base, lo); nhi = kj_rank_at<IdxT>(base, hi); }
    // the reference's checkpoint quirk (indexes with bwtlen = m * 2^16 only, kj_host.cpp): the last 129 positions rank lower by a per-letter
    // constant.  Such indexes are routed to the 64-bit kernels, so the 32-bit ones do not carry the test.
    if (sizeof(IdxT) == 8) { if (hi >= (IdxT)ix.quirk_lo) { const IdxT d = (IdxT)ix.quirk_d[c]; nhi -= d; if (lo >= (IdxT)ix.quirk_lo) nlo -= d; } }
    if (nlo >= nhi) return false;
    lo = nlo; hi = nhi; return true;
}
static KJ_DEV int kj_hibit64(uint64_t x) { uint32_t h = (uint32_t)(x >> 32); return h ? 63 - kj_clz(h) : 31 - kj_clz((uint32_t)x); }
static KJ_DEV uint32_t kj_letter(const KjDevIndex& ix, uint64_t k) {
    uint64_t wd = k / KJ_LETTERS_PER_WORD; uint32_t s = (uint32_t)(k - wd * KJ_LETTERS_PER_WORD) * 5u;
    return (uint32_t)(ix.letters[wd] >> s) & 31u;
}
#if defined(KJ_EMU)
// emulator counters.  Phase A/B: rounds, round_steps (max over lanes, summed), lane_steps, chains, blocks, lookaheads; Greedy queue: pops_frag,
// pops_var, var_steps, var_pushed; taxon look-up of the kept rows (kj_ids_and_lca_fn): id_reads (reads that got there), kept (their kept
// intervals), sa_waves (waves of up to 32 rows), sa_lf_steps (LF steps summed over lanes), sa_dep_steps (max over the lanes of a wave, summed);
// long-read queue: lq_tops (look-ups of the top entry), lq_slots (queue slots they read: the sorted head plus the late entries scanned)
struct KjEmuStats { unsigned long long rounds, round_steps, lane_steps, chains, blocks, lookaheads, pops_frag, pops_var, var_steps, var_pushed,
                                       id_reads, kept, sa_waves, sa_lf_steps, sa_dep_steps, lq_tops, lq_slots; };
extern thread_local KjEmuStats kj_emu_stats;
#endif
// get_suffix (bwt.c:105-121) reduced to the taxon of the sequence the suffix lies in
// get_suffix (bwt.c:105-121): entry of the sampled suffix array (is_seq = false) or sequence number (walk ended on a terminator)
template <class IdxT>
static KJ_DEV uint64_t kj_sa_locate(const KjDevIndex& ix, uint64_t k, bool& is_seq) {
    uint32_t c = 1;
    KJ_ROLLED
    while (c != 0 && (k & ix.sa_check)) {
        if constexpr (KjIsCompact<IdxT>::v) { const bool q = k >= ix.quirk_lo; k = kj_clf(ix, k, c); if (q) k -= ix.quirk_d[c]; }
        else if constexpr (KjIsTiered<IdxT>::v) { const bool q = k >= ix.quirk_lo; k = kj_clf<KJ_CREC_TIER>(ix, k, c); if (q) k -= ix.quirk_d[c]; }
        else if constexpr (KjIsSpread<IdxT>::v) { const bool q = k >= ix.quirk_lo; k = kj_clf<KJ_CREC_SPREAD>(ix, k, c); if (q) k -= ix.quirk_d[c]; }
        else { c = kj_letter(ix, k); const bool q = k >= ix.quirk_lo; k = (uint64_t)kj_rank<IdxT>(ix, c, (IdxT)k); if (q) k -= ix.quirk_d[c]; }
#if defined(KJ_EMU)
        kj_emu_stats.sa_lf_steps++;
#endif
    }
    is_seq = c == 0;
    return is_seq ? k : (uint64_t)((int64_t)(k >> ix.sa_exp) - ix.sa_bias);
}
template <class IdxT>
static KJ_DEV uint32_t kj_sa_taxon(const KjDevIndex& ix, uint64_t k) {
    bool is_seq; const uint64_t e = kj_sa_locate<IdxT>(ix, k, is_seq);
    return is_seq ? ix.seq_tax[e] : ix.sa_tax[e];
}
// entry k of the dense row -> taxon array (kj_bld_row_tax): the walk's taxon.  Rows [0, C[1]) hold the suffixes that start with a terminator: no
// match interval contains them and no walk passes through them (an LF step onto a terminator ends the walk), and the sampled ones among them
// lie below the first suffix-array entry, so they have no taxon.
template <class IdxT>
static KJ_DEV uint32_t kj_row_taxon(const KjDevIndex& ix, uint64_t k) { return k < ix.C[1] ? KJ_TAX_BAD : kj_sa_taxon<IdxT>(ix, k); }

// ---------------------------------------------------------------------------------------------
// Backward-search chains (the inner loops of greedyExact / maxMatches, bwt.c:267-275, 355-363).
// One lane owns the chain of one end position j.  A chain is run in two phases so that the many chains that die
// after ~log20(N) letters are handled at full warp width and only real matches are followed to their end:
//   phase A: k-mer table look-up (first k letters in one access; exactness-preserving because callers only use
//            chains with l >= Lmin >= k, and for j >= k an empty k-mer interval implies a match start >= 2, so the
//            `i<=1` break cannot be affected) followed by a few single steps, all lanes together;
//   phase B: the surviving chains are completed a few at a time in descending j, replaying the reference's
//            sequential rules (growing L, `if (i<=1) break`) between groups.
// ---------------------------------------------------------------------------------------------
#define KJ_PHASE_A_LETTERS 9      // letters matched in phase A (k-mer + single steps)
// chain state: OPEN = alive but not finished (phase-A survivor); EXACT = finished, i = leftmost start of the match ending at j and
// [lo,hi) its interval; KDEAD = failed inside the k-mer look-up: the match is shorter than k letters, its start lies in [j-k+2, j+1]
#define KJ_ST_OPEN 0
#define KJ_ST_EXACT 1
#define KJ_ST_KDEAD 2
template <class IdxT> struct KjChain { IdxT lo, hi; int i; int st; };

template <class IdxT>
static KJ_DEV void kj_chain_start(const KjDevIndex& ix, const uint8_t* frag, int j, uint32_t Lmin, KjChain<IdxT>& ch) {
    const int k = ix.kmer_k; int i = j; int budget = KJ_PHASE_A_LETTERS - 1;
    ch.st = KJ_ST_OPEN;
    if (k > 0 && j >= k && Lmin >= (uint32_t)k) {
        uint32_t idx = 0;
        KJ_ROLLED
        for (int t = 0; t < k; t++) idx = idx * 20u + (uint32_t)(frag[j - t] - 1u);
        IdxT lo, hi;
        if (sizeof(IdxT) == 4) { const KjKmer32 e = ((const KjKmer32*)ix.kmer)[idx]; lo = (IdxT)e.lo; hi = (IdxT)e.hi; }
        else { const KjKmer e = ((const KjKmer*)ix.kmer)[idx]; lo = (IdxT)e.lo; hi = (IdxT)e.hi; }
        if (lo >= hi) { ch.lo = 0; ch.hi = 0; ch.i = j + 1; ch.st = KJ_ST_KDEAD; return; }       // failed inside the k-mer: reported as length 0
        ch.lo = lo; ch.hi = hi; i = j - k + 1; budget = KJ_PHASE_A_LETTERS - k;
    } else {
        const uint32_t c = frag[j]; ch.lo = (IdxT)ix.C[c]; ch.hi = (IdxT)ix.C[c + 1];      // InitialSI (bwt.c:146-152)
    }
    KJ_ROLLED
    while (i > 0 && budget > 0) { if (!kj_update_si<IdxT>(ix, frag[i - 1], ch.lo, ch.hi)) { ch.st = KJ_ST_EXACT; break; } i--; budget--; }
    if (i == 0) ch.st = KJ_ST_EXACT;
    ch.i = i;
}
template <class IdxT>
static KJ_DEV void kj_chain_finish(const KjDevIndex& ix, const uint8_t* frag, KjChain<IdxT>& ch) {
    int i = ch.i;
    KJ_ROLLED
    while (i > 0) { if (!kj_update_si<IdxT>(ix, frag[i - 1], ch.lo, ch.hi)) break; i--; }
    ch.i = i; ch.st = KJ_ST_EXACT;
}
// complete the selected chains (one lane each)
template <class IdxT>
static KJ_DEV void kj_finish_selected(const Warp& w, const KjDevIndex& ix, const uint8_t* frag, bool sel, KjChain<IdxT>& ch) {
#if defined(KJ_EMU)
    const int i0 = ch.i;
#endif
    if (sel) kj_chain_finish<IdxT>(ix, frag, ch);
    w.sync();
#if defined(KJ_EMU)
    { const uint32_t st = sel ? (uint32_t)(i0 - ch.i) + 1u : 0u; const uint32_t mx = warp_max_u32(w, st); const uint32_t nsel = (uint32_t)kj_popc(w.ballot(sel));
      uint32_t sum = st; for (int m = 16; m > 0; m >>= 1) sum += w.shfl_xor(sum, m);
      if (w.lane == 0) { kj_emu_stats.rounds++; kj_emu_stats.round_steps += mx; kj_emu_stats.lane_steps += sum; kj_emu_stats.chains += nsel; } }
#endif
}

// ---------------------------------------------------------------------------------------------
// Which open chains of a block have to be completed at all?  On a true FM index the leftmost match start i_j is
// monotone in the end position (item[i..j+1] occurs => item[i..j] occurs, so i_j <= i_{j+1}).  Every chain that ENDED below
// an open chain therefore bounds its start from below: an exact chain j' < j gives i_j >= i_j', a chain that failed inside the
// k-mer gives i_j >= j'-k+2.  lb = that bound from the nearest ended chain below (it is the largest one), taken from this block or
// from the phase-A results of the next lower block (lb_ext).  With lb, many open chains are provably irrelevant without running
// them (their match cannot reach the current L / cannot start left of an already recorded match, and lb >= 2 excludes the
// `i<=1` break), which is exact: skipped chains are the ones whose result the reference computes and then discards.
// The reference's checkpoint quirk (bwtlen = m * 2^16) breaks the monotonicity; such indexes run with ix.mono = 0 (no bounds).
// ---------------------------------------------------------------------------------------------
template <class IdxT>
static KJ_DEV int kj_chain_lbval(const KjChain<IdxT>& ch, int j, int kk) { return ch.st == KJ_ST_EXACT ? ch.i : (j - kk + 2 > 0 ? j - kk + 2 : 0); }
template <class IdxT>
static KJ_DEV int kj_chain_lb(const Warp& w, const KjChain<IdxT>& ch, bool ran, int j, int kk, int lb_ext) {
    const uint32_t inf = w.ballot(ran && ch.st != KJ_ST_OPEN);
    const uint32_t below = w.lane < 31 ? inf & ~((2u << w.lane) - 1u) : 0u;
    const int v = w.shfl(kj_chain_lbval<IdxT>(ch, j, kk), below ? kj_ffs(below) - 1 : 0);
    return below ? v : lb_ext;
}
// the bound a block hands to the block above it: lbval of its first ended chain (0 if it has none)
template <class IdxT>
static KJ_DEV int kj_block_lb_ext(const Warp& w, const KjChain<IdxT>& ch, bool ran, int j, int kk) {
    const uint32_t inf = w.ballot(ran && ch.st != KJ_ST_OPEN);
    const int v = w.shfl(kj_chain_lbval<IdxT>(ch, j, kk), inf ? kj_ffs(inf) - 1 : 0);
    return inf ? v : 0;
}
// exclusive prefix maximum / minimum over the lanes (lane 0 gets `init`)
static KJ_DEV uint32_t kj_prefix_max_excl(const Warp& w, uint32_t v, uint32_t init) {
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = w.shfl(v, w.lane - d); if (w.lane >= d && o > v) v = o; }
    const uint32_t e = w.shfl(v, w.lane - 1);
    return w.lane == 0 ? init : (e > init ? e : init);
}
static KJ_DEV uint32_t kj_prefix_min_excl(const Warp& w, uint32_t v, uint32_t init) {
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = w.shfl(v, w.lane - d); if (w.lane >= d && o < v) v = o; }
    const uint32_t e = w.shfl(v, w.lane - 1);
    return w.lane == 0 ? init : (e < init ? e : init);
}
#define KJ_GROUP_LATE 8            // chains completed per round once the first round (segment tops only) did not settle a block

// ---------------------------------------------------------------------------------------------
// fragment queue (std::multimap<unsigned,Fragment*,greater>, ConsumerThread.hpp:83): highest key first,
// FIFO among equal keys.  key64 = val<<32 | (0xffffff-order)<<8 | 1  (0 = free slot); payload =
// arr(2) segchecked(1) start(15) len(14).  Originals get order = arr<<16 | scan position (their
// insertion order, ConsumerThread.cpp:196-268); SEG pieces and greedy variants take a running counter.
// ---------------------------------------------------------------------------------------------
// Long kernels: key64 = val<<40 | (0xffffffff-order)<<8 | 1 (a score is below 2^22); payload = arr(2) segchecked(1) . start(21 of the high
// word) | len(32); originals get order = arr<<22 | scan position, so late entries start at 2^24.
#define KJ_ORDER_LATE (1u << 20)
#define KJ_ORDER_LATE_LONG (1u << 24)
template <bool LONG = false>
struct KjQueue { uint64_t* key; typename KjW<LONG>::pay* pay; uint8_t* ord; uint32_t cap, n, late, next, nsorted; bool dirty; };    // scalars: uniform
template <bool LONG = false>
static KJ_DEV uint64_t kj_qkey(uint32_t val, uint32_t order) {
    if constexpr (LONG) return ((uint64_t)val << 40) | ((uint64_t)(0xffffffffu - order) << 8) | 1ull;
    else return ((uint64_t)val << 32) | ((uint64_t)(0xffffffu - order) << 8) | 1ull;
}
template <bool LONG = false>
static KJ_DEV uint32_t kj_qval(uint64_t key) { return (uint32_t)(key >> (LONG ? 40 : 32)); }
template <bool LONG = false>
static KJ_DEV typename KjW<LONG>::pay kj_qpay(uint32_t arr, bool segchecked, uint32_t start, uint32_t len) {
    if constexpr (LONG) return ((uint64_t)((arr << 30) | ((segchecked ? 1u : 0u) << 29) | start) << 32) | len;
    else return (arr << 30) | ((segchecked ? 1u : 0u) << 29) | (start << 14) | len;
}
template <bool LONG>
static KJ_DEV void kj_qpay_dec(typename KjW<LONG>::pay p, uint32_t& arr, bool& segchecked, uint32_t& start, uint32_t& len) {
    if constexpr (LONG) { const uint32_t hi = (uint32_t)((uint64_t)p >> 32); arr = hi >> 30; segchecked = (hi >> 29) & 1u; start = hi & 0x1fffffffu; len = (uint32_t)p; }
    else { arr = p >> 30; segchecked = (p >> 29) & 1u; start = (p >> 14) & 0x7fffu; len = p & 0x3fffu; }
}
// long kernels: insertion order of a fragment of array a, closed by the stop before scan position pos (< 2^21) or the leftover of a frame
static KJ_DEV uint32_t kj_frag_order_long(uint32_t a, bool leftover, uint32_t frame, uint32_t pos) { return (a << 22) | (leftover ? (1u << 21) + frame : pos); }

// emit from several lanes at once (emit predicate per lane)
template <bool LONG = false>
static KJ_DEV void kj_queue_emit(KjWarpCtx& cx, KjQueue<LONG>& q, bool emit, uint32_t val, uint32_t order, typename KjW<LONG>::pay pay) {
    uint32_t mask = cx.w.ballot(emit);
    if (!mask) return;
    uint32_t cnt = (uint32_t)kj_popc(mask);
    if (q.n + cnt > q.cap) { if (cx.w.lane == 0) kj_flag_error(cx, 1u); return; }
    if (emit) { uint32_t s = q.n + (uint32_t)kj_popc(mask & lanemask_lt(cx.w.lane)); q.key[s] = kj_qkey<LONG>(val, order); q.pay[s] = pay; }
    q.n += cnt;
}
// Long kernels: the fragments of a long read (tens of thousands) are sorted once, keys and payloads together, by a warp bitonic sort in the work
// space: O(n log^2 n / 32) steps, and every comparator takes the larger key to the lower index, so the missing elements of the next power of two
// act as zero keys at the end and their comparators are skipped.  Afterwards [0, nsorted) is in pop order; entries pushed later (SEG pieces,
// KJ_ORDER_LATE_LONG and above) are appended behind it and found by a scan over the live late entries only (kj_queue_top_long; a popped one is
// replaced by the last).
static KJ_DEV void kj_queue_rank_long(KjWarpCtx& cx, KjQueue<true>& q) {
    cx.w.sync();
    const uint32_t n = q.n; uint32_t np = 1; while (np < n) np <<= 1;
    KJ_ROLLED
    for (uint32_t k = 2; k <= np; k <<= 1) {
        KJ_ROLLED
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            KJ_ROLLED
            for (uint32_t t = (uint32_t)cx.w.lane; t < np / 2; t += 32) {
                uint32_t i, p;
                if (j == k >> 1) { const uint32_t b = t / j, o = t - b * j; i = b * k + o; p = b * k + k - 1u - o; }     // first step of a merge: mirrored pairs
                else { const uint32_t b = t / j, o = t - b * j; i = b * 2u * j + o; p = i + j; }
                if (p < n) {
                    const uint64_t ki = q.key[i], kp = q.key[p];
                    if (ki < kp) { q.key[i] = kp; q.key[p] = ki; const uint64_t x = q.pay[i]; q.pay[i] = q.pay[p]; q.pay[p] = x; }
                }
            }
            cx.w.sync();
        }
    }
    q.nsorted = n; q.next = 0; q.dirty = false;
}
// the top entry of a long read's queue: the head of the sorted run or the largest late entry.  Returns its key (0: empty) and slot (uniform).
// min_val only grows over a read (MEM's longest, Greedy's best score): late entries below it can never be popped, and the scan drops them.
static KJ_DEV uint64_t kj_queue_top_long(KjWarpCtx& cx, KjQueue<true>& q, uint32_t& slot, uint32_t min_val) {
#if defined(KJ_EMU)
    if (cx.w.lane == 0) { kj_emu_stats.lq_tops++; kj_emu_stats.lq_slots += 1u + (q.n - q.nsorted); }
#endif
    const uint64_t ks = q.next < q.nsorted ? q.key[q.next] : 0ull;
    slot = q.next;
    if (q.n == q.nsorted) return ks;
    cx.w.sync();
    uint64_t best = 0; uint32_t bs = 0, out = q.nsorted;
    KJ_ROLLED
    for (uint32_t b = q.nsorted; b < q.n; b += 32) {
        const uint32_t s = b + (uint32_t)cx.w.lane; uint64_t k = 0, p = 0;
        if (s < q.n) { k = q.key[s]; p = q.pay[s]; }
        const bool live = s < q.n && kj_qval<true>(k) >= min_val; const uint32_t m = cx.w.ballot(live);
        cx.w.sync();
        if (live) { const uint32_t d = out + (uint32_t)kj_popc(m & lanemask_lt(cx.w.lane)); q.key[d] = k; q.pay[d] = p; if (k > best) { best = k; bs = d; } }
        out += (uint32_t)kj_popc(m);
    }
    q.n = out;
    cx.w.sync();
    const uint64_t g = warp_max_u64(cx.w, best);
    if (g <= ks) return ks;
    slot = cx.w.shfl(bs, kj_ffs(cx.w.ballot(best == g)) - 1);
    return g;
}
// remove the entry kj_queue_top_long returned and return its payload
static KJ_DEV uint64_t kj_queue_take_long(KjWarpCtx& cx, KjQueue<true>& q, uint32_t slot) {
    const uint64_t p = q.pay[slot];
    if (slot < q.nsorted) { q.next++; return p; }
    cx.w.sync();
    if (cx.w.lane == 0) { q.key[slot] = q.key[q.n - 1]; q.pay[slot] = q.pay[q.n - 1]; }      // the late entries stay packed: a scan reads live ones only
    q.n--;
    cx.w.sync();
    return p;
}
// After translation the fragments are ranked once (keys are unique): ord[k] = slot of the k-th entry in pop order.  As long as
// no SEG piece has been pushed (rare) a pop is three broadcast shared-memory reads instead of a warp arg-max.
static KJ_DEV void kj_queue_sort(KjWarpCtx& cx, KjQueue<>& q) {
    cx.w.sync();
    KJ_ROLLED
    for (uint32_t i = (uint32_t)cx.w.lane; i < q.n; i += 32) {
        const uint64_t mine = q.key[i]; uint32_t rank = 0;
        KJ_ROLLED
        for (uint32_t j = 0; j < q.n; j++) rank += q.key[j] > mine ? 1u : 0u;
        q.ord[rank] = (uint8_t)i;
    }
    q.nsorted = q.n <= 255u ? q.n : 0u; q.next = 0; q.dirty = q.n > 255u;
    cx.w.sync();
}
// pop the top entry if its sort value is >= min_val (getNextFragment's gate, ConsumerThread.cpp:276-283)
template <bool LONG = false>
static KJ_DEV bool kj_queue_pop(KjWarpCtx& cx, KjQueue<LONG>& q, uint32_t min_val, uint32_t& val, typename KjW<LONG>::pay& pay) {
    if constexpr (LONG) {
        uint32_t slot; const uint64_t g = kj_queue_top_long(cx, q, slot, min_val);
        if (g == 0) return false;
        val = kj_qval<true>(g);
        if (val < min_val) return false;
        pay = kj_queue_take_long(cx, q, slot);
        return true;
    }
    if (!q.dirty) {
        if (q.next >= q.nsorted) return false;
        const uint32_t slot = q.ord[q.next]; const uint64_t k = q.key[slot];
        val = (uint32_t)(k >> 32);
        if (val < min_val) return false;
        pay = q.pay[slot]; q.next++;
        return true;
    }
    cx.w.sync();
    uint64_t best = 0; uint32_t slot = 0;
    KJ_ROLLED
    for (uint32_t s = (uint32_t)cx.w.lane; s < q.n; s += 32) { uint64_t k = q.key[s]; if (k > best) { best = k; slot = s; } }
    uint64_t g = warp_max_u64(cx.w, best);
    if (g == 0) return false;
    val = (uint32_t)(g >> 32);
    if (val < min_val) return false;
    uint32_t own = cx.w.ballot(best == g);
    int src = kj_ffs(own) - 1;
    uint32_t p = 0;
    if (cx.w.lane == src) { p = q.pay[slot]; q.key[slot] = 0; }
    pay = cx.w.shfl(p, src);
    cx.w.sync();
    return true;
}
// switch to scanning pops (a SEG piece is about to be pushed): consumed entries of the sorted prefix are cleared first
static KJ_DEV void kj_queue_make_dirty(KjWarpCtx& cx, KjQueue<>& q) {
    if (q.dirty) return;
    cx.w.sync();
    KJ_ROLLED
    for (uint32_t k = (uint32_t)cx.w.lane; k < q.next; k += 32) q.key[q.ord[k]] = 0;
    q.dirty = true;
    cx.w.sync();
}

// ---------------------------------------------------------------------------------------------
// six-frame translation + stop splitting of one mate  (getAllFragmentsBits, ConsumerThread.cpp:190-270)
// arrays: aa[2*mate+0][count] forward codon starting at base `count`; aa[2*mate+1][r] reverse-strand codon
// in the reference's scan order (r = n-3-count), so every frame is a stride-3 walk in array order.
// ---------------------------------------------------------------------------------------------
static KJ_DEV uint32_t kj_nuc(uint8_t ch) {          // nuc2int (ConsumerThread.cpp:32-37): A0 C1 G2 T/U3, else invalid
    uint32_t u = ch & 0xDFu;
    return u == 'A' ? 0u : u == 'C' ? 1u : u == 'G' ? 2u : (u == 'T' || u == 'U') ? 3u : 4u;
}
// fragments = maximal stop-free runs of every frame (a stride-3 walk of an array); na1/na2 = array lengths of the two mates
// (0 = mate absent), nframes = 3 for translated DNA, 1 for protein input (one "frame" whose residues sit at indices 3e).
template <bool LONG = false>
static KJ_DEV void kj_split_frames(KjWarpCtx& cx, KjQueue<LONG>& q, const int na1, const int na2, const int n1, const int n2, const bool greedy, const int nframes) {
    const Warp& w = cx.w; const KjTables& tb = *cx.tb;
    const uint8_t* aa = cx.smem + cx.L.aa_off; const uint32_t st = cx.L.aa_stride;
    // fragments = maximal stop-free runs of every frame (a stride-3 walk of an array).  Per frame the stop positions
    // become a bit mask (ballot), so each lane finds "am I the last residue of a run, and where does it start" with bit
    // operations instead of a serial scan.  Insertion order (ConsumerThread.cpp:196-268): runs closed by a stop in scan
    // order of that stop; leftovers afterwards in frame order 0,1,2 where frame = count % 3 in FORWARD coordinates.
    const uint32_t m = cx.rp->m;
    KJ_ROLLED
    for (int r = 0; r < nframes; r++) {
        const int ne1 = (na1 - r + 2) / 3, ne2 = (na2 - r + 2) / 3;      // elements e: array index r + 3e
        const int nemax = ne1 > ne2 ? ne1 : ne2;
        int run_open[4] = {0, 0, 0, 0};                                  // first element after the last stop of the earlier chunks (uniform)
        uint32_t p_open[4] = {0, 0, 0, 0}, p_carry[4] = {0, 0, 0, 0};    // greedy: score prefix at run_open-1 / at the end of the previous chunk (uniform)
        KJ_ROLLED
        for (int e0 = 0; e0 < nemax; e0 += 32) {
            const int e = e0 + w.lane;
            bool in[4], stop[4]; uint32_t sm[4], pre[4];
            #pragma unroll
            for (int a = 0; a < 4; a++) {
                const int ne = (nframes == 1 && (a & 1)) ? 0 : (a < 2 ? ne1 : ne2); in[a] = e < ne;
                const uint32_t c = in[a] ? aa[(uint32_t)a * st + (uint32_t)(r + 3 * e)] : 0u;
                stop[a] = in[a] && c == 0; pre[a] = (greedy && in[a]) ? (uint32_t)tb.b62[c][c] : 0u;     // BLOSUM62 diagonal (calcScore, 415-421); b62[0][0] = 0
            }
            #pragma unroll
            for (int a = 0; a < 4; a++) sm[a] = w.ballot(stop[a]);
            if (greedy) {
                // fragment self-scores = differences of a running prefix sum over the frame (four independent scans interleaved)
                for (int d = 1; d < 32; d <<= 1) {
                    #pragma unroll
                    for (int a = 0; a < 4; a++) { const uint32_t o = w.shfl(pre[a], w.lane - d); if (w.lane >= d) pre[a] += o; }
                }
                #pragma unroll
                for (int a = 0; a < 4; a++) pre[a] += p_carry[a];
            }
            #pragma unroll
            for (int a = 0; a < 4; a++) {
                const int ne = (nframes == 1 && (a & 1)) ? 0 : (a < 2 ? ne1 : ne2); const int n = a < 2 ? n1 : n2; const uint8_t* A = aa + (uint32_t)a * st;
                if (e0 < ne) {                                           // uniform
                    // a run ends at e if e is a residue and e+1 is a stop or the end
                    const bool is_res = in[a] && !stop[a];
                    const bool next_stop = (e + 1 >= ne) || (w.lane < 31 ? ((sm[a] >> (w.lane + 1)) & 1u) != 0 : A[r + 3 * (e + 1)] == 0);
                    const bool is_end = is_res && next_stop;
                    const uint32_t below = sm[a] & lanemask_lt(w.lane);
                    const int prev_stop_lane = below ? 31 - kj_clz(below) : 0;
                    uint32_t p_before = 0;
                    if (greedy) { p_before = w.shfl(pre[a], prev_stop_lane); if (!below) p_before = p_open[a]; }    // prefix at the element before the run
                    uint32_t run_start = 0, run_len = 0, run_score = 0;
                    if (is_end) {
                        const int s = below ? e0 + prev_stop_lane + 1 : run_open[a];    // first element after the previous stop
                        run_start = (uint32_t)(r + 3 * s); run_len = (uint32_t)(e - s + 1);
                        run_score = pre[a] - p_before;
                    }
                    const bool leftover = e + 1 >= ne;
                    const int frame = (a & 1) ? (((n - 3 - r) % 3) + 3) % 3 : r;
                    uint32_t order;
                    if constexpr (LONG) order = kj_frag_order_long((uint32_t)a, leftover, (uint32_t)frame, (uint32_t)(r + 3 * (e + 1)));
                    else order = ((uint32_t)a << 16) | (leftover ? 40000u + (uint32_t)frame : (uint32_t)(r + 3 * (e + 1)));
                    const bool emit = is_end && run_len >= m && (!greedy || run_score >= cx.rp->min_score);
                    kj_queue_emit<LONG>(cx, q, emit, greedy ? run_score : run_len, order, kj_qpay<LONG>((uint32_t)a, false, run_start, run_len));
                    if (sm[a]) { const int last = 31 - kj_clz(sm[a]); run_open[a] = e0 + last + 1; if (greedy) p_open[a] = w.shfl(pre[a], last); }
                    if (greedy) p_carry[a] = w.shfl(pre[a], 31);
                }
            }
        }
    }
}

// The same splitting with the four arrays one after the other (one copy of the run logic instead of four interleaved ones: a quarter of the code).
// Greedy only: there the instruction cache, not the dependent latency of this step, is the scarce resource (see kj_warp.h).  The
// queue slots are filled in another order; the keys (value, reference insertion order) are the same, and only they decide the pop order.
template <bool LONG = false>
static KJ_DEV void kj_split_frames_rolled(KjWarpCtx& cx, KjQueue<LONG>& q, const int na1, const int na2, const int n1, const int n2, const bool greedy, const int nframes) {
    const Warp& w = cx.w; const KjTables& tb = *cx.tb;
    const uint8_t* aa = cx.smem + cx.L.aa_off; const uint32_t st = cx.L.aa_stride;
    const uint32_t m = cx.rp->m;
    KJ_ROLLED
    for (int ra = 0; ra < 4 * nframes; ra++) {
        const int r = ra >> 2, a = ra & 3;
        const int ne = (nframes == 1 && (a & 1)) ? 0 : ((a < 2 ? na1 : na2) - r + 2) / 3;      // elements e: array index r + 3e
        const int n = a < 2 ? n1 : n2; const uint8_t* A = aa + (uint32_t)a * st;
        const int frame = (a & 1) ? (((n - 3 - r) % 3) + 3) % 3 : r;
        int run_open = 0; uint32_t p_open = 0, p_carry = 0;                                    // uniform: first element after the last stop / score prefix there / at the end of the previous chunk
        KJ_ROLLED
        for (int e0 = 0; e0 < ne; e0 += 32) {
            const int e = e0 + w.lane; const bool in = e < ne;
            const uint32_t c = in ? A[r + 3 * e] : 0u;
            const bool stop = in && c == 0; uint32_t pre = (greedy && in) ? (uint32_t)tb.b62[c][c] : 0u;
            const uint32_t sm = w.ballot(stop);
            if (greedy) {
                KJ_ROLLED
                for (int d = 1; d < 32; d <<= 1) { const uint32_t o = w.shfl(pre, w.lane - d); if (w.lane >= d) pre += o; }
                pre += p_carry;
            }
            const bool is_res = in && !stop;
            const bool next_stop = (e + 1 >= ne) || (w.lane < 31 ? ((sm >> (w.lane + 1)) & 1u) != 0 : A[r + 3 * (e + 1)] == 0);
            const bool is_end = is_res && next_stop;
            const uint32_t below = sm & lanemask_lt(w.lane);
            const int prev_stop_lane = below ? 31 - kj_clz(below) : 0;
            uint32_t p_before = 0;
            if (greedy) { p_before = w.shfl(pre, prev_stop_lane); if (!below) p_before = p_open; }
            uint32_t run_start = 0, run_len = 0, run_score = 0;
            if (is_end) {
                const int s = below ? e0 + prev_stop_lane + 1 : run_open;
                run_start = (uint32_t)(r + 3 * s); run_len = (uint32_t)(e - s + 1);
                run_score = pre - p_before;
            }
            const bool leftover = e + 1 >= ne;
            uint32_t order;
            if constexpr (LONG) order = kj_frag_order_long((uint32_t)a, leftover, (uint32_t)frame, (uint32_t)(r + 3 * (e + 1)));
            else order = ((uint32_t)a << 16) | (leftover ? 40000u + (uint32_t)frame : (uint32_t)(r + 3 * (e + 1)));
            const bool emit = is_end && run_len >= m && (!greedy || run_score >= cx.rp->min_score);
            kj_queue_emit<LONG>(cx, q, emit, greedy ? run_score : run_len, order, kj_qpay<LONG>((uint32_t)a, false, run_start, run_len));
            if (sm) { const int last = 31 - kj_clz(sm); run_open = e0 + last + 1; if (greedy) p_open = w.shfl(pre, last); }
            if (greedy) p_carry = w.shfl(pre, 31);
        }
    }
}

// Both mates are translated and split in the SAME loops (array a = 2*mate + strand): the four arrays are independent, so
// their load/ballot/bit-twiddling chains overlap instead of running back to back (the kernel is bound by dependent latency).
template <bool LONG = false>
static KJ_DEV void kj_translate_pair(KjWarpCtx& cx, KjQueue<LONG>& q, const uint8_t* s1, int n1, bool do1, const uint8_t* s2, int n2, bool do2, bool greedy, const bool small_code) {
    const Warp& w = cx.w; const KjTables& tb = *cx.tb;
    uint8_t* aa = cx.smem + cx.L.aa_off; const uint32_t st = cx.L.aa_stride;
    const int na1 = do1 ? n1 - 2 : 0, na2 = do2 ? n2 - 2 : 0;
    const int namax = na1 > na2 ? na1 : na2;
    // 30 codon positions per pass: every lane decodes ONE base per mate, its two successors come from the next lanes
    KJ_ROLLED
    for (int b = 0; b < namax; b += 30) {
        const int pos = b + w.lane;
        const uint32_t x0 = (do1 && pos < n1) ? kj_nuc(s1[pos]) : 4u, y0 = (do2 && pos < n2) ? kj_nuc(s2[pos]) : 4u;
        const uint32_t x1 = w.shfl(x0, w.lane + 1), x2 = w.shfl(x0, w.lane + 2), y1 = w.shfl(y0, w.lane + 1), y2 = w.shfl(y0, w.lane + 2);
        if (w.lane < 30) {
            if (pos < na1) {
                const bool ok = (x0 | x1 | x2) < 4u;
                aa[pos] = ok ? tb.codon_aa[x0 << 4 | x1 << 2 | x2] : (uint8_t)0;
                aa[st + (uint32_t)(na1 - 1 - pos)] = ok ? tb.codon_aa[(3u - x2) << 4 | (3u - x1) << 2 | (3u - x0)] : (uint8_t)0;
            }
            if (pos < na2) {
                const bool ok = (y0 | y1 | y2) < 4u;
                aa[2u * st + (uint32_t)pos] = ok ? tb.codon_aa[y0 << 4 | y1 << 2 | y2] : (uint8_t)0;
                aa[3u * st + (uint32_t)(na2 - 1 - pos)] = ok ? tb.codon_aa[(3u - y2) << 4 | (3u - y1) << 2 | (3u - y0)] : (uint8_t)0;
            }
        }
    }
    w.sync();
    if (small_code) kj_split_frames_rolled<LONG>(cx, q, na1, na2, n1, n2, greedy, 3);      // Greedy is faster with the quarter-size splitting code (A/B)
    else kj_split_frames<LONG>(cx, q, na1, na2, n1, n2, greedy, 3);
}

// copy the characters of item (arr,start,len) into the contiguous fragment buffer
static KJ_DEV void kj_load_frag(KjWarpCtx& cx, uint32_t arr, uint32_t start, uint32_t len) {
    const uint8_t* A = cx.smem + cx.L.aa_off + arr * cx.L.aa_stride;
    uint8_t* frag = cx.smem + cx.L.frag_off;
    KJ_ROLLED
    for (uint32_t t = (uint32_t)cx.w.lane; t < len; t += 32) frag[t] = A[start + 3u * t];
    cx.w.sync();
}

// ---------------------------------------------------------------------------------------------
// SEG low-complexity filter (SeqBufferSeg with SegParametersNewAa + overlaps, blast_seg.c:2027-2332)
// on frag[0..n).  Output: ascending [begin,end] regions in the segs array; returns their number.
// ---------------------------------------------------------------------------------------------
struct KjSeg { int begin, end; };
#define KJ_SEG_DOWNSET 5      // (window+1)/2 - 1
#define KJ_SEG_UPSET 7        // window - downset
#define KJ_SEG_MAXTRIM 50

// entropy class of every 12-window: bit0 = H <= locut, bit1 = H <= hicut   (s_SeqEntropy/s_Entropy, 1596-1798).
// A window with >= 8 distinct residues has H >= 2.617 > hicut (checked on the host over all partitions), so only the
// rare low-diversity windows need the composition count.  Returns whether any window can trigger SEG at all.
// packed variant: the 12 residues of a window live in three 32-bit words; per distinct residue (<= 7 on the slow path)
// the count is three byte-wise compares + popcounts instead of a 12-step nibble-counter loop
static KJ_DEV bool kj_seg_flags(KjWarpCtx& cx, int n, const bool compact) {
    const uint8_t* frag = cx.smem + cx.L.frag_off; uint8_t* hf = cx.smem + cx.L.hflag_off; const KjTables& tb = *cx.tb;
    bool any_low = false;
    KJ_ROLLED
    for (int p0 = 0; p0 + KJ_SEG_WINDOW <= n; p0 += 32) {
        const int p = p0 + cx.w.lane; uint32_t flags = 0;
        if (p + KJ_SEG_WINDOW <= n) {
            const uint32_t* aw = (const uint32_t*)(frag + (p & ~3)); const uint32_t sh = (uint32_t)(p & 3) * 8u;
            const uint32_t a0 = aw[0], a1 = aw[1], a2 = aw[2], a3 = aw[3];
            const uint32_t w0 = kj_funnel_r(a0, a1, sh), w1 = kj_funnel_r(a1, a2, sh), w2 = kj_funnel_r(a2, a3, sh);
            uint32_t seen = 0;
            // compact (rolled): faster for Greedy in an A/B run (with the unified update in kj_seg_trim), neutral for MEM
            if (compact) { KJ_ROLLED for (int t = 0; t < 4; t++) { seen |= 1u << ((w0 >> (8 * t)) & 0xffu); seen |= 1u << ((w1 >> (8 * t)) & 0xffu); seen |= 1u << ((w2 >> (8 * t)) & 0xffu); } }
            else for (int t = 0; t < 4; t++) { seen |= 1u << ((w0 >> (8 * t)) & 0xffu); seen |= 1u << ((w1 >> (8 * t)) & 0xffu); seen |= 1u << ((w2 >> (8 * t)) & 0xffu); }
            if (kj_popc(seen) < 8) {
                int32_t x = 0;
                KJ_ROLLED
                while (seen) {
                    const uint32_t a = (uint32_t)kj_ffs(seen) - 1u; seen &= seen - 1u;
                    const uint32_t a4 = a * 0x01010101u;
                    const uint32_t c = (uint32_t)(kj_popc(kj_vcmpeq4(w0, a4)) + kj_popc(kj_vcmpeq4(w1, a4)) + kj_popc(kj_vcmpeq4(w2, a4))) >> 3;
                    x += (int32_t)c * tb.seg_logfix[c];
                }
                flags = (x <= tb.seg_locut_fix ? 1u : 0u) | (x <= tb.seg_hicut_fix ? 2u : 0u);
            }
            hf[p] = (uint8_t)flags;
        }
        any_low = cx.w.any((flags & 1u) != 0) || any_low;
    }
    cx.w.sync();
    return any_low;
}

// s_Trim for regions longer than 127 residues (long reads / protein input).  Same search, but each lane keeps the
// composition of its sliding window as a descending-sorted count vector (the reference's state vector, s_StateOn
// 1628-1650): a count changes by +-1 per step, so the vector stays sorted by swapping the changed letter to the edge
// of its run of equal counts.  s_GetProb then walks the 20 sorted counts in the reference's order.
// (a real function, like kj_seg_trim: the trim search is large and rarely the warp's hot path -- inlined copies of it cost
// instruction-cache space in every kernel.  Returns best_start << 16 | best_end inside s[0..n2).)
// CntT: the count type (uint16_t; the long kernels' regions can exceed 65,535 residues: uint32_t, 3,840 of the scratch's >= 4,800 bytes);
// RetT, SH: the packing of the result (start << SH | end).
template <class CntT, class RetT, int SH>
static KJ_DEV RetT kj_seg_trim_long_t(const Warp w, uint8_t* scratch, const uint8_t* s, int n2, const double* lnf) {
    CntT* sv = (CntT*)scratch;                                        // [20][32] counts, descending per lane
    uint8_t* at = (uint8_t*)(sv + 20 * 32);                            // [20][32] letter stored at sorted position k
    uint8_t* where = at + 20 * 32;                                     // [20][32] sorted position of letter a
    int minlen = 1; if (n2 - KJ_SEG_MAXTRIM > minlen) minlen = n2 - KJ_SEG_MAXTRIM;
    const int nlens = n2 - minlen;
    double g_prob = 1.0; int g_lend = 0, g_rend = n2 - 1;            // uniform
    const int ln = w.lane;
    KJ_ROLLED
    for (int pass = 0; pass * 32 < nlens; pass++) {
        const int len = n2 - (pass * 32 + ln);
        const bool act = (pass * 32 + ln) < nlens;
        KJ_ROLLED
        for (int k = 0; k < 20; k++) { sv[k * 32 + ln] = 0; at[k * 32 + ln] = (uint8_t)k; where[k * 32 + ln] = (uint8_t)k; }
        double my_prob = 1.0; int my_i = 0;
        if (act) {
            #define KJ_SV_SWAP(p_, q_) { const uint32_t la_ = at[(p_) * 32 + ln], lb_ = at[(q_) * 32 + ln]; at[(p_) * 32 + ln] = (uint8_t)lb_; at[(q_) * 32 + ln] = (uint8_t)la_; \
                where[la_ * 32 + ln] = (uint8_t)(q_); where[lb_ * 32 + ln] = (uint8_t)(p_); }
            #define KJ_SV_ADD(letter) { const uint32_t a_ = (letter) - 1u; uint32_t p_ = where[a_ * 32 + ln]; const uint32_t v_ = sv[p_ * 32 + ln]; uint32_t q_ = p_; \
                while (q_ > 0 && sv[(q_ - 1) * 32 + ln] == v_) q_--; if (q_ != p_) KJ_SV_SWAP(p_, q_); sv[q_ * 32 + ln] = (CntT)(v_ + 1u); }
            #define KJ_SV_DEL(letter) { const uint32_t a_ = (letter) - 1u; uint32_t p_ = where[a_ * 32 + ln]; const uint32_t v_ = sv[p_ * 32 + ln]; uint32_t q_ = p_; \
                while (q_ < 19 && sv[(q_ + 1) * 32 + ln] == v_) q_++; if (q_ != p_) KJ_SV_SWAP(p_, q_); sv[q_ * 32 + ln] = (CntT)(v_ - 1u); }
            KJ_ROLLED
            for (int t = 0; t < len; t++) KJ_SV_ADD(s[t]);
            KJ_ROLLED
            for (int i = 0; i + len <= n2; i++) {
                // s_GetProb (1941-1962) = s_LnAss (1890-1930) + s_LnPerm (1865-1879) - len*ln20, same operation order
                double ans1 = lnf[20], ans2 = lnf[len];
                int k = 0;
                KJ_ROLLED
                while (k < 20) {
                    const uint32_t v = sv[k * 32 + ln];
                    int cls = 1; while (k + cls < 20 && sv[(k + cls) * 32 + ln] == v) cls++;
                    ans1 = kj_dsub(ans1, lnf[cls]);                   // one class of equal counts (the zero class included)
                    if (v) for (int rep = 0; rep < cls; rep++) ans2 = kj_dsub(ans2, lnf[v]);
                    k += cls;
                }
                double prob = kj_dsub(kj_dadd(ans1, ans2), kj_dmul((double)len, 2.9957322735539909));
                if (prob < my_prob) { my_prob = prob; my_i = i; }
                if (i + len < n2) { KJ_SV_DEL(s[i]); KJ_SV_ADD(s[i + len]); }
            }
            #undef KJ_SV_ADD
            #undef KJ_SV_DEL
            #undef KJ_SV_SWAP
        }
        w.sync();
        double mn = my_prob;
        for (int mm = 16; mm > 0; mm >>= 1) { double o = w.shfl_d(mn, w.lane ^ mm); mn = o < mn ? o : mn; }
        if (mn < g_prob) {
            int src = kj_ffs(w.ballot(my_prob == mn)) - 1;
            int wi = w.shfl(my_i, src); int wlen = n2 - (pass * 32 + src);
            g_prob = mn; g_lend = wi; g_rend = wlen + wi - 1;
        }
    }
    return ((RetT)g_lend << SH) | (RetT)g_rend;
}
KJ_NOINLINE uint32_t kj_seg_trim_long(const Warp w, uint8_t* scratch, const uint8_t* s, int n2, const double* lnf) {
    return kj_seg_trim_long_t<uint16_t, uint32_t, 16>(w, scratch, s, n2, lnf);
}

// s_Trim (blast_seg.c:1971-2015): the sub-window of s[0..n2) with minimal s_GetProb; first in
// (len descending, start ascending) order wins ties.  One lane per window length, sliding start.
KJ_NOINLINE uint32_t kj_seg_trim(const Warp w, uint8_t* scratch, const uint8_t* s, int n2, const double* lnf) {
    if (n2 > 127) return kj_seg_trim_long(w, scratch, s, n2, lnf);
    uint8_t* cnt = scratch;                         // [20][32]
    uint8_t* hist = scratch + 20u * 32u;            // [n2+1][32] number of letters having count v
    int minlen = 1; if (n2 - KJ_SEG_MAXTRIM > minlen) minlen = n2 - KJ_SEG_MAXTRIM;
    const int nlens = n2 - minlen;
    double g_prob = 1.0; int g_lend = 0, g_rend = n2 - 1;            // uniform
    KJ_ROLLED
    for (int pass = 0; pass * 32 < nlens; pass++) {
        const int len = n2 - (pass * 32 + w.lane);
        const bool act = (pass * 32 + w.lane) < nlens;
        KJ_ROLLED
        for (int a = 0; a < 20; a++) cnt[a * 32 + w.lane] = 0;
        KJ_ROLLED
        for (int v = 0; v <= n2; v++) hist[v * 32 + w.lane] = 0;
        uint64_t m0 = 0, m1 = 0; int nz = 0;                          // bit v set <=> hist[v] > 0 (v < 128)
        double my_prob = 1.0; int my_i = 0;
        if (act) {
            #define KJ_SEG_ADD(letter) { uint32_t a_ = (letter) - 1u; uint32_t c_ = cnt[a_ * 32 + w.lane]; \
                if (c_ > 0) { uint8_t h_ = --hist[c_ * 32 + w.lane]; if (h_ == 0) { if (c_ < 64) m0 &= ~(1ull << c_); else m1 &= ~(1ull << (c_ - 64)); } } else nz++; \
                cnt[a_ * 32 + w.lane] = (uint8_t)(c_ + 1); hist[(c_ + 1) * 32 + w.lane]++; if (c_ + 1 < 64) m0 |= 1ull << (c_ + 1); else m1 |= 1ull << (c_ + 1 - 64); }
            KJ_ROLLED
            for (int t = 0; t < len; t++) KJ_SEG_ADD(s[t]);
            KJ_ROLLED
            for (int i = 0; i + len <= n2; i++) {
                // s_GetProb (1941-1962) = s_LnAss (1890-1930) + s_LnPerm (1865-1879) - len*ln20, same operation order
                double ans1 = lnf[20], ans2 = lnf[len];
                uint64_t a0 = m0, a1 = m1;
                KJ_ROLLED
                while (a0 | a1) {
                    int v;                                           // highest set bit of the 128-bit mask = next larger count
                    if (a1) { v = 64 + kj_hibit64(a1); a1 &= ~(1ull << (v - 64)); }
                    else { v = kj_hibit64(a0); a0 &= ~(1ull << v); }
                    int cls = hist[v * 32 + w.lane];
                    ans1 = kj_dsub(ans1, lnf[cls]);
                    KJ_ROLLED
                    for (int rep = 0; rep < cls; rep++) ans2 = kj_dsub(ans2, lnf[v]);
                }
                if (nz < 20) ans1 = kj_dsub(ans1, lnf[20 - nz]);
                double prob = kj_dsub(kj_dadd(ans1, ans2), kj_dmul((double)len, 2.9957322735539909));
                if (prob < my_prob) { my_prob = prob; my_i = i; }
                // one update body for "remove s[i]" and "add s[i+len]" (half the code of the two specialised ones)
                if (i + len < n2) {
                    KJ_ROLLED
                    for (int k_ = 0; k_ < 2; k_++) {
                        const uint32_t a_ = (uint32_t)(k_ ? s[i + len] : s[i]) - 1u; const uint32_t c_ = cnt[a_ * 32 + w.lane]; const uint32_t n_ = k_ ? c_ + 1u : c_ - 1u;
                        if (c_ > 0) { uint8_t h_ = --hist[c_ * 32 + w.lane]; if (h_ == 0) { if (c_ < 64) m0 &= ~(1ull << c_); else m1 &= ~(1ull << (c_ - 64)); } } else nz++;
                        cnt[a_ * 32 + w.lane] = (uint8_t)n_;
                        if (n_ > 0) { hist[n_ * 32 + w.lane]++; if (n_ < 64) m0 |= 1ull << n_; else m1 |= 1ull << (n_ - 64); } else nz--;
                    }
                }
            }
            #undef KJ_SEG_ADD
        }
        w.sync();
        // arg-min over lanes, lowest lane (longest window) wins ties
        double mn = my_prob;
        for (int mm = 16; mm > 0; mm >>= 1) { double o = w.shfl_d(mn, w.lane ^ mm); mn = o < mn ? o : mn; }
        if (mn < g_prob) {
            int src = kj_ffs(w.ballot(my_prob == mn)) - 1;
            int wi = w.shfl(my_i, src); int wlen = n2 - (pass * 32 + src);
            g_prob = mn; g_lend = wi; g_rend = wlen + wi - 1;
        }
    }
    return ((uint32_t)g_lend << 16) | (uint32_t)g_rend;
}
// the same for the long kernels: best_start << 32 | best_end
KJ_NOINLINE uint64_t kj_seg_trim_wide(const Warp w, uint8_t* scratch, const uint8_t* s, int n2, const double* lnf) {
    if (n2 > 127) return kj_seg_trim_long_t<uint32_t, uint64_t, 32>(w, scratch, s, n2, lnf);
    const uint32_t t = kj_seg_trim(w, scratch, s, n2, lnf);
    return ((uint64_t)(t >> 16) << 32) | (t & 0xffffu);
}

// s_SegSeq (blast_seg.c:2027-2113) on frag[s0 .. s0+n).  LEVEL 0 collects regions; LEVEL 1 is the
// "trigger window fell into the left trim" recursion, of which the caller keeps only the last region
// created (the list head, 2093-2097), so deeper recursion levels can never influence the result.
// Everything behind the window flags runs out of line (kj_seg_regions): a fragment with a low-complexity window is the exception, and
// inlined copies of the region search cost instruction-cache space in the hot loop of every kernel.
struct KjSegArgs { Warp w; const uint8_t* frag; const uint8_t* hf; KjSeg* segs; uint8_t* scratch; const double* lnf; int cap; uint32_t* err; };
template <int LEVEL, bool LONG>
static KJ_DEV int kj_seg_level(const KjSegArgs& A, int s0, int n, KjSeg* segs, int nsegs) {
    const uint8_t* frag = A.frag; const uint8_t* hf = A.hf;
    if (KJ_SEG_WINDOW > n) return nsegs;
    const int first = KJ_SEG_DOWNSET, last = n - KJ_SEG_UPSET; int lowlim = first;
    KJ_ROLLED
    for (int i = first; i <= last; i++) {
        if (hf[s0 + i - KJ_SEG_DOWNSET] & 1) {
            int j = i;
            KJ_ROLLED
            while (j >= lowlim && (hf[s0 + j - KJ_SEG_DOWNSET] & 2)) j--;
            const int loi = j + 1;         // s_FindLow
            j = i;
            KJ_ROLLED
            while (j <= last && (hf[s0 + j - KJ_SEG_DOWNSET] & 2)) j++;
            const int hii = j - 1;               // s_FindHigh
            int leftend = loi - KJ_SEG_DOWNSET, rightend = hii + KJ_SEG_UPSET - 1;
            if constexpr (LONG) {
                const int n2 = rightend - leftend + 1; const uint64_t tr = kj_seg_trim_wide(A.w, A.scratch, frag + s0 + leftend, n2, A.lnf);
                leftend += (int)(tr >> 32); rightend -= n2 - (int)(uint32_t)tr - 1;
            } else
            { const int n2 = rightend - leftend + 1; const uint32_t tr = kj_seg_trim(A.w, A.scratch, frag + s0 + leftend, n2, A.lnf);
              leftend += (int)(tr >> 16); rightend -= n2 - (int)(tr & 0xffffu) - 1; }
            if (LEVEL == 0 && i + KJ_SEG_UPSET - 1 < leftend) {
                const int lend = loi - KJ_SEG_DOWNSET, rend = leftend - 1;
                KjSeg tmp; tmp.begin = -1; tmp.end = -1;
                int got = kj_seg_level<1, LONG>(A, s0 + lend, rend - lend + 1, &tmp, 0);
                if (got > 0 && nsegs + 2 < A.cap) { if (A.w.lane == 0) segs[nsegs] = tmp; nsegs++; }
            }
            if (LEVEL == 0) {
                if (nsegs + 2 < A.cap) { if (A.w.lane == 0) { segs[nsegs].begin = leftend + s0; segs[nsegs].end = rightend + s0; } nsegs++; }
                else if (A.w.lane == 0) {
#if defined(KJ_EMU)
                    *A.err |= 8u;
#else
                    atomicOr(A.err, 8u);
#endif
                }
            }
            else { segs[0].begin = leftend + s0; segs[0].end = rightend + s0; nsegs = 1; }      // LEVEL 1: register struct, keep the last
            i = hii < rightend + KJ_SEG_DOWNSET ? hii : rightend + KJ_SEG_DOWNSET;
            lowlim = i + 1;
        }
    }
    return nsegs;
}
// regions + s_MergeSegs (2122-2152) for a fragment whose window flags are set; returns the number of regions (ascending)
template <bool LONG>
static KJ_DEV int kj_seg_regions_t(const KjSegArgs& A, int n) {
    KjSeg* segs = A.segs;
    int ns = kj_seg_level<0, LONG>(A, 0, n, segs, 0);
    A.w.sync();
    if (ns > 1) {
        // creation order == ascending; the reference walks the reversed list from its head
        if (A.w.lane == 0) {
            int cur = ns - 1, nx = cur - 1;                      // merged entries are marked begin = -1
            KJ_ROLLED
            while (nx >= 0) {
                if (segs[cur].begin - segs[nx].end - 1 < 0) {
                    if (segs[cur].end < segs[nx].end) segs[cur].end = segs[nx].end;
                    if (segs[cur].begin > segs[nx].begin) segs[cur].begin = segs[nx].begin;
                    segs[nx].begin = -1;
                } else cur = nx;
                nx--;
            }
            int o = 0;
            KJ_ROLLED
            for (int t = 0; t < ns; t++) if (segs[t].begin >= 0) segs[o++] = segs[t];
            segs[ns].begin = o;                                  // pass the count through shared memory
        }
        A.w.sync();
        ns = segs[ns].begin;
        A.w.sync();
    }
    return ns;
}
KJ_NOINLINE int kj_seg_regions(const KjSegArgs A, int n) { return kj_seg_regions_t<false>(A, n); }
KJ_NOINLINE int kj_seg_regions_long(const KjSegArgs A, int n) { return kj_seg_regions_t<true>(A, n); }
// full SEG on frag[0..n): flags (inline, every fragment), regions (out of line, rare)
template <bool LONG = false>
static KJ_DEV int kj_seg(KjWarpCtx& cx, int n, const bool compact) {
    if (n < KJ_SEG_WINDOW) return 0;
    if (!kj_seg_flags(cx, n, compact)) return 0;                      // no window at or below locut: s_SegSeq cannot trigger
    KjSegArgs A; A.w = cx.w; A.frag = cx.smem + cx.L.frag_off; A.hf = cx.smem + cx.L.hflag_off; A.segs = (KjSeg*)(cx.smem + cx.L.segs_off);
    A.scratch = cx.smem + cx.L.segcnt_off; A.lnf = cx.ix->lnfact; A.cap = (int)KJ_SEG_CAP(cx.rp->max_frag); A.err = cx.err;
    if constexpr (LONG) return kj_seg_regions_long(A, n);
    else return kj_seg_regions(A, n);
}

// ---------------------------------------------------------------------------------------------
// winners ("kept" suffix intervals): first kept_cap_smem in shared memory, the rest in global scratch
// ---------------------------------------------------------------------------------------------
static KJ_DEV KjKept* kj_kept_ptr(KjWarpCtx& cx, uint32_t idx) {
    if (idx < cx.rp->kept_cap_smem) return (KjKept*)(cx.smem + cx.L.kept_off) + idx;
    uint32_t s = idx - cx.rp->kept_cap_smem;
    if (s >= cx.rp->scratch_entries) { kj_flag_error(cx, 2u); s = cx.rp->scratch_entries - 1; }
    return cx.spill + s;
}

// taxon ids of the kept intervals in order, k ascending, stop once the set exceeds 20 entries
// (ids_from_SI, ConsumerThread.cpp:799-835); then LCA (util.cpp:194-263).  Runs once per read, out of line.
// The rows of ALL kept intervals, in order, are resolved 32 at a time (a read whose matches sit in several small intervals waits for one
// wave, not one per interval); the in-order de-duplication and the stop rule are then replayed over the wave, so rows fetched beyond the
// stop are never observed.  A row's taxon is one load from the dense row -> taxon array where the index has one (ix.row_tax), else the
// SA walk; accessions (verbose output) always take the walk, which ends on the suffix-array entry they are stored by.
// Returns compact taxon (KJ_TAX_BAD for "none") | number of ids << 32.
struct KjIdsArgs { Warp w; const KjDevIndex* ix; const KjKept* kept_smem; const KjKept* spill; uint32_t kept_cap, spill_cap; uint32_t* ids; uint32_t* accs; };     // accs: nullptr or [20] + count at [20]
template <class IdxT>
KJ_NOINLINE uint64_t kj_ids_and_lca_fn(const KjIdsArgs A, uint32_t nkept) {
    const Warp& w = A.w; const KjDevIndex& ix = *A.ix;
    uint32_t* ids = A.ids;
    uint32_t nids = 0, nacc = 0;                                          // uniform
    uint32_t* accs = A.accs;
    const uint32_t* row_tax = accs ? nullptr : ix.row_tax;
#if defined(KJ_EMU)
    if (w.lane == 0) { kj_emu_stats.id_reads++; kj_emu_stats.kept += nkept; }
#endif
    auto kept_at = [&](uint32_t x) { const uint32_t sx = x - A.kept_cap; return x < A.kept_cap ? A.kept_smem[x] : A.spill[sx < A.spill_cap ? sx : A.spill_cap - 1]; };
    uint32_t e = 0, off = 0;                                              // uniform: the next row to resolve is row `off` of kept interval e
    KjKept kk; kk.lo = 0; kk.len = 0; kk.aux = 0;
    if (nkept) kk = kept_at(0);
    KJ_ROLLED
    while (e < nkept && nids <= 20) {
        const uint32_t t = (uint32_t)w.lane, left = kk.len - off;
        uint64_t row = kk.lo + off + t;
        uint32_t nact = left < 32u ? left : 32u, next_e = e + (off + nact >= kk.len ? 1u : 0u), next_off = next_e != e ? 0u : off + nact;
        if (left < 32u && e + 1u < nkept) {
            // the wave spans several intervals.  Lane j holds interval e + j: its rows still to resolve (capped at 33: a wave takes 32) and their
            // inclusive prefix sum over the lanes; lane t takes the t-th row, which lies in the first interval whose prefix sum exceeds t
            const uint32_t x = e + t;
            uint64_t lo = 0; uint32_t rem = 0;
            if (x < nkept) { const KjKept kx = kept_at(x); lo = kx.lo; rem = kx.len; if (t == 0) { lo += off; rem -= off; } rem = rem < 33u ? rem : 33u; }
            uint32_t incl = rem, j = 0;
            KJ_ROLLED
            for (int d = 1; d < 32; d <<= 1) { const uint32_t o = w.shfl(incl, w.lane - d); if (w.lane >= d) incl += o; }
            KJ_ROLLED
            for (uint32_t s = 16; s > 0; s >>= 1) { if (w.shfl(incl, (int)(j + s - 1)) <= t) j += s; }
            row = w.shfl64(lo - (uint64_t)(incl - rem), (int)j) + t;          // lo_j + (t - first wave position of interval j)
            const uint32_t total = w.shfl(incl, 31);
            nact = total < 32u ? total : 32u;
            // the cursor moves past the intervals the wave finished (prefix sum <= 32; at least interval e) into the one it stopped in
            const uint32_t nfull = (uint32_t)kj_popc(w.ballot(x < nkept && incl <= 32u));
            next_e = e + nfull; next_off = 32u - w.shfl(incl, (int)nfull - 1);
        }
        uint32_t tax = KJ_TAX_BAD, acc = 0xffffffffu;
#if defined(KJ_EMU)
        const unsigned long long lf0 = kj_emu_stats.sa_lf_steps;
#endif
        if (t < nact) {
            if (row_tax) tax = row_tax[row];
            else { bool is_seq; const uint64_t en = kj_sa_locate<IdxT>(ix, row, is_seq); tax = is_seq ? ix.seq_tax[en] : ix.sa_tax[en]; if (accs) acc = is_seq ? ix.seq_acc[en] : ix.sa_acc[en]; }
        }
#if defined(KJ_EMU)
        { const uint32_t mx = warp_max_u32(w, (uint32_t)(kj_emu_stats.sa_lf_steps - lf0)); if (w.lane == 0) { kj_emu_stats.sa_waves++; kj_emu_stats.sa_dep_steps += mx; } }
#endif
        if (next_e != e && next_e < nkept) kk = kept_at(next_e);
        e = next_e; off = next_off;
        KJ_ROLLED
        for (uint32_t s = 0; s < nact && nids <= 20; s++) {
            uint32_t id = w.shfl(tax, (int)s);
            if (id == KJ_TAX_BAD) continue;
            if (accs) {          // match_dbnames (ConsumerThread.cpp:821-823): first 20 distinct accessions of the visited sequences
                const uint32_t a = w.shfl(acc, (int)s);
                if (a != 0xffffffffu && nacc < 20u) { const bool dupa = (uint32_t)w.lane < nacc && accs[w.lane] == a; if (!w.any(dupa)) { if (w.lane == 0) accs[nacc] = a; nacc++; w.sync(); } }
            }
            bool dup = (uint32_t)w.lane < nids && ids[w.lane] == id;
            if (!w.any(dup)) { if (w.lane == 0) ids[nids] = id; nids++; w.sync(); }
        }
    }
    if (accs && w.lane == 0) accs[20] = nacc;
    const uint64_t hi = (uint64_t)nids << 32;
    if (nids == 0) return hi | KJ_TAX_BAD;
    w.sync();
    if (nids == 1) return hi | ids[0];                                    // returned without a nodes.dmp check (ConsumerThread.cpp:625)
    // lca_from_ids: drop ids absent from nodes.dmp (depth 0), lift to the shallowest depth, climb in lockstep
    uint32_t id = (uint32_t)w.lane < nids ? ids[w.lane] : KJ_TAX_BAD;
    uint32_t depth = id != KJ_TAX_BAD ? ix.tax_depth[id] : 0u;
    bool present = depth > 0;
    uint32_t pm = w.ballot(present);
    if (!pm) return hi | KJ_TAX_BAD;
    uint32_t shallow = warp_min_u32(w, present ? depth : 0xffffffffu);
    if (present) for (uint32_t d = depth; d > shallow; d--) id = ix.tax_parent[id];
    int first = kj_ffs(pm) - 1;
    KJ_ROLLED
    for (uint32_t guard = 0; guard <= shallow + 1; guard++) {
        uint32_t f = w.shfl(id, first);
        bool diff = present && id != f;
        if (!w.any(diff)) return hi | f;
        if (present) id = ix.tax_parent[id];
    }
    return hi | KJ_TAX_BAD;
}
template <class IdxT>
static KJ_DEV uint32_t kj_ids_and_lca(KjWarpCtx& cx, uint32_t nkept) {
    KjIdsArgs A; A.w = cx.w; A.ix = cx.ix; A.kept_smem = (const KjKept*)(cx.smem + cx.L.kept_off); A.spill = cx.spill;
    A.kept_cap = cx.rp->kept_cap_smem; A.spill_cap = cx.rp->scratch_entries; A.ids = (uint32_t*)(cx.smem + cx.L.ids_off);
    A.accs = cx.want_acc ? (uint32_t*)(cx.smem + cx.L.accs_off) : nullptr;
    const uint64_t r = kj_ids_and_lca_fn<IdxT>(A, nkept);
    cx.nids = (uint32_t)(r >> 32);
    return (uint32_t)r;
}

// ---------------------------------------------------------------------------------------------
// MEM mode  (classify_length, ConsumerThread.cpp:543-628, with greedyExact, bwt.c:347-380)
// ---------------------------------------------------------------------------------------------

// SEG gate of getNextFragment (ConsumerThread.cpp:285-339): returns true if the item was split (pieces pushed)
template <bool LONG = false>
static KJ_DEV bool kj_seg_gate(KjWarpCtx& cx, KjQueue<LONG>& q, uint32_t arr, uint32_t start, uint32_t len, bool greedy) {
    int ns = kj_seg<LONG>(cx, (int)len, greedy);
    if (ns == 0) return false;
    if constexpr (!LONG) kj_queue_make_dirty(cx, q);          // (the long kernels' queue keeps late entries apart: kj_queue_top_long)
    const KjSeg* segs = (const KjSeg*)(cx.smem + cx.L.segs_off);
    const uint8_t* frag = cx.smem + cx.L.frag_off; const KjTables& tb = *cx.tb;
    uint32_t st = 0;
    KJ_ROLLED
    for (int s = 0; s <= ns; s++) {
        int plen = (s < ns ? segs[s].begin : (int)len) - (int)st;         // non-masked piece [st, st+plen)
        if (plen > (int)cx.rp->m) {                                        // strict '>' for pieces (298, 312)
            uint32_t val = (uint32_t)plen; bool ok = true;
            if (greedy) { uint32_t sc = 0; for (int t = 0; t < plen; t++) { uint32_t a = frag[st + t]; sc += (uint32_t)tb.b62[a][a]; } val = sc; ok = sc >= cx.rp->min_score; }
            kj_queue_emit<LONG>(cx, q, cx.w.lane == 0 && ok, val, (LONG ? KJ_ORDER_LATE_LONG : KJ_ORDER_LATE) + q.late, kj_qpay<LONG>(arr, true, start + 3u * st, (uint32_t)plen));
            if (ok) q.late++;
        }
        if (s < ns) st = (uint32_t)segs[s].end + 1u;
    }
    return true;
}

// One popped fragment: search, deferred SEG gate, merge into the kept list.  Returns true if it had a match >= L.
template <class IdxT, bool LONG = false>
static KJ_DEV bool kj_mem_item(KjWarpCtx& cx, KjQueue<LONG>& q, typename KjW<LONG>::pay pay, uint32_t& longest, uint32_t& nkept) {
    const Warp& w = cx.w; const KjDevIndex& ix = *cx.ix; const KjRunParams& rp = *cx.rp;
    const uint8_t* frag = cx.smem + cx.L.frag_off;
    uint32_t arr, start, len; bool segchecked;
    if constexpr (LONG) kj_qpay_dec<LONG>(pay, arr, segchecked, start, len);
    else { arr = pay >> 30; start = (pay >> 14) & 0x7fffu; len = pay & 0x3fffu; segchecked = (pay >> 29) & 1u; }
        kj_load_frag(cx, arr, start, len);
        // SEG is deferred until the fragment is known to matter: every match inside a SEG piece is also a match inside the
        // whole fragment (for each end position the piece's match is a suffix of the fragment's), so a fragment whose
        // search finds nothing >= L cannot contribute through its pieces either, and un-pushed useless pieces are not
        // observable (they never change `longest`, the kept list or the relative order of other queue entries).
        // greedyExact(f, seq, len, max(m,longest), -1) (bwt.c:347-380): chains for j = len-1 .. L-1, L growing
        uint32_t L = rp.m > longest ? rp.m : longest;
        uint32_t item_best = 0, item_cnt = 0;                             // uniform
        const bool mono = ix.mono != 0; const int kk = ix.kmer_k;
        // blocks of 32 end positions, j descending.  Every lane with j >= 0 runs phase A (chains below the scan range j >= L-1 only
        // serve as bounds); the block below is started early only when the lowest open chains of this block need its bound.
        // One loop with a single phase-A site and a single completion site (code size: the instruction cache is the scarce resource).
        int jhi = (int)len - 1, jstart = jhi, round = 0; bool start_la = false, have_nxt = false;
        KjChain<IdxT> cur, nxt;
        cur.lo = 0; cur.hi = 0; cur.i = 0; cur.st = KJ_ST_EXACT; nxt = cur;
        KJ_ROLLED
        for (;;) {
            if (jstart >= 0) {                                                              // phase A of the block whose top end position is jstart
                KjChain<IdxT> t; t.lo = 0; t.hi = 0; t.i = 0; t.st = KJ_ST_EXACT;
                if (jstart - w.lane >= (int)L - 1 || (start_la && jstart - w.lane >= 0)) kj_chain_start<IdxT>(ix, frag, jstart - w.lane, rp.m, t);
                w.sync();
                if (start_la) { nxt = t; have_nxt = true; } else { cur = t; round = 0; }
                jstart = -1;
#if defined(KJ_EMU)
                if (w.lane == 0) { if (start_la) kj_emu_stats.lookaheads++; else kj_emu_stats.blocks++; }
#endif
            }
            // (chains below the scan range as extra bounds were slower in an A/B run: their rank traffic costs more than the skipped chains save)
            const int j = jhi - w.lane; const bool act = j >= (int)L - 1;
            // `if (i<=1) break` (bwt.c:376): lanes below the first finished lane with i<=1 were never run by the reference
            const uint32_t brk = w.ballot(act && cur.st == KJ_ST_EXACT && cur.i <= 1);
            const int cut = brk ? kj_ffs(brk) - 1 : 31;
            const bool open = act && cur.st == KJ_ST_OPEN && w.lane <= cut;
            const uint32_t om = w.ballot(open);
            uint32_t nm = 0; bool need = false;
            if (om) {                                                                       // phase B: which open chains have to be completed?
                int lb = 0;
                if (mono) {
                    int lb_ext = 0;
                    if (round > 0 && !have_nxt && jhi - 32 >= 0) {
                        // (not before the first round: a full-length match ends the fragment with one chain.)  The lowest open chain
                        // has no ended chain below it in this block: fetch the bound from the next block's phase A
                        const uint32_t inf = w.ballot(act && cur.st != KJ_ST_OPEN);
                        if ((31 - kj_clz(om)) > (inf ? 31 - kj_clz(inf) : -1)) { jstart = jhi - 32; start_la = true; continue; }
                    }
                    if (have_nxt) lb_ext = kj_block_lb_ext<IdxT>(w, nxt, jhi - 32 - w.lane >= 0, jhi - 32 - w.lane, kk);
                    lb = kj_chain_lb<IdxT>(w, cur, act, j, kk, lb_ext);
                }
                // L as the reference holds it when it reaches lane x: the finished chains above x (the open ones above x are completed
                // before x can be skipped for good: the test is repeated every round)
                const uint32_t exl = (act && cur.st == KJ_ST_EXACT && w.lane <= cut) ? (uint32_t)(j - cur.i + 1) : 0u;
                const uint32_t Lb = kj_prefix_max_excl(w, exl, L);
                need = open && j >= (int)Lb - 1 && !(lb >= 2 && (uint32_t)(j - lb + 1) < Lb);
                nm = w.ballot(need);
            }
            if (nm) {
                // first round: only the top chain of every run of open chains (it settles the whole run when it reaches the bound);
                // later rounds: the next few chains in descending j as well
                const bool top = need && !(w.lane > 0 && ((nm >> (w.lane - 1)) & 1u));
                const int group = (round == 0 && mono) ? 0 : KJ_GROUP_LATE;
                const bool sel = need && (top || kj_popc(nm & lanemask_lt(w.lane)) < group);
                kj_finish_selected<IdxT>(w, ix, frag, sel, cur);
                round++;
                continue;
            }
            // the block is settled
            const bool valid = act && w.lane <= cut;
            const uint32_t l = (valid && cur.st == KJ_ST_EXACT) ? (uint32_t)(j - cur.i + 1) : 0u;
            const uint32_t lmax = warp_max_u32(w, l);
            if (lmax >= L) {
                if (lmax > item_best) { item_best = lmax; item_cnt = 0; }
                L = lmax;
                const uint32_t wm = w.ballot(l == item_best && l > 0);
                // aux: where the matched text lies (verbose output).  The long kernels keep its 21-bit position only: every kept match is `longest` long.
                if (l == item_best && l > 0) { KjKept* k = kj_kept_ptr(cx, nkept + item_cnt + (uint32_t)kj_popc(wm & lanemask_lt(w.lane))); k->lo = (uint64_t)cur.lo; k->len = (uint32_t)(cur.hi - cur.lo);
                                               k->aux = LONG ? (arr << 29) | (start + 3u * (uint32_t)cur.i) : (arr << 29) | ((start + 3u * (uint32_t)cur.i) << 14) | l; }
                item_cnt += (uint32_t)kj_popc(wm);
            }
            jhi -= 32;
            if (brk || jhi < (int)L - 1) break;
            round = 0;
            if (have_nxt) { cur = nxt; have_nxt = false; } else { jstart = jhi; start_la = false; }
        }
        w.sync();
        // the SEG gate of getNextFragment (ConsumerThread.cpp:285-339), now that the fragment has a match >= L: if SEG masks
        // something the fragment is replaced by its pieces exactly as in the reference and this search result is dropped
        if (item_cnt > 0 && rp.seg && !segchecked && kj_seg_gate<LONG>(cx, q, arr, start, len, false)) return true;
        if (item_cnt > 0) {
            // winners were appended j-descending; the reference's chain (greedyExact, bwt.c:347-380) is newest (smallest j) first.  The
            // kaijux / kaijup front-ends search with maxMatches(..., 1) instead, whose list keeps the first-found match at the head and
            // the others newest first behind it (insert_SI_sorted, bwt.c:225-252): there only the entries after the first are reversed.
            const uint32_t keep = rp.name_mode ? 1u : 0u;
            KJ_ROLLED
            for (uint32_t t = (uint32_t)w.lane; t < (item_cnt - keep) / 2; t += 32) {
                KjKept* a = kj_kept_ptr(cx, nkept + keep + t); KjKept* b = kj_kept_ptr(cx, nkept + item_cnt - 1 - t);
                KjKept x = *a; *a = *b; *b = x;
            }
            w.sync();
            if (w.lane == 0) kj_kept_ptr(cx, nkept)->aux |= 0x80000000u;  // the head of this fragment's list: its text goes to the fragment column (longest_fragments, 579-590)
            w.sync();
            if (item_best > longest) {                                    // replace (ConsumerThread.cpp:574-585)
                if (nkept > 0) {
                    KJ_ROLLED
                    for (uint32_t t0 = 0; t0 < item_cnt; t0 += 32) {      // move down, chunk by chunk (src index > dst index)
                        uint32_t t = t0 + (uint32_t)w.lane; KjKept x; x.lo = 0; x.len = 0; x.aux = 0;
                        if (t < item_cnt) x = *kj_kept_ptr(cx, nkept + t);
                        w.sync();
                        if (t < item_cnt) *kj_kept_ptr(cx, t) = x;
                        w.sync();
                    }
                }
                nkept = item_cnt; longest = item_best;
            } else if (item_best == longest) nkept += item_cnt;           // append (586-591)
        }
    return item_cnt > 0;
}

// fragment column of the verbose output in MEM mode: the text of the head match of every contributing fragment, "TEXT,TEXT," (614-623)
KJ_NOINLINE uint32_t kj_emit_text(const Warp w, char* text, uint32_t at, uint32_t cap, const uint8_t* src, uint32_t stride, uint32_t len, const char* letters) {
    if (at + len + 1u > cap) return 0xffffffffu;
    KJ_ROLLED
    for (uint32_t t = (uint32_t)w.lane; t < len; t += 32) text[at + t] = letters[src[stride * t]];
    if (w.lane == 0) text[at + len] = ',';
    return at + len + 1u;
}
template <bool LONG = false>
static KJ_DEV void kj_emit_fragments_mem(KjWarpCtx& cx, uint32_t nkept, uint32_t longest) {
    KJ_ROLLED
    for (uint32_t e = 0; e < nkept; e++) {
        const uint32_t aux = kj_kept_ptr(cx, e)->aux;
        if (!(aux >> 31)) continue;
        const uint32_t arr = (aux >> 29) & 3u, pos = LONG ? aux & 0x1fffffffu : (aux >> 14) & 0x7fffu, len = LONG ? longest : aux & 0x3fffu;
        const uint32_t at = kj_emit_text(cx.w, cx.text, cx.text_len, cx.text_cap, cx.smem + cx.L.aa_off + arr * cx.L.aa_stride + pos, 3u, len, cx.tb->letters);
        if (at == 0xffffffffu) { if (cx.w.lane == 0) kj_flag_error(cx, 128u); return; }
        cx.text_len = at;
    }
    cx.w.sync();
}
template <class IdxT, bool LONG = false>
static KJ_DEV uint32_t kj_classify_mem(KjWarpCtx& cx, KjQueue<LONG>& q, uint32_t& best_out) {
    uint32_t longest = 0, nkept = 0;                                      // uniform
    uint32_t val; typename KjW<LONG>::pay pay;
    KJ_ROLLED
    while (kj_queue_pop<LONG>(cx, q, longest, val, pay)) kj_mem_item<IdxT, LONG>(cx, q, pay, longest, nkept);
    best_out = 0;
    if (nkept == 0) return KJ_TAX_BAD;
    cx.w.sync();
    uint32_t t = kj_ids_and_lca<IdxT>(cx, nkept);
    if (t != KJ_TAX_BAD) best_out = longest;
    if (cx.text && t != KJ_TAX_BAD) kj_emit_fragments_mem<LONG>(cx, nkept, longest);
    return t;
}

// ---------------------------------------------------------------------------------------------
// ConsumerThread::doWork for one item (ConsumerThread.cpp:630-749): gates, translation, mode dispatch.
// Returns the compact taxon (KJ_TAX_BAD = unclassified).
// ---------------------------------------------------------------------------------------------
template <class IdxT, bool LONG = false> static KJ_DEV uint32_t kj_classify_greedy(KjWarpCtx& cx, KjQueue<LONG>& q, double query_len, uint32_t& best_out);

// Protein input (-p, ConsumerThread.cpp:640-646, 659-696): the read is upper-cased and split at every letter outside
// "ACDEFGHIKLMNPQRSTVWY"; pieces of at least m residues (Greedy: and score >= min_score) are queued in order, the tail last.
// The residues are stored like one reading frame of a translated read (residue e at array index 3e), so the queue
// payloads, kj_load_frag and the SEG pieces need no second addressing mode.
template <bool LONG = false>
static KJ_DEV void kj_protein_fragments(KjWarpCtx& cx, KjQueue<LONG>& q, const uint8_t* s1, int n1, bool greedy, const bool small_code) {
    const Warp& w = cx.w; const KjTables& tb = *cx.tb;
    uint8_t* aa = cx.smem + cx.L.aa_off;
    KJ_ROLLED
    for (int t = w.lane; t < n1; t += 32) {
        const uint32_t u = s1[t] & 0xDFu;                                // in 'A'..'Z' exactly for ASCII letters (toupper)
        aa[3 * t] = (u >= 'A' && u <= 'Z') ? tb.aa_index[u - 'A'] : (uint8_t)0;
    }
    w.sync();
    if (small_code) kj_split_frames_rolled<LONG>(cx, q, 3 * n1 - 2, 0, n1, 0, greedy, 1);
    else kj_split_frames<LONG>(cx, q, 3 * n1 - 2, 0, n1, 0, greedy, 1);
}

// ---------------------------------------------------------------------------------------------
// Greedy in two kernels (ROLE 1 = front end, ROLE 2 = search; ROLE 0 = everything in one kernel, as MEM runs).  Greedy is bound by instruction
// fetch (see kj_warp.h): translation, frame splitting and queue ranking are 6 KB of its hot code that the search does not need.
// The front end leaves, per item, the four translated arrays and the ranked fragment queue in a record in global memory (1.5 KB for PE150);
// the search kernel copies the record into the same places of its work space and continues exactly where the single kernel would.
//   record: [0] uint32 queue length (0xffffffff = unclassified by the length gates), [16] keys, pays, ranks, [..] the aa arrays
// ---------------------------------------------------------------------------------------------
static KJ_HD uint32_t kj_prep_keys_off() { return 16u; }
static KJ_HD uint32_t kj_prep_pays_off(const KjRunParams& p) { return 16u + 8u * p.item_cap; }
static KJ_HD uint32_t kj_prep_ords_off(const KjRunParams& p) { return kj_prep_pays_off(p) + 4u * kj_align(p.item_cap, 2); }
static KJ_HD uint32_t kj_prep_aa_off(const KjRunParams& p) { return kj_align(kj_prep_ords_off(p) + kj_align(p.item_cap, 8), 16); }
static KJ_HD uint32_t kj_prep_stride(const KjRunParams& p) { return kj_align(kj_prep_aa_off(p) + 4u * kj_align(p.max_len + 4, 8), 16); }
static KJ_DEV void kj_prep_store(KjWarpCtx& cx, const KjQueue<>& q, bool ok, uint8_t* rec) {
    const Warp& w = cx.w; const KjRunParams& rp = *cx.rp;
    w.sync();
    if (w.lane == 0) *(uint32_t*)rec = ok ? q.n : 0xffffffffu;
    if (ok) {
        uint64_t* rk = (uint64_t*)(rec + kj_prep_keys_off()); uint32_t* rp_ = (uint32_t*)(rec + kj_prep_pays_off(rp)); uint8_t* ro = rec + kj_prep_ords_off(rp);
        KJ_ROLLED
        for (uint32_t i = (uint32_t)w.lane; i < q.n; i += 32) { rk[i] = q.key[i]; rp_[i] = q.pay[i]; ro[i] = q.ord[i]; }
        const uint32_t* a = (const uint32_t*)(cx.smem + cx.L.aa_off); uint32_t* ra = (uint32_t*)(rec + kj_prep_aa_off(rp));
        KJ_ROLLED
        for (uint32_t i = (uint32_t)w.lane; i < cx.L.aa_stride; i += 32) ra[i] = a[i];          // 4 arrays x stride bytes = stride words
    }
    w.sync();
}
static KJ_DEV bool kj_prep_load(KjWarpCtx& cx, KjQueue<>& q, const uint8_t* rec) {
    const Warp& w = cx.w; const KjRunParams& rp = *cx.rp;
    const uint32_t n = *(const uint32_t*)rec;
    if (n == 0xffffffffu) return false;
    const uint64_t* rk = (const uint64_t*)(rec + kj_prep_keys_off()); const uint32_t* rp_ = (const uint32_t*)(rec + kj_prep_pays_off(rp)); const uint8_t* ro = rec + kj_prep_ords_off(rp);
    KJ_ROLLED
    for (uint32_t i = (uint32_t)w.lane; i < n; i += 32) { q.key[i] = rk[i]; q.pay[i] = rp_[i]; q.ord[i] = ro[i]; }
    uint32_t* a = (uint32_t*)(cx.smem + cx.L.aa_off); const uint32_t* ra = (const uint32_t*)(rec + kj_prep_aa_off(rp));
    KJ_ROLLED
    for (uint32_t i = (uint32_t)w.lane; i < cx.L.aa_stride; i += 32) a[i] = ra[i];
    q.n = n; q.late = 0; q.next = 0; q.nsorted = n <= 255u ? n : 0u; q.dirty = n > 255u;          // as kj_queue_sort leaves it
    w.sync();
    return true;
}

// LONG: the long-read instance (ROLE 0 only)
template <int MODE, class IdxT, int ROLE = 0, bool LONG = false>
static KJ_DEV uint32_t kj_classify_item(KjWarpCtx& cx, const uint8_t* s1, int n1, const uint8_t* s2, int n2, bool paired, uint32_t& best_out, uint8_t* rec = nullptr) {
    static_assert(!LONG || ROLE == 0, "the long-read kernels run every item in one kernel");
    const KjRunParams& rp = *cx.rp;
    best_out = 0; cx.nids = 0;
    KjQueue<LONG> q; q.key = (uint64_t*)(cx.smem + cx.L.qkey_off); q.pay = (typename KjW<LONG>::pay*)(cx.smem + cx.L.qpay_off);
    q.ord = cx.smem + cx.L.qord_off; q.cap = rp.item_cap; q.n = 0; q.late = 0; q.next = 0; q.nsorted = 0; q.dirty = true;
    const bool greedy = MODE == 1;
    // the one-kernel Greedy path trades the interleaved (4 arrays at once) frame splitting for a quarter of its code; the front-end kernel of the
    // two-kernel path has the instruction cache to itself and keeps the fast one
    const bool small_code = MODE == 1 && ROLE == 0;
    const int m3 = (int)rp.m * 3;
    if (ROLE != 2) {
        bool ok = true;
        if (rp.protein) {
            if (n1 < (int)rp.m) ok = false;                                  // (640-646)
            else kj_protein_fragments<LONG>(cx, q, s1, n1, greedy, small_code);
        } else {
            // short-read gate (648-653): SE len1 < 3m; PE only if BOTH mates are short
            if ((!paired && n1 < m3) || (paired && n1 < m3 && n2 < m3)) ok = false;
            else kj_translate_pair<LONG>(cx, q, s1, n1, n1 >= m3, s2, n2, paired && n2 >= m3, greedy, small_code);   // a short mate is skipped individually (699, 705)
        }
        // a long read's queue holds tens of thousands of fragments: ranked once in both modes, so that no pop scans them all
        if constexpr (LONG) { if (ok) kj_queue_rank_long(cx, q); }
        else {
        if (ok && MODE == 1) kj_queue_sort(cx, q);     // greedy pops every fragment (and many variants): ranking once pays (A/B); MEM stops after a few pops (slower with it)
        if constexpr (ROLE == 1) { kj_prep_store(cx, q, ok, rec); return KJ_TAX_BAD; }
        }
        if (!ok) return KJ_TAX_BAD;
    } else if constexpr (!LONG) { if (!kj_prep_load(cx, q, rec)) return KJ_TAX_BAD; }
    double query_len;                                                    // E-value query length (659, 698, 704)
    if (rp.protein) query_len = (double)n1;
    else { query_len = (double)n1 / 3.0; if (paired) query_len += (double)n2 / 3.0; }
    if (MODE == 0) return kj_classify_mem<IdxT, LONG>(cx, q, best_out);
    else return kj_classify_greedy<IdxT, LONG>(cx, q, query_len, best_out);
}
