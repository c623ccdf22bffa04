// kj_core_greedy.h -- Greedy mode: classify_greedyblosum (ConsumerThread.cpp:424-541) with maxMatches /
// maxMatches_withStart (bwt.c:261-336), addAllMismatchVariantsAtPosSI (346-395) and eval_match_scores (751-797).
//
// The reference's priority queue decides which equal-score matches survive the 20-SI and 21-id caps, so the
// queue is emulated per read (one warp), not relaxed: un-substituted fragments live in the shared-memory
// key queue of kj_core.h, substituted variants (sequence = source run + <= 8 point substitutions + truncation)
// in a per-warp global scratch ring that stays L2-resident.  Inside one pop the lanes parallelise what the
// reference does serially: all seed end positions j of maxMatches, the 19 substitution probes of one
// position, and the scoring of the recorded matches.
#pragma once
#include "kj_core.h"

template <bool LONG = false>
struct alignas(16) KjVariant {
    uint64_t lo, hi;           // resume interval (Fragment::si0/si1, ConsumerThread.hpp:52)
    typename KjW<LONG>::pay pay;   // source run (a queue payload, kj_qpay) -- len already truncated
    int32_t diff;              // accumulated substitution score delta (Fragment::diff)
    typename KjW<LONG>::pos matchlen; uint8_t num_mm; uint8_t pad;
    uint32_t subs[KJ_MAX_MM];  // pos << 5 | letter
    uint32_t pad2;
};
static_assert(sizeof(KjVariant<>) == 64, "KjVariant is one 64-byte record");
// per-warp ring in global scratch: keys[variant_cap] (scanned, contiguous) followed by the payload records
template <bool LONG = false>
static KJ_HD uint32_t kj_greedy_scratch_bytes(const KjRunParams& rp) { return rp.mode == 1 ? rp.variant_cap * (uint32_t)(sizeof(KjVariant<LONG>) + 8u) : 64u; }

template <bool LONG = false>
struct KjMatch { uint64_t lo; uint32_t len; typename KjW<LONG>::pos qi, ql; };    // one SI: interval + query position/length
static_assert(sizeof(KjMatch<false>) == 16 && sizeof(KjMatch<true>) == 24, "kj_smem_layout sizes the result arrays with these");

// key(s) = kj_qkey(score, order), 0 = free.  (Keeping the first keys in shared memory was slower in an A/B run.)
template <bool LONG = false>
struct KjVQueue { uint64_t* gkey; KjVariant<LONG>* v; uint32_t n, live;      // n: high-water mark, live: entries not yet popped (uniform)
    KJ_DEV uint64_t& key(uint32_t s) const { return gkey[s]; } };

// compact live variants to the front (called when the ring is full); out of line: rare.  Returns the number of live entries.
template <class V>
static KJ_DEV uint32_t kj_vq_compact_t(const Warp& w, uint64_t* gkey, V* v, uint32_t n) {
    uint32_t out = 0;
    KJ_ROLLED
    for (uint32_t b = 0; b < n; b += 32) {
        uint32_t s = b + (uint32_t)w.lane; bool live = s < n && gkey[s] != 0;
        V tmp; uint64_t tk = 0; if (live) { tmp = v[s]; tk = gkey[s]; }
        uint32_t mask = w.ballot(live);
        w.sync();
        if (live) { const uint32_t d = out + (uint32_t)kj_popc(mask & lanemask_lt(w.lane)); v[d] = tmp; gkey[d] = tk; }
        out += (uint32_t)kj_popc(mask);
        w.sync();
    }
    return out;
}
KJ_NOINLINE uint32_t kj_vq_compact_fn(const Warp w, uint64_t* gkey, KjVariant<>* v, uint32_t n) { return kj_vq_compact_t(w, gkey, v, n); }
KJ_NOINLINE uint32_t kj_vq_compact_long_fn(const Warp w, uint64_t* gkey, KjVariant<true>* v, uint32_t n) { return kj_vq_compact_t(w, gkey, v, n); }
template <bool LONG>
static KJ_DEV void kj_vq_compact(KjWarpCtx& cx, KjVQueue<LONG>& vq) {
    if constexpr (LONG) vq.n = kj_vq_compact_long_fn(cx.w, vq.gkey, vq.v, vq.n);
    else vq.n = kj_vq_compact_fn(cx.w, vq.gkey, vq.v, vq.n);
    vq.live = vq.n;
}

// inclusive warp scan helper (uint32)
static KJ_DEV uint32_t kj_scan_incl(const Warp& w, uint32_t v) {
    for (int d = 1; d < 32; d <<= 1) { uint32_t o = w.shfl(v, w.lane - d); if (w.lane >= d) v += o; }
    return v;
}

// LONG: positions, lengths and prefix sums in 32 bits, scores unclamped, and the match start rides above bit KJ_LONG_LO_BITS of `lo` (not 48)
template <class IdxT, bool LONG>
static KJ_DEV uint32_t kj_classify_greedy(KjWarpCtx& cx, KjQueue<LONG>& q, double query_len, uint32_t& best_out) {
    typedef typename KjW<LONG>::pos PosT; typedef KjMatch<LONG> Match;
    constexpr int QI_SHIFT = LONG ? KJ_LONG_LO_BITS : 48; constexpr uint64_t LO_MASK = (1ull << QI_SHIFT) - 1ull;
    const Warp& w = cx.w; const KjDevIndex& ix = *cx.ix; const KjRunParams& rp = *cx.rp; const KjTables& tb = *cx.tb;
    uint8_t* frag = cx.smem + cx.L.frag_off;
    PosT* pre = (PosT*)(cx.smem + cx.L.pre_off);                         // pre[t] = sum diag(frag[0..t))
    Match* res = (Match*)(cx.smem + cx.L.res_off);                      // per-j chain results, then recorded matches
    Match* cls = (Match*)(cx.smem + cx.L.res2_off);                     // recorded matches sorted into classes
    uint32_t* psub = (uint32_t*)(cx.smem + cx.L.ids_off + 64u);           // the id set is only filled after the loop
    KjVQueue<LONG> vq; vq.gkey = (uint64_t*)cx.gscratch; vq.v = (KjVariant<LONG>*)((uint8_t*)cx.gscratch + 8u * rp.variant_cap); vq.n = 0; vq.live = 0;
    uint32_t best = 0, nbest = 0;                                        // best_match_score, best_matches_SI.size()  (uniform)
    best_out = 0;

    KJ_ROLLED
    for (;;) {
        // ---------------- getNextFragment(best): top of both queues (ConsumerThread.cpp:272-283)
        w.sync();
        uint64_t kb = 0; uint32_t slot_b = 0;
        KJ_ROLLED
        for (uint32_t s = (uint32_t)w.lane; s < vq.n; s += 32) { uint64_t k = vq.key(s); if (k > kb) { kb = k; slot_b = s; } }
        uint64_t gb = warp_max_u64(w, kb);
        uint64_t ka = 0, ga = 0; uint32_t slot_a = 0;
        if constexpr (LONG) ga = kj_queue_top_long(cx, q, slot_a, best);
        else if (!q.dirty) { if (q.next < q.nsorted) { slot_a = q.ord[q.next]; ga = q.key[slot_a]; } }      // sorted prefix: the top is known
        else {
            KJ_ROLLED
            for (uint32_t s = (uint32_t)w.lane; s < q.n; s += 32) { uint64_t k = q.key[s]; if (k > ka) { ka = k; slot_a = s; } }
            ga = warp_max_u64(w, ka);
        }
        const uint64_t g = ga > gb ? ga : gb;
        if (g == 0) break;
        if (kj_qval<LONG>(g) < best) break;
        uint32_t arr, start, len, num_mm = 0, matchlen = 0; int diff = 0; uint64_t si0 = 0, si1 = 0; bool segchecked; uint32_t nsub = 0; uint32_t mysub = 0;
        if (ga >= gb) {
            typename KjW<LONG>::pay p = 0;
            if constexpr (LONG) p = kj_queue_take_long(cx, q, slot_a);
            else if (!q.dirty) { p = q.pay[slot_a]; q.next++; }
            else {
                int src = kj_ffs(w.ballot(ka == g)) - 1;
                if (w.lane == src) { p = q.pay[slot_a]; q.key[slot_a] = 0; }
                p = w.shfl(p, src);
            }
            kj_qpay_dec<LONG>(p, arr, segchecked, start, len);
#if defined(KJ_EMU)
            if (w.lane == 0) kj_emu_stats.pops_frag++;
#endif
        } else {
#if defined(KJ_EMU)
            if (w.lane == 0) kj_emu_stats.pops_var++;
#endif
            int src = kj_ffs(w.ballot(kb == g)) - 1; uint32_t sl = w.shfl(slot_b, src);
            const KjVariant<LONG>& V = vq.v[sl];
            if constexpr (LONG) { kj_qpay_dec<LONG>(V.pay, arr, segchecked, start, len); segchecked = true; }
            else { uint32_t p = V.pay; arr = p >> 30; start = (p >> 14) & 0x7fffu; len = p & 0x3fffu; segchecked = true; }
            num_mm = V.num_mm; matchlen = V.matchlen; diff = V.diff; si0 = V.lo; si1 = V.hi; nsub = num_mm;
            if ((uint32_t)w.lane < nsub) { mysub = V.subs[w.lane]; psub[w.lane] = mysub; }        // parent substitutions, re-read when variants are pushed
            w.sync();
            if (w.lane == 0) vq.key(sl) = 0;
            vq.live--;
        }
        kj_load_frag(cx, arr, start, len);
        if ((uint32_t)w.lane < nsub) frag[mysub >> 5] = (uint8_t)(mysub & 31u);
        w.sync();
        if (rp.seg && !segchecked && kj_seg_gate<LONG>(cx, q, arr, start, len, true)) continue;

        // prefix sums of the BLOSUM62 diagonal (calcScore, ConsumerThread.cpp:397-421)
        {
            uint32_t carry = 0;
            KJ_ROLLED
            for (uint32_t b = 0; b < len; b += 32) {
                uint32_t t = b + (uint32_t)w.lane; uint32_t a = t < len ? frag[t] : 0u;
                uint32_t d = t < len ? (uint32_t)tb.b62[a][a] : 0u;
                uint32_t sc = kj_scan_incl(w, d) + carry;
                if (t < len) pre[t + 1] = (PosT)sc;
                carry = w.shfl(sc, 31);
            }
            if (w.lane == 0) pre[0] = 0;
            w.sync();
        }

        // ---------------- search
        uint32_t nrec = 0;                                                // recorded matches (uniform)
        if (num_mm > 0) {
            // maxMatches_withStart (bwt.c:298-336): extend the stored interval leftwards from len - matchlen
            // one chain: lanes 0/1 compute the lower/upper interval end (kj_finish_paired on a one-chain selection)
            KjChain<IdxT> one; one.lo = (IdxT)si0; one.hi = (IdxT)si1; one.i = (int)len - (int)matchlen; one.st = KJ_ST_OPEN;
#if defined(KJ_EMU)
            const int i0_ = one.i;
#endif
            kj_chain_finish<IdxT>(ix, frag, one);                          // every lane runs the same chain: identical addresses, one sector per step
#if defined(KJ_EMU)
            if (w.lane == 0) kj_emu_stats.var_steps += (unsigned long long)(i0_ - one.i + 1);
#endif
            const IdxT lo = one.lo, hi = one.hi; const int i = one.i;
            uint32_t l = len - (uint32_t)i;
            uint32_t Lreq = (num_mm == rp.e) ? rp.m : matchlen;           // ConsumerThread.cpp:445-450
            if (l >= Lreq) { if (w.lane == 0) { cls[0].lo = (uint64_t)lo; cls[0].len = (uint32_t)(hi - lo); cls[0].qi = (PosT)i; cls[0].ql = (PosT)l; } nrec = 1; }
            w.sync();
        } else {
            // maxMatches(f, seq, len, seed_length, 0) (bwt.c:261-296): one chain per end position j.  Every chain above the `i<=1` break
            // is run by the reference, but only those whose match starts left of every longer-ending recorded match are kept: with the
            // bounds of kj_chain_lb most open chains are known not to be recorded without completing them.
            const int L = (int)rp.seed_length;
            const bool mono = ix.mono != 0; const int kk = ix.kmer_k;
            int jlow = (int)len; uint32_t qi_above = 0xffffffffu;                  // processed range [jlow, len-1]; smallest start of a qualifying finished chain of the blocks above
            int jhi = (int)len - 1, jstart = jhi, round = 0; bool start_la = false, have_nxt = false;
            KjChain<IdxT> cur, nxt;
            cur.lo = 0; cur.hi = 0; cur.i = 0; cur.st = KJ_ST_EXACT; nxt = cur;
            KJ_ROLLED
            for (;;) {                                                             // same skeleton as kj_mem_item: one phase-A site, one completion site
                if (jstart >= 0) {
                    KjChain<IdxT> t; t.lo = 0; t.hi = 0; t.i = 0; t.st = KJ_ST_EXACT;
                    if (jstart - w.lane >= L - 1 || (start_la && jstart - w.lane >= 0)) kj_chain_start<IdxT>(ix, frag, jstart - w.lane, rp.seed_length, t);
                    w.sync();
                    if (start_la) { nxt = t; have_nxt = true; } else { cur = t; round = 0; }
                    jstart = -1;
                }
                const int j = jhi - w.lane; const bool act = j >= L - 1;
                const uint32_t brk = w.ballot(act && cur.st == KJ_ST_EXACT && cur.i <= 1);        // `if (i<=1) break` (bwt.c:292)
                const int cut = brk ? kj_ffs(brk) - 1 : 31;
                const bool open = act && cur.st == KJ_ST_OPEN && w.lane <= cut;
                const uint32_t om = w.ballot(open);
                uint32_t nm = 0; bool need = false;
                if (om) {
                    int lb = 0;
                    if (mono) {
                        int lb_ext = 0;
                        if (round > 0 && !have_nxt && jhi - 32 >= 0) {
                            const uint32_t inf = w.ballot(act && cur.st != KJ_ST_OPEN);
                            if ((31 - kj_clz(om)) > (inf ? 31 - kj_clz(inf) : -1)) { jstart = jhi - 32; start_la = true; continue; }
                        }
                        if (have_nxt) lb_ext = kj_block_lb_ext<IdxT>(w, nxt, jhi - 32 - w.lane >= 0, jhi - 32 - w.lane, kk);
                        lb = kj_chain_lb<IdxT>(w, cur, act, j, kk, lb_ext);
                    }
                    // an open chain is not recorded if its match is shorter than L or cannot start left of a qualifying finished chain above it
                    const bool qual = act && cur.st == KJ_ST_EXACT && w.lane <= cut && j - cur.i + 1 >= L;
                    const uint32_t pmin = kj_prefix_min_excl(w, qual ? (uint32_t)cur.i : 0xffffffffu, qi_above);
                    need = open && !(lb >= 2 && (j - lb + 1 < L || (uint32_t)lb >= pmin));
                    nm = w.ballot(need);
                }
                if (nm) {
                    const bool top = need && !(w.lane > 0 && ((nm >> (w.lane - 1)) & 1u));
                    const int group = (round == 0 && mono) ? 0 : KJ_GROUP_LATE;
                    const bool sel = need && (top || kj_popc(nm & lanemask_lt(w.lane)) < group);
                    kj_finish_selected<IdxT>(w, ix, frag, sel, cur);
                    round++;
                    continue;
                }
                const bool valid = act && w.lane <= cut;
                if (valid) {
                    if (cur.st == KJ_ST_OPEN) { res[j].lo = 0; res[j].len = 0; res[j].qi = 0; res[j].ql = 0; }       // skipped: provably not recorded
                    else { res[j].lo = (uint64_t)cur.lo; res[j].len = (uint32_t)(cur.hi - cur.lo); res[j].qi = (PosT)cur.i; res[j].ql = (PosT)(j - cur.i + 1); }
                }
                { const bool qual = valid && cur.st == KJ_ST_EXACT && j - cur.i + 1 >= L; const uint32_t mn = warp_min_u32(w, qual ? (uint32_t)cur.i : 0xffffffffu); if (mn < qi_above) qi_above = mn; }
                const int nact = (jhi - (L - 1) + 1) < 32 ? (jhi - (L - 1) + 1) : 32;
                jlow = jhi - (brk ? cut + 1 : nact) + 1;
                jhi -= 32;
                if (brk || jhi < L - 1) break;
                round = 0;
                if (have_nxt) { cur = nxt; have_nxt = false; } else { jstart = jhi; start_la = false; }
            }
            w.sync();
            // recorded matches: l >= L and start strictly left of the previously recorded one (bwt.c:276-281).  With a true FM index
            // the starts are monotone in j, so "same start as j+1" is the only way to be skipped (32-bit kernels).  The reference's
            // checkpoint quirk for bwtlen = m * 2^16 can break chains early; those indexes run on the 64-bit kernels, which keep the
            // general rule: recorded starts decrease strictly, so "previously recorded" = the minimum start of the qualifying chains
            // seen so far (j descending), an exclusive prefix minimum.
            // pass 1: flags + found order (j descending); pass 2: class position = (#longer) + (#same length found earlier)
            const int nproc = (int)len - jlow;                             // processed j = len-1-t, t in [0,nproc)
            uint32_t cur_qi = 0xffffffffu;                                 // start of the last recorded match (uniform)
            KJ_ROLLED
            for (int b = 0; b < nproc; b += 32) {
                int t = b + w.lane; int j = (int)len - 1 - t; bool rec = false;
                {
                    uint32_t mine = 0xffffffffu;                           // my start if my chain qualifies
                    if (t < nproc) { Match r = res[j]; if (r.ql >= (uint32_t)L) mine = r.qi; }
                    uint32_t pm = mine;                                    // inclusive prefix minimum over the lanes
                    for (int dd = 1; dd < 32; dd <<= 1) { const uint32_t o = w.shfl(pm, w.lane - dd); if (w.lane >= dd && o < pm) pm = o; }
                    uint32_t ex = w.shfl(pm, w.lane - 1); if (w.lane == 0) ex = 0xffffffffu;     // exclusive
                    if (cur_qi < ex) ex = cur_qi;
                    rec = mine != 0xffffffffu && mine < ex;
                    { const uint32_t last = w.shfl(pm, 31); if (last < cur_qi) cur_qi = last; }
                }
                uint32_t mk = w.ballot(rec);
                if (rec) { Match r = res[j]; cls[nrec + (uint32_t)kj_popc(mk & lanemask_lt(w.lane))] = r; }   // found order, temporarily in cls
                nrec += (uint32_t)kj_popc(mk);
            }
            w.sync();
            // stable sort by ql descending into res (insert_SI_sorted, bwt.c:225-252)
            KJ_ROLLED
            for (uint32_t b = 0; b < nrec; b += 32) {
                uint32_t t = b + (uint32_t)w.lane;
                if (t < nrec) {
                    Match r = cls[t]; uint32_t pos = 0;
                    KJ_ROLLED
                    for (uint32_t u = 0; u < nrec; u++) { uint32_t q2 = cls[u].ql; pos += (q2 > r.ql || (q2 == r.ql && u < t)) ? 1u : 0u; }
                    res[pos] = r;
                }
            }
            w.sync();
            KJ_ROLLED
            for (uint32_t t = (uint32_t)w.lane; t < nrec; t += 32) cls[t] = res[t];
            w.sync();
        }
        if (nrec == 0) continue;                                           // "No match for this fragment" (457-462)
        // class structure of the (usually few) recorded matches as a bit mask: bit t set <=> cls[t] opens a class of equal length
        const bool small = nrec <= 32u;
        uint32_t heads = 0, my_ql = 0;
        if (small) {
            const bool in = (uint32_t)w.lane < nrec;
            my_ql = in ? cls[w.lane].ql : 0u;
            const uint32_t prev_ql = w.shfl(my_ql, w.lane - 1);
            heads = w.ballot(in && (w.lane == 0 || my_ql != prev_ql));
        }

        // ---------------- substitution variants (465-479 + addAllMismatchVariantsAtPosSI 346-395)
        if (rp.e > 0 && num_mm < rp.e) {
            // walk: class head, then its samelen chain fn..f2 if the class has >1 member (and stop), else the next class head
            uint32_t c0 = 0;
            KJ_ROLLED
            while (c0 < nrec) {
                uint32_t c1;
                if (small) { const uint32_t rest = heads & ~((2u << c0) - 1u); c1 = rest ? (uint32_t)kj_ffs(rest) - 1u : nrec; }
                else { c1 = c0 + 1; const uint32_t qlc = cls[c0].ql; while (c1 < nrec && cls[c1].ql == qlc) c1++; }
                const uint32_t nmem = c1 - c0;
                KJ_ROLLED
                for (uint32_t wi = 0; wi < nmem; wi++) {
                    const Match sm = cls[wi == 0 ? c0 : c1 - wi];
                    const uint32_t mre1 = (uint32_t)sm.qi + sm.ql;         // match_right_end + 1
                    if (sm.qi > 0 && mre1 >= rp.m) {
                        const uint32_t new_len = mre1 < len ? mre1 : len;   // erase_pos (474)
                        const uint32_t pos = (uint32_t)sm.qi - 1u; const uint32_t o = frag[pos];
                        int sc0 = (int)pre[new_len] + diff; if (sc0 < 0) sc0 = 0;
                        const int score = sc0 - (int)tb.b62[o][o];          // (363)
                        const bool lane_sub = w.lane < 19;
                        const uint32_t sub = lane_sub ? tb.subst[o][w.lane] : 0u;
                        const int after = lane_sub ? score + (int)tb.b62[o][sub] : 0;
                        const bool pass = lane_sub && after >= (int)best && after >= (int)rp.min_score;
                        const uint32_t failmask = ~w.ballot(pass) & 0x7ffffu;
                        const int n_ok = failmask ? kj_ffs(failmask) - 1 : 19;      // first failing substitute ends the loop (391)
                        IdxT lo = (IdxT)sm.lo, hi = (IdxT)(sm.lo + sm.len); bool ok = false;
                        if (w.lane < n_ok) ok = kj_update_si<IdxT>(ix, sub, lo, hi);
                        w.sync();
                        const uint32_t okmask = w.ballot(ok); const uint32_t cnt = (uint32_t)kj_popc(okmask);
                        if (cnt) {
                            // the pop scans keys[0..n): squeeze out popped entries once the ring passes 64 slots and at least half are holes
                            if (vq.n + cnt > rp.variant_cap || (vq.n + cnt > 64u && vq.live * 2u <= vq.n)) { kj_vq_compact<LONG>(cx, vq); }
                            if (vq.n + cnt > rp.variant_cap) { if (w.lane == 0) kj_flag_error(cx, 4u); }
                            else {
                                const uint32_t rk = (uint32_t)kj_popc(okmask & lanemask_lt(w.lane));
                                KjVariant<LONG>* V = vq.v + (vq.n + rk);           // dereferenced by `ok` lanes only
                                // the parent's substitutions that survive the truncation, then the new one
                                uint32_t ns = 0;
                                KJ_ROLLED
                                for (uint32_t u = 0; u < nsub; u++) {
                                    const uint32_t sv = psub[u];
                                    if ((sv >> 5) < new_len) { if (ok) V->subs[ns] = sv; ns++; }
                                }
                                if (ok) {
                                    V->subs[ns] = (pos << 5) | sub;
                                    V->lo = (uint64_t)lo; V->hi = (uint64_t)hi; V->pay = kj_qpay<LONG>(arr, true, start, new_len);
                                    V->diff = diff + (int)tb.b62[o][sub] - (int)tb.b62[sub][sub];
                                    V->matchlen = (PosT)(sm.ql + 1u); V->num_mm = (uint8_t)(ns + 1u); V->pad = 0; V->pad2 = 0;
                                    vq.key(vq.n + rk) = kj_qkey<LONG>((uint32_t)after, (LONG ? KJ_ORDER_LATE_LONG : KJ_ORDER_LATE) + q.late + rk);
                                }
                                vq.n += cnt; vq.live += cnt; q.late += cnt;
#if defined(KJ_EMU)
                                if (w.lane == 0) kj_emu_stats.var_pushed += cnt;
#endif
                            }
                        }
                        w.sync();
                    }
                }
                if (nmem > 1) break;
                c0 = c1;
            }
        }

        if (cls[0].ql < rp.m) continue;                                    // "Match ... is too short" (482-488)

        // ---------------- eval_match_scores (751-797): [class0: f2..fn][class1: f2..fn]...[heads, last class first]
        KjKept* bl = (KjKept*)(cx.smem + cx.L.kept_off);                   // best_matches_SI (<= 20)
        if (small) {
            // candidates = the classes with ql >= m, a prefix of cls (sorted by descending length)
            const uint32_t candmask = w.ballot((uint32_t)w.lane < nrec && my_ql >= rp.m);
            const uint32_t ncand = (uint32_t)kj_popc(candmask), K = (uint32_t)kj_popc(heads & candmask);
            // evaluation position of candidate t: non-heads keep their relative order, heads go last in reverse class order
            const uint32_t t = (uint32_t)w.lane;
            if (t < ncand) {
                const Match r = cls[t]; const bool head = (heads >> t) & 1u;
                const uint32_t cidx = (uint32_t)kj_popc(heads & ((2u << t) - 1u)) - 1u;           // class index of t
                const uint32_t pos = head ? (ncand - K) + (K - 1u - cidx) : t - (cidx + 1u);
                int sc = (int)pre[r.qi + r.ql] - (int)pre[r.qi] + diff; if (sc < 0) sc = 0;
                res[pos].lo = r.lo | ((uint64_t)r.qi << QI_SHIFT); res[pos].len = r.len; res[pos].qi = LONG ? (PosT)sc : (PosT)(sc > 65535 ? 65535 : sc); res[pos].ql = r.ql;      // (the match start rides in the free top bits of lo: the verbose output needs it)
            }
            w.sync();
            // the sequential best-list update of the reference, closed form: the list ends up holding the entries that equal the final
            // maximum, in evaluation order, as long as fewer than 20 are held (a higher score empties the list first)
            Match e; e.lo = 0; e.len = 0; e.qi = 0; e.ql = 0; if (t < ncand) e = res[t];
            const uint32_t sc = t < ncand ? (uint32_t)e.qi : 0u; const bool valid = t < ncand && sc >= rp.min_score;
            const uint32_t mx = warp_max_u32(w, valid ? sc : 0u);
            if (mx > 0 && mx >= best) {
                if (mx > best) { best = mx; nbest = 0; cx.text_len = 0; }
                const uint32_t eq = w.ballot(valid && sc == mx);
                const uint32_t slot = nbest + (uint32_t)kj_popc(eq & lanemask_lt(w.lane));
                const bool take = valid && sc == mx && slot < KJ_MAX_BEST_SI;
                if (take) { bl[slot].lo = e.lo & LO_MASK; bl[slot].len = e.len; bl[slot].aux = 0; }
                if (cx.text) {       // best_matches (ConsumerThread.cpp:779-790): the matched text of every entry of the best list, in list order
                    const uint32_t mylen = take ? (uint32_t)e.ql + 1u : 0u; const uint32_t endp = kj_scan_incl(w, mylen);
                    const uint32_t at = cx.text_len + endp - mylen, tot = w.shfl(endp, 31);
                    if (cx.text_len + tot > cx.text_cap) { if (w.lane == 0) kj_flag_error(cx, 128u); }
                    else {
                        if (take) { const uint32_t qi0 = (uint32_t)(e.lo >> QI_SHIFT); for (uint32_t u = 0; u + 1u < mylen; u++) cx.text[at + u] = tb.letters[frag[qi0 + u]]; cx.text[at + mylen - 1u] = ','; }
                        cx.text_len += tot;
                    }
                }
                nbest += (uint32_t)kj_popc(eq); if (nbest > KJ_MAX_BEST_SI) nbest = KJ_MAX_BEST_SI;
            }
            w.sync();
        } else {
            uint32_t K = 0, ncand = 0;                                     // classes with ql >= m, members in them
            { uint32_t c0 = 0; while (c0 < nrec && cls[c0].ql >= rp.m) { uint32_t c1 = c0 + 1; while (c1 < nrec && cls[c1].ql == cls[c0].ql) c1++; K++; ncand = c1; c0 = c1; } }
            KJ_ROLLED
            for (uint32_t b = 0; b < ncand; b += 32) {
                uint32_t t = b + (uint32_t)w.lane;
                if (t < ncand) {
                    Match r = cls[t]; bool head = (t == 0) || cls[t - 1].ql != r.ql;
                    uint32_t cidx = 0, heads_before = 0;                   // class index of t, number of heads at indices < t
                    KJ_ROLLED
                    for (uint32_t u = 1; u <= t; u++) if (cls[u].ql != cls[u - 1].ql) cidx++;
                    heads_before = cidx + (head ? 0u : 1u);
                    uint32_t pos = head ? (ncand - K) + (K - 1u - cidx) : t - heads_before;
                    int sc = (int)pre[r.qi + r.ql] - (int)pre[r.qi] + diff; if (sc < 0) sc = 0;
                    res[pos].lo = r.lo | ((uint64_t)r.qi << QI_SHIFT); res[pos].len = r.len; res[pos].qi = LONG ? (PosT)sc : (PosT)(sc > 65535 ? 65535 : sc); res[pos].ql = r.ql;
                }
            }
            w.sync();
            KJ_ROLLED
            for (uint32_t t = 0; t < ncand; t++) {
                const Match r = res[t]; const uint32_t sc = r.qi;
                if (sc < rp.min_score) continue;
                bool took = false;
                if (sc > best) { best = sc; nbest = 0; cx.text_len = 0; if (w.lane == 0) { bl[0].lo = r.lo & LO_MASK; bl[0].len = r.len; bl[0].aux = 0; } nbest = 1; took = true; }
                else if (sc == best && nbest < KJ_MAX_BEST_SI) { if (w.lane == 0) { bl[nbest].lo = r.lo & LO_MASK; bl[nbest].len = r.len; bl[nbest].aux = 0; } nbest++; took = true; }
                if (took && cx.text) {
                    const uint32_t at = kj_emit_text(w, cx.text, cx.text_len, cx.text_cap, frag + (uint32_t)(r.lo >> QI_SHIFT), 1u, r.ql, tb.letters);
                    if (at == 0xffffffffu) { if (w.lane == 0) kj_flag_error(cx, 128u); } else cx.text_len = at;
                }
            }
            w.sync();
        }
    }

    if (nbest == 0) return KJ_TAX_BAD;
    if (rp.use_evalue) {                                                   // E-value gate (500-513) as an integer threshold
        // minimal passing score = number of score break points below the query length (kj_build_evalue_breaks)
        uint32_t thr = 0;
        KJ_ROLLED
        for (uint32_t b = 0; b < rp.n_ev_breaks; b += 32) {
            const uint32_t k = b + (uint32_t)w.lane;
            const uint32_t below = w.ballot(k < rp.n_ev_breaks && rp.ev_breaks[k] < query_len);
            thr += (uint32_t)kj_popc(below);
            if (below != 0xffffffffu) break;                               // breaks ascend: the first lane that is not below ends the count
        }
        if (best < thr) return KJ_TAX_BAD;
    }
    w.sync();
    uint32_t t = kj_ids_and_lca<IdxT>(cx, nbest);
    if (t != KJ_TAX_BAD) best_out = best;
    return t;
}
