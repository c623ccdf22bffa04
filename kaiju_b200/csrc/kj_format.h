// kj_format.h -- the per-read output line of kj_classify_files (kj_fmt_len / kj_fmt_write in kj_ingest.h), one definition for the device and
// the host (the CPU test restates the reference's ostream formatting and compares it with this code, tests/test_format_lines.py).
//
// Formats (include/kaiju_b200.h KJ_OUT_*; the reference's lines):
//   0 KJ_OUT_KAIJU     "C\t<name>\t<taxid>\n" / "U\t<name>\t0\n"                                   (ConsumerThread.cpp:724-739)
//   1 KJ_OUT_KAIJU_IDS  C: + "\t<best>\t<id>,<id>,...,"
//   2 KJ_OUT_KAIJU_V    C: "C\t<name>\t<taxid>\t<best>\t<id>,...,\t<accession>,...,\t<fragments>\n" (ConsumerThread.cpp:527-536, 614-623)
//   3 KJ_OUT_NAMES     "C\t<name>\t<best>\t<label>,...,\t\n"; "U\t<name>\t0\n" for a read the front-end gate stops
//                      (ConsumerThreadx.cpp:202-207, ConsumerThreadp.cpp:16-20, 66-70), "U\t<name>\n" for one that matches nothing
//   4 KJ_OUT_NAMES_V   as 3 with the fragment strings after the last tab (ConsumerThreadx.cpp:108-113, 182-187)
#pragma once
#include <stdint.h>
#include "../../include/kaiju_b200.h"

#ifdef __CUDACC__
#define KJ_FMT_HD __host__ __device__ __forceinline__
#else
#define KJ_FMT_HD static inline
#endif

// Everything the line of read r is made of; arrays indexed by the read (relative to the rows being formatted), `frag` by r * frag_stride.
// Null where the format does not use it.
struct KjFmtIn {
    int fmt;
    const uint64_t* tax; const uint32_t* best;
    const uint64_t* ids; const uint8_t* nids;                       // formats 1-4: taxon-id set, KJ_MAX_MATCH_IDS per read, ascending
    const uint32_t* acc; const uint8_t* nacc;                       // format 2: accession ranks, KJ_MAX_MATCH_ACC per read, ascending
    const char* frag; uint64_t frag_stride; const uint32_t* fraglen;     // formats 2, 4: fragment strings
    const uint8_t* gate;                                            // formats 3, 4: 1 = the read is stopped by the front-end gate
    const char* names; const uint32_t* name_off;                    // read names: names[name_off[r], name_off[r + 1])
    const char* acc_str; const uint64_t* acc_off; uint64_t n_acc;   // KJ_STR_ACCESSION: string k = acc_str[acc_off[k], acc_off[k + 1])
    const char* lab_str; const uint64_t* lab_off; uint64_t n_lab;   // KJ_STR_TAXON, by dense taxon index
    const uint64_t* tax_id; uint32_t n_present, n_tax;              // the context's taxon ids (two ascending runs, kj_count_kernel): id -> dense index
};

KJ_FMT_HD uint32_t kj_fmt_dec_len(uint64_t v) { uint32_t l = 1; while (v >= 10) { v /= 10; l++; } return l; }
KJ_FMT_HD void kj_fmt_dec(char* p, uint64_t v, uint32_t l) { for (uint32_t k = l; k-- > 0;) { p[k] = (char)('0' + (uint32_t)(v % 10)); v /= 10; } }

// dense index of taxon id `id` (n_tax if unknown)
KJ_FMT_HD uint32_t kj_fmt_dense(const KjFmtIn& in, uint64_t id) {
    uint32_t lo = 0, hi = in.n_present;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (in.tax_id[mid] < id) lo = mid + 1; else hi = mid; }
    if (lo < in.n_present && in.tax_id[lo] == id) return lo;
    lo = in.n_present; hi = in.n_tax;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (in.tax_id[mid] < id) lo = mid + 1; else hi = mid; }
    return lo < in.n_tax && in.tax_id[lo] == id ? lo : in.n_tax;
}
// string k of a table: [*b, *b + length)
KJ_FMT_HD uint32_t kj_fmt_str(const char* blob, const uint64_t* off, uint64_t n, uint64_t k, const char** b) {
    if (k >= n) { *b = blob; return 0; }
    *b = blob + off[k]; return (uint32_t)(off[k + 1] - off[k]);
}
// 0: "U\t<name>\t0", 1: "U\t<name>" (name formats: passed the gate, matched nothing), 2: classified
KJ_FMT_HD int kj_fmt_status(const KjFmtIn& in, uint64_t r) {
    if (in.fmt < KJ_OUT_NAMES) return in.tax[r] ? 2 : 0;
    if (in.gate[r]) return 0;
    return in.tax[r] && in.nids[r] ? 2 : 1;
}

// The line of read r.  out == nullptr: only its length.  Otherwise it is written at out by a group of nl lanes (a warp, or nl = 1): lane 0 writes
// the separators and numbers, the string columns are copied lane-strided.  Every lane returns the length.
KJ_FMT_HD uint32_t kj_fmt_line(const KjFmtIn& in, uint64_t r, char* out, uint32_t lane, uint32_t nl) {
    const int st = kj_fmt_status(in, r); const bool w0 = out && lane == 0;
    uint32_t at = 0;
    auto ch = [&](char c) { if (w0) out[at] = c; at++; };
    auto str = [&](const char* s, uint32_t l) { if (out) for (uint32_t k = lane; k < l; k += nl) out[at + k] = s[k]; at += l; };
    auto dec = [&](uint64_t v) { const uint32_t l = kj_fmt_dec_len(v); if (w0) kj_fmt_dec(out + at, v, l); at += l; };
    ch(st == 2 ? 'C' : 'U'); ch('\t');
    str(in.names + in.name_off[r], in.name_off[r + 1] - in.name_off[r]);
    if (st == 0) { ch('\t'); ch('0'); ch('\n'); return at; }
    if (st == 1) { ch('\n'); return at; }
    ch('\t');
    const uint32_t ni = in.fmt >= KJ_OUT_KAIJU_IDS ? in.nids[r] : 0u; const uint64_t* ids = in.ids + r * KJ_MAX_MATCH_IDS;
    if (in.fmt < KJ_OUT_NAMES) {
        dec(in.tax[r]);
        if (in.fmt >= KJ_OUT_KAIJU_IDS) { ch('\t'); dec(in.best[r]); ch('\t'); for (uint32_t k = 0; k < ni; k++) { dec(ids[k]); ch(','); } }
        if (in.fmt == KJ_OUT_KAIJU_V) {
            ch('\t');
            for (uint32_t k = 0, na = in.nacc[r]; k < na; k++) { const char* s; const uint32_t l = kj_fmt_str(in.acc_str, in.acc_off, in.n_acc, in.acc[r * KJ_MAX_MATCH_ACC + k], &s); str(s, l); ch(','); }
            ch('\t'); str(in.frag + r * in.frag_stride, in.fraglen[r]);
        }
    } else {
        dec(in.best[r]); ch('\t');
        for (uint32_t k = 0; k < ni; k++) { const char* s; const uint32_t l = kj_fmt_str(in.lab_str, in.lab_off, in.n_lab, kj_fmt_dense(in, ids[k]), &s); str(s, l); ch(','); }
        ch('\t');
        if (in.fmt == KJ_OUT_NAMES_V) str(in.frag + r * in.frag_stride, in.fraglen[r]);
    }
    ch('\n');
    return at;
}

// BLOSUM62 self-score of an upper-case residue (calcScore, ConsumerThread.cpp:397-421); 0 for the letters that split a protein read
KJ_FMT_HD uint32_t kj_fmt_self_score(uint32_t c) {
    switch (c) { case 'A': return 4; case 'R': return 5; case 'N': return 6; case 'D': return 6; case 'C': return 9; case 'Q': return 5; case 'E': return 5; case 'G': return 6;
                 case 'H': return 8; case 'I': return 4; case 'L': return 4; case 'K': return 5; case 'M': return 5; case 'F': return 6; case 'P': return 7; case 'S': return 4;
                 case 'T': return 5; case 'W': return 11; case 'Y': return 7; case 'V': return 4; default: return 0; }
}
