// kj_host.cpp -- loaders for the reference's on-disk formats and the host-side transcoder to the device layout.
#include "kj_host.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <climits>
#include <atomic>
#include <thread>
#include <unordered_map>

std::string& kj_err() { static thread_local std::string e; return e; }
extern "C" const char* kj_last_error(void) { return kj_err().c_str(); }
extern "C" int kj_version(void) { return 101; }

// ------------------------------------------------------------------------------------------------
// .fmi  (written by kaiju-mkfmi, mkfmi.c:68-77): BWT header (bwt.c:40-45), suffix-array header + body
// (suffixArray.c:261-277, 325-328), FM index (fmicommon.h:175-184, compactfmi.c:176-179).
// ------------------------------------------------------------------------------------------------
namespace {
struct Reader {
    FILE* fp; bool ok = true;
    explicit Reader(FILE* f) : fp(f) {}
    template <class T> T get() { T v{}; if (fread(&v, sizeof(T), 1, fp) != 1) ok = false; return v; }
    void bytes(void* p, size_t n) { if (n && fread(p, 1, n, fp) != n) ok = false; }
    void skip(int64_t n) { if (fseeko(fp, (off_t)n, SEEK_CUR) != 0) ok = false; }
};
uint64_t taxon_of_name(const std::string& name) {
    // ConsumerThread.cpp:812-832: digits after the LAST '_', or the whole name when there is none
    const char* s = name.c_str(); const char* u = strrchr(s, '_');
    unsigned long v = strtoul(u ? u + 1 : s, nullptr, 10);
    return v == ULONG_MAX ? UINT64_MAX : (uint64_t)v;
}
}  // namespace

extern "C" int kj_fmi_load(const char* path, kj_fmi** out) {
    if (!path || !out) { kj_err() = "kj_fmi_load: null argument"; return KJ_ERR_ARG; }
    FILE* fp = fopen(path, "rb");
    if (!fp) { kj_err() = std::string("could not open ") + path; return KJ_ERR_IO; }
    // every count read from the file is checked against the file size before memory is allocated for it (corrupt headers)
    fseeko(fp, 0, SEEK_END); const int64_t fsize = (int64_t)ftello(fp); fseeko(fp, 0, SEEK_SET);
    kj_fmi* f = new kj_fmi(); Reader r(fp);
    f->len = r.get<int64_t>(); f->nseq = r.get<int32_t>(); f->alen = r.get<int32_t>();
    if (!r.ok || f->alen <= 1 || f->alen > 64 || f->nseq < 0 || f->len <= 0) { fclose(fp); delete f; kj_err() = "not a .fmi file (BWT header)"; return KJ_ERR_IO; }
    f->alphabet.resize((size_t)f->alen); r.bytes(&f->alphabet[0], (size_t)f->alen);
    f->sa_len = r.get<int64_t>(); f->ncheck = r.get<int64_t>(); f->chpt_exp = r.get<int32_t>(); f->nbytes = r.get<int32_t>();
    f->sbits = r.get<int32_t>(); f->pbits = r.get<int32_t>(); f->mask = r.get<int64_t>(); f->check = r.get<int64_t>();
    int32_t nseq2 = r.get<int32_t>();
    if (!r.ok || nseq2 != f->nseq || f->nbytes <= 0 || f->nbytes > 8 || f->ncheck < 0 || f->chpt_exp < 0 || f->chpt_exp > 30 ||
        (int64_t)f->nseq * 13 > fsize || f->ncheck > fsize / f->nbytes) { fclose(fp); delete f; kj_err() = "not a .fmi file (suffix-array header)"; return KJ_ERR_IO; }
    f->ids.resize((size_t)f->nseq); f->seq_taxon.resize((size_t)f->nseq);
    for (int32_t i = 0; i < f->nseq && r.ok; i++) {
        uint8_t l = r.get<uint8_t>(); std::string& s = f->ids[(size_t)i]; s.resize(l); r.bytes(l ? &s[0] : nullptr, l);
        f->seq_taxon[(size_t)i] = taxon_of_name(s);
    }
    {   // accessions (ConsumerThread.cpp:809-823): the name up to its last '_'; ranks in lexicographic order of the distinct strings
        std::vector<std::string> acc; acc.reserve((size_t)f->nseq);
        for (const std::string& s : f->ids) { const size_t u = s.rfind('_'); if (u != std::string::npos) acc.push_back(s.substr(0, u)); }
        std::sort(acc.begin(), acc.end()); acc.erase(std::unique(acc.begin(), acc.end()), acc.end());
        f->acc_names.swap(acc); f->seq_acc.assign((size_t)f->nseq, 0xffffffffu);
        for (int32_t i = 0; i < f->nseq; i++) { const std::string& s = f->ids[(size_t)i]; const size_t u = s.rfind('_');
            if (u != std::string::npos) f->seq_acc[(size_t)i] = (uint32_t)(std::lower_bound(f->acc_names.begin(), f->acc_names.end(), s.substr(0, u)) - f->acc_names.begin()); }
    }
    r.skip((int64_t)f->nseq * 4); r.skip((int64_t)f->nseq * 8);          // seqTermOrder, seqlengths: not needed for classification
    f->sa.resize((size_t)(f->ncheck * f->nbytes)); r.bytes(f->sa.data(), f->sa.size());
    int32_t alen2 = r.get<int32_t>(); f->bwtlen = r.get<int64_t>(); f->N1 = r.get<int32_t>(); f->N2 = r.get<int32_t>();
    if (!r.ok || alen2 != f->alen || f->bwtlen <= 0 || f->bwtlen > fsize || f->N1 < 0 || f->N2 < 0) { fclose(fp); delete f; kj_err() = "not a .fmi file (FMI header)"; return KJ_ERR_IO; }
    f->bwt.resize((size_t)f->bwtlen); r.bytes(f->bwt.data(), f->bwt.size());
    r.skip((int64_t)f->N1 * f->alen * 8); r.skip((int64_t)f->N2 * f->alen * 2);   // index1/index2: rank tables are rebuilt in the device layout
    f->startLcode.resize((size_t)f->alen + 1); r.bytes(f->startLcode.data(), sizeof(int32_t) * ((size_t)f->alen + 1));
    bool ok = r.ok; fclose(fp);
    if (!ok) { delete f; kj_err() = "truncated .fmi file"; return KJ_ERR_IO; }
    *out = f; return KJ_OK;
}
extern "C" void kj_fmi_view(const kj_fmi* f, kj_index_view* v) {
    v->alen = f->alen; v->alphabet = f->alphabet.c_str(); v->bwtlen = f->bwtlen; v->bwt = f->bwt.data(); v->startLcode = f->startLcode.data();
    v->db_len = f->len; v->nseq = f->nseq; v->ncheck = f->ncheck; v->chpt_exp = f->chpt_exp; v->nbytes = f->nbytes; v->pbits = f->pbits;
    v->sa = f->sa.data(); v->seq_taxon = f->seq_taxon.data(); v->seq_accession = f->seq_acc.empty() ? nullptr : f->seq_acc.data();
}
extern "C" void kj_fmi_free(kj_fmi* f) { delete f; }
extern "C" const char* kj_fmi_accession(const kj_fmi* f, uint32_t rank) { return (f && rank < f->acc_names.size()) ? f->acc_names[rank].c_str() : nullptr; }
extern "C" const char* kj_fmi_seq_name(const kj_fmi* f, int32_t i) { return (f && i >= 0 && i < f->nseq) ? f->ids[(size_t)i].c_str() : nullptr; }

// nodes.dmp (parseNodesDmp, util.cpp:79-99): first integer = node, next integer = parent; bad lines skipped
extern "C" int kj_nodes_load(const char* path, kj_nodes** out) {
    if (!path || !out) { kj_err() = "kj_nodes_load: null argument"; return KJ_ERR_ARG; }
    FILE* fp = fopen(path, "r");
    if (!fp) { kj_err() = std::string("could not open ") + path; return KJ_ERR_IO; }
    kj_nodes* t = new kj_nodes(); char* line = nullptr; size_t cap = 0; ssize_t n;
    while ((n = getline(&line, &cap, fp)) > 0) {
        const char* p = line; if (*p < '0' || *p > '9') continue;
        char* e; uint64_t node = strtoull(p, &e, 10); p = e;
        while (*p && (*p < '0' || *p > '9')) p++;
        if (!*p) continue;
        t->node.push_back(node); t->parent.push_back(strtoull(p, nullptr, 10));
    }
    free(line); fclose(fp); *out = t; return KJ_OK;
}
extern "C" void kj_nodes_view(const kj_nodes* t, kj_taxonomy_view* v) { v->n = t->node.size(); v->node = t->node.data(); v->parent = t->parent.data(); }
extern "C" void kj_nodes_free(kj_nodes* t) { delete t; }

// ------------------------------------------------------------------------------------------------
// tables
// ------------------------------------------------------------------------------------------------
namespace {
const char* kAaOrder = "ARNDCQEGHILKMFPSTWYV";                     // aa2int (ConsumerThread.cpp:45-65)
const int8_t kB62[20][20] = {                                       // BLOSUM62 in kAaOrder (ConsumerThread.cpp:66-107)
 { 4,-1,-2,-2, 0,-1,-1, 0,-2,-1,-1,-1,-1,-2,-1, 1, 0,-3,-2, 0}, {-1, 5, 0,-2,-3, 1, 0,-2, 0,-3,-2, 2,-1,-3,-2,-1,-1,-3,-2,-3},
 {-2, 0, 6, 1,-3, 0, 0, 0, 1,-3,-3, 0,-2,-3,-2, 1, 0,-4,-2,-3}, {-2,-2, 1, 6,-3, 0, 2,-1,-1,-3,-4,-1,-3,-3,-1, 0,-1,-4,-3,-3},
 { 0,-3,-3,-3, 9,-3,-4,-3,-3,-1,-1,-3,-1,-2,-3,-1,-1,-2,-2,-1}, {-1, 1, 0, 0,-3, 5, 2,-2, 0,-3,-2, 1, 0,-3,-1, 0,-1,-2,-1,-2},
 {-1, 0, 0, 2,-4, 2, 5,-2, 0,-3,-3, 1,-2,-3,-1, 0,-1,-3,-2,-2}, { 0,-2, 0,-1,-3,-2,-2, 6,-2,-4,-4,-2,-3,-3,-2, 0,-2,-2,-3,-3},
 {-2, 0, 1,-1,-3, 0, 0,-2, 8,-3,-3,-1,-2,-1,-2,-1,-2,-2, 2,-3}, {-1,-3,-3,-3,-1,-3,-3,-4,-3, 4, 2,-3, 1, 0,-3,-2,-1,-3,-1, 3},
 {-1,-2,-3,-4,-1,-2,-3,-4,-3, 2, 4,-2, 2, 0,-3,-2,-1,-2,-1, 1}, {-1, 2, 0,-1,-3, 1, 1,-2,-1,-3,-2, 5,-1,-3,-1, 0,-1,-3,-2,-2},
 {-1,-1,-2,-3,-1, 0,-2,-3,-2, 1, 2,-1, 5, 0,-2,-1,-1,-1,-1, 1}, {-2,-3,-3,-3,-2,-3,-3,-3,-1, 0, 0,-3, 0, 6,-4,-2,-2, 1, 3,-1},
 {-1,-2,-2,-1,-3,-1,-1,-2,-2,-3,-3,-1,-2,-4, 7,-1,-1,-4,-3,-2}, { 1,-1, 1, 0,-1, 0, 0, 0,-1,-2,-2, 0,-1,-2,-1, 4, 1,-3,-2,-2},
 { 0,-1, 0,-1,-1,-1,-1,-2,-2,-1,-1,-1,-1,-2,-1, 1, 5,-2,-2, 0}, {-3,-3,-4,-4,-2,-2,-3,-2,-2,-3,-2,-3,-1, 1,-4,-3,-2,11, 2,-3},
 {-2,-2,-2,-3,-2,-1,-2,-3, 2,-1,-1,-2,-1, 3,-3,-2,-2, 2, 7,-1}, { 0,-3,-3,-3,-1,-2,-2,-3,-3, 3, 1,-2, 1,-1,-2,-2, 0,-3,-1, 4} };
// substitution try-order per residue (the reference's blosum_subst map, ConsumerThread.cpp:10-30)
const char* kSubst[20] = {
 "A:SVTGCPMKLIEQRYFHDNW", "R:KQHENTSMAYPLGDVWFIC", "N:SHDTKGEQRYPMAVFLICW", "D:ENSQTPKHGRAVYFMICWL", "C:AVTSMLIYWFPKHGQDNRE",
 "Q:EKRSMHDNYTPAVWLGFIC", "E:QDKSHNRTPAVYMGWFLIC", "G:SNADWTPKHEQRVYFMCLI", "H:YNEQRSFKDWTPMGAVLIC", "I:VLMFYTCASWPKHEQDNRG",
 "L:MIVFYTCAWSKQRPHENGD", "K:REQSNTPMHDAVYLGWFIC", "M:LVIFQYWTSKCRAPHENGD", "F:YWMLIVHTSCAKGEQDNRP", "P:TSKEQDAVMHGNRYLICWF",
 "S:TNAKGEQDPMHCRVYFLIW", "T:SVNAPMKLIEQCDRYWFHG", "W:YFMTLHGQCVSKIERAPDN", "Y:FWHVMLIQTSKECNRAPGD", "V:IMLTAYFCSPKEQWHGDNR" };
// standard genetic code, index n0<<4|n1<<2|n2 with A0 C1 G2 T3 (the reference's codon2aa, ConsumerThread.cpp:117-181)
const char* kCode = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF";

int build_tables(const std::string& alphabet, KjTables& tb) {
    memset(&tb, 0, sizeof(tb));
    const int alen = (int)alphabet.size();
    // translation_table (sequence.c:68-97): letters not in the alphabet map to the last index
    uint8_t trans[256]; memset(trans, (uint8_t)(alen - 1), sizeof trans);
    for (int a = 0; a < alen; a++) trans[(uint8_t)alphabet[(size_t)a]] = (uint8_t)a;
    for (int c = 0; c < 64; c++) tb.codon_aa[c] = kCode[c] == '*' ? 0 : trans[(uint8_t)kCode[c]];
    for (int a = 0; a < alen && a < KJ_MAX_ALEN; a++) tb.letters[a] = alphabet[(size_t)a];
    for (const char* v = "ACDEFGHIKLMNPQRSTVWY"; *v; v++) tb.aa_index[*v - 'A'] = trans[(uint8_t)*v];     // the valid set of a protein read (ConsumerThread.cpp:664)
    int ai_of[256]; for (int i = 0; i < 256; i++) ai_of[i] = -1;
    for (int i = 0; i < 20; i++) ai_of[(uint8_t)kAaOrder[i]] = i;
    for (int a = 0; a < alen; a++) for (int b = 0; b < alen; b++) {
        int ia = ai_of[(uint8_t)alphabet[(size_t)a]], ib = ai_of[(uint8_t)alphabet[(size_t)b]];
        tb.b62[a][b] = (ia >= 0 && ib >= 0) ? kB62[ia][ib] : 0;
    }
    for (int i = 0; i < 20; i++) {
        int a = trans[(uint8_t)kSubst[i][0]];
        for (int k = 0; k < 19; k++) tb.subst[a][k] = trans[(uint8_t)kSubst[i][2 + k]];
    }
    // SEG window entropy in fixed point; verify on all partitions of 12 that the integer decisions equal
    // the reference's FP64 decisions (s_Entropy, blast_seg.c:1596-1626; kSegLocut 2.2, kSegHicut 2.5)
    for (int c = 1; c <= KJ_SEG_WINDOW; c++) tb.seg_logfix[c] = (int32_t)llround(log2(12.0 / c) * 16777216.0);
    tb.seg_locut_fix = (int32_t)llround(2.2 * 12.0 * 16777216.0);
    tb.seg_hicut_fix = (int32_t)llround(2.5 * 12.0 * 16777216.0);
    int part[13]; bool okp = true;
    // enumerate partitions of 12 (descending parts)
    struct Rec { static void go(int left, int maxp, int* part, int n, const KjTables& tb, bool& ok) {
        if (left == 0) {
            double ent = 0.0; int64_t x = 0;
            for (int i = 0; i < n; i++) { ent += ((double)part[i]) * log(((double)part[i]) / 12.0) / 0.69314718055994530941723212145818; x += (int64_t)part[i] * tb.seg_logfix[part[i]]; }
            ent = fabs(ent / 12.0);
            if ((ent <= 2.2) != (x <= tb.seg_locut_fix) || (ent > 2.5) != (x > tb.seg_hicut_fix)) ok = false;
            if (n >= 8 && !(ent > 2.5)) ok = false;          // the kernel's >= 8 distinct residues shortcut
            return;
        }
        for (int p = std::min(left, maxp); p >= 1; p--) { part[n] = p; go(left - p, p, part, n + 1, tb, ok); }
    } };
    Rec::go(12, 12, part, 0, tb, okp);
    if (!okp) { kj_err() = "SEG fixed-point entropy classes disagree with FP64"; return KJ_ERR_UNSUPPORTED; }
    return KJ_OK;
}
}  // namespace

extern "C" int kj_check_params_c(const kj_params* p) { return p ? kj_check_params(*p) : KJ_ERR_ARG; }
int kj_check_params(const kj_params& p) {
    if (p.mode != 0 && p.mode != 1) { kj_err() = "mode must be 0 (MEM) or 1 (GREEDY)"; return KJ_ERR_ARG; }
    if (p.min_fragment_length == 0 || p.min_fragment_length > 1000) { kj_err() = "min_fragment_length out of range"; return KJ_ERR_ARG; }
    if (p.mode == 0 && p.use_evalue) { kj_err() = "E-value calculation is only possible in Greedy mode"; return KJ_ERR_ARG; }   // kaiju.cpp:202
    if (p.mode == 1 && p.mismatches > KJ_MAX_MM) { kj_err() = "more than 8 mismatches (-e) are not supported"; return KJ_ERR_UNSUPPORTED; }
    if (p.mode == 1 && (p.min_score == 0 || p.seed_length == 0)) { kj_err() = "min_score and seed_length must be > 0"; return KJ_ERR_ARG; }
    if (p.use_evalue && !(p.min_evalue > 0.0)) { kj_err() = "E-value threshold must be greater than 0"; return KJ_ERR_ARG; }
    return KJ_OK;
}

// ------------------------------------------------------------------------------------------------
// transcoder: reference in-memory index -> device layout
// ------------------------------------------------------------------------------------------------
static inline uint64_t host_rank(const KjHostIndex& H, uint32_t c, uint64_t k);
// Everything of the device index that is small or independent of the BWT body: tables, byte-code -> letter map, geometry (layout choice,
// quirk flag), the re-indexed taxonomy, sequence -> taxon, suffix-array sampling parameters, ln(n!) table.  `copies` > 1 describes the
// collection in which every sequence occurs `copies` times in a row (kj_create_scaled): bwtlen, nseq and db_len scale, sequence
// K*s + c inherits the taxon of sequence s.
int kj_build_host_meta(const kj_index_view& v, const kj_taxonomy_view& t, uint32_t copies, KjHostIndex& H, uint8_t lcode[256]) {
    if (!v.bwt || !v.startLcode || !v.alphabet || !v.sa || !v.seq_taxon || v.bwtlen <= 0 || v.nseq < 0 || v.ncheck < 0 || v.chpt_exp < 0 || v.chpt_exp > 30 || v.nbytes <= 0 || v.nbytes > 8) {
        kj_err() = "kj_create: incomplete index view"; return KJ_ERR_ARG; }
    if (v.alen < 2 || v.alen > KJ_MAX_ALEN) { kj_err() = "alphabet size not supported"; return KJ_ERR_UNSUPPORTED; }
    if (copies < 1 || copies > 65536) { kj_err() = "copies out of range"; return KJ_ERR_ARG; }
    const int alen = v.alen; const uint64_t n = (uint64_t)v.bwtlen * copies;
    if (n >= (1ull << 38)) { kj_err() = "index too large (>= 2^38 rows)"; return KJ_ERR_UNSUPPORTED; }      // checked before anything large is built
    if ((uint64_t)v.nseq * copies >= 0x7fffffffull) { kj_err() = "too many sequences"; return KJ_ERR_UNSUPPORTED; }
    H.alen = alen; H.bwtlen = n; H.nseq = (uint32_t)((uint64_t)v.nseq * copies); H.db_length = (double)(v.db_len - v.nseq) * (double)copies;
    int rc = build_tables(std::string(v.alphabet, (size_t)alen), H.tables); if (rc) return rc;
    // byte code -> letter (fmi_fill_codes, compactfmi.c:75-89)
    memset(lcode, 0, 256);
    for (int a = 0; a < alen; a++) {
        int s = v.startLcode[a], e = v.startLcode[a + 1];
        if (s < 0 || e > 256 || s > e) { kj_err() = "corrupt startLcode"; return KJ_ERR_IO; }
        for (int k = s; k < e; k++) lcode[k] = (uint8_t)a;
    }
    // KJ_FORCE_WIDE: exercise the 64-bit kernels on small test indexes.  Indexes with the reference's checkpoint quirk (below) also
    // take the 64-bit kernels: only those carry the rank correction, so that ordinary indexes pay nothing for the 1-in-65536 case.
    // KJ_FORCE_COMPACT: the compact layout (kj_layout.h) for any index, to test it on small ones; otherwise it is chosen on the device when the
    // wide construction does not fit in HBM (kj_choose_layout).
    const bool quirk = (n & 65535ull) == 0 && n >= 131072ull;
    H.wide = getenv("KJ_FORCE_COMPACT") ? KJ_LAYOUT_COMPACT : (n >= 0xffffff00ull || getenv("KJ_FORCE_WIDE") || quirk) ? KJ_LAYOUT_WIDE : KJ_LAYOUT_NARROW;
    H.nb = n / kj_rank_rows(H.wide) + 1;
    // The reference's checkpoint quirk (fmicommon.h:60-73, 88-89, 114-158; pinned against the reference's own FMindex/get_suffix and CLI in
    // tests/test_oracle_vs_ref.py::test_bwtlen_multiple_of_65536):
    // with bwtlen = m * 2^16, m >= 2, positions k >= bwtlen - 128 resolve to the first-level row that holds C[] instead of counts, so
    // FMindex(c, k) comes out smaller by #c in BWT[0, bwtlen - 2^16).  Reproduced, not fixed: results must equal the reference's.
    H.quirk_lo = quirk ? n - 128ull : ~0ull; memset(H.quirk_d, 0, sizeof H.quirk_d);      // quirk_d is filled once ranks exist
    // ---- taxonomy re-indexing
    std::unordered_map<uint64_t, uint64_t> par_of; par_of.reserve((size_t)t.n * 2 + 16);
    for (uint64_t i = 0; i < t.n; i++) par_of.emplace(t.node[i], t.parent[i]);          // emplace keeps the first (util.cpp:91)
    std::vector<uint64_t> present; present.reserve(par_of.size());
    for (auto& kv : par_of) present.push_back(kv.first);
    std::sort(present.begin(), present.end());
    std::vector<uint64_t> extra;
    for (auto& kv : par_of) if (!par_of.count(kv.second)) extra.push_back(kv.second);
    for (int32_t i = 0; i < v.nseq; i++) { uint64_t x = v.seq_taxon[i]; if (x != UINT64_MAX && !par_of.count(x)) extra.push_back(x); }
    std::sort(extra.begin(), extra.end()); extra.erase(std::unique(extra.begin(), extra.end()), extra.end());
    const size_t np = present.size(), nt = np + extra.size();
    if (nt >= 0xfffffff0ull) { kj_err() = "too many taxa"; return KJ_ERR_UNSUPPORTED; }
    H.tax_id = present; H.tax_id.insert(H.tax_id.end(), extra.begin(), extra.end()); H.n_present = (uint32_t)np;
    auto index_of = [&](uint64_t id) -> uint32_t {
        auto it = std::lower_bound(present.begin(), present.end(), id);
        if (it != present.end() && *it == id) return (uint32_t)(it - present.begin());
        auto jt = std::lower_bound(extra.begin(), extra.end(), id);
        return (uint32_t)(np + (size_t)(jt - extra.begin()));
    };
    H.tax_parent.resize(nt); H.tax_depth.assign(nt, 0);
    for (size_t i = 0; i < np; i++) H.tax_parent[i] = index_of(par_of[present[i]]);
    for (size_t i = np; i < nt; i++) H.tax_parent[i] = (uint32_t)i;
    // depth = 1 + hops to the self-parent root or to a node missing from nodes.dmp (util.cpp:217-222)
    {
        std::vector<uint32_t> stack;
        for (size_t i = 0; i < np; i++) {
            if (H.tax_depth[i]) continue;
            uint32_t cur = (uint32_t)i; stack.clear();
            while (true) {
                if (cur >= np) { break; }                                   // absent node: contributes depth "0" below it -> child depth 1+... handled on unwind
                if (H.tax_depth[cur]) break;
                if (H.tax_parent[cur] == cur) { H.tax_depth[cur] = 1; break; }
                if (stack.size() > nt) { kj_err() = "cycle in nodes.dmp"; return KJ_ERR_IO; }
                stack.push_back(cur); cur = H.tax_parent[cur];
            }
            // depth of `cur`: present -> tax_depth[cur]; absent -> the hop onto it still counted (depth++ then loop ends)
            uint32_t d = cur >= np ? 1u : H.tax_depth[cur];
            while (!stack.empty()) { uint32_t x = stack.back(); stack.pop_back(); d += 1; H.tax_depth[x] = d; }
        }
    }
    // ---- sequence -> compact taxon; sampled SA -> compact taxon
    H.seq_tax.resize((size_t)v.nseq * copies);
    for (int32_t i = 0; i < v.nseq; i++) { const uint32_t x = v.seq_taxon[i] == UINT64_MAX ? KJ_TAX_BAD : index_of(v.seq_taxon[i]); for (uint32_t c = 0; c < copies; c++) H.seq_tax[(size_t)i * copies + c] = x; }
    H.seq_acc.clear(); H.sa_acc.clear();
    if (v.seq_accession && copies == 1) H.seq_acc.assign(v.seq_accession, v.seq_accession + v.nseq);
    H.sa_exp = v.chpt_exp; H.sa_check = (1ull << v.chpt_exp) - 1ull;                         // suffixArray_set_masks (suffixArray.c:34-37)
    H.sa_bias = ((int64_t)((int64_t)H.nseq - 1) >> v.chpt_exp) + 1;                          // bwt.c:115-116
    kj_lnfact_table(H.lnfact);
    return KJ_OK;
}

// ln(n!) exactly as the reference's s_lnfact (blast_seg.c:1852-1856): its table lnfact[0..10000] ("%.6f" prints of lgamma, blast_seg.c:53-1306), and
// Stirling's formula above it.  The long-read kernels trim SEG regions of up to a fragment's length, so the table runs to the longest fragment of a
// KJ_MAX_LONG_READ_LEN read; the first KJ_LNFACT_REF entries are the only ones a device-native index file stores.
void kj_lnfact_table(std::vector<double>& t) {
    const size_t had = t.size() >= KJ_LNFACT_REF ? KJ_LNFACT_REF : 0;
    t.resize(KJ_LNFACT_LEN);
    if (!had) {
        for (int i = 0; i < KJ_LNFACT_REF; i++) { char b[64]; snprintf(b, sizeof b, "%.6f", lgamma((double)i + 1.0)); t[(size_t)i] = strtod(b, nullptr); }
        t[0] = t[1] = 0.0;
    }
    for (int n = KJ_LNFACT_REF; n < KJ_LNFACT_LEN; n++) t[(size_t)n] = ((n + 0.5) * log((double)n) - n + 0.9189385332);
}

int kj_build_host_index(const kj_index_view& v, const kj_taxonomy_view& t, KjHostIndex& H) {
    uint8_t lcode[256];
    int rc = kj_build_host_meta(v, t, 1, H, lcode); if (rc) return rc;
    const int alen = v.alen; const uint64_t n = (uint64_t)v.bwtlen; const uint64_t nb = H.nb;
    const bool quirk = H.quirk_lo != ~0ull;
    // rank records + packed letters, chunked over threads
    const uint32_t RB = kj_rank_rows(H.wide), RW = kj_rank_words(H.wide);
    const uint64_t CH = 192ull * 2048;                                  // positions per chunk (multiple of 192, 64 and 12)
    const uint64_t nch = (n + CH - 1) / CH;
    std::vector<uint64_t> ccount((size_t)(nch + 1) * alen, 0);
    unsigned nthr = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    auto par = [&](auto fn) {
        std::vector<std::thread> th; for (unsigned tI = 0; tI < nthr; tI++) th.emplace_back([&, tI] { for (uint64_t c = tI; c < nch; c += nthr) fn(c); });
        for (auto& x : th) x.join();
    };
    par([&](uint64_t c) { uint64_t* cc = &ccount[(size_t)(c + 1) * alen]; uint64_t e = std::min(n, (c + 1) * CH); for (uint64_t k = c * CH; k < e; k++) cc[lcode[v.bwt[k]]]++; });
    for (uint64_t c = 1; c <= nch; c++) for (int a = 0; a < alen; a++) ccount[(size_t)c * alen + a] += ccount[(size_t)(c - 1) * alen + a];
    const uint64_t* total = &ccount[(size_t)nch * alen];
    H.C[0] = 0; for (int a = 0; a < alen; a++) H.C[a + 1] = H.C[a] + total[a];
    if (H.C[alen] != n) { kj_err() = "letter counts do not add up"; return KJ_ERR_IO; }
    try { H.rank.assign((size_t)kj_rank_array_words(H.wide, alen, nb), 0ull); H.letters.assign((size_t)kj_letters_words(H.wide, n), 0); }
    catch (...) { kj_err() = "out of host memory building the rank table"; return KJ_ERR_NOMEM; }
    if (H.wide == KJ_LAYOUT_COMPACT) {
        // records: 5 bit-planes per 64-row half + the counts from the superblock start to the record's midpoint; then the superblock table
        const uint64_t nsb = kj_csb_count(n); std::vector<uint64_t> sbt((size_t)nsb * KJ_CSB_STRIDE, 0);
        std::vector<std::thread> th;
        for (unsigned tI = 0; tI < nthr; tI++) th.emplace_back([&, tI] {
            for (uint64_t sb = tI; sb < nsb; sb += nthr) {
                uint64_t cnt[KJ_CSB_STRIDE] = {0};
                for (uint64_t b = sb << (KJ_CSB_SHIFT - 7); b < nb && b < (sb + 1) << (KJ_CSB_SHIFT - 7); b++) {
                    uint64_t* R = &H.rank[(size_t)b * KJ_RANK_WORDS_COMPACT];
                    for (uint32_t i = 0; i < 128; i++) {
                        if (i == 64) for (int a = 0; a < KJ_CSB_STRIDE; a++) ((uint16_t*)(R + KJ_CPT_COUNT_WORD))[a] = (uint16_t)cnt[a];
                        const uint64_t k = b * 128 + i; const uint32_t l = k < n ? lcode[v.bwt[k]] : 31u;
                        if (k < n) cnt[l]++;
                        for (int bit = 0; bit < 5; bit++) R[5 * (i >> 6) + bit] |= (uint64_t)((l >> bit) & 1u) << (i & 63);
                    }
                }
                for (int a = 0; a < KJ_CSB_STRIDE; a++) sbt[(size_t)sb * KJ_CSB_STRIDE + a] = cnt[a];
            }
        });
        for (auto& x : th) x.join();
        uint64_t run[KJ_CSB_STRIDE] = {0};
        for (uint64_t sb = 0; sb < nsb; sb++) for (int a = 0; a < KJ_CSB_STRIDE; a++) {
            H.letters[(size_t)sb * KJ_CSB_STRIDE + a] = (a < alen ? H.C[a] : 0) + run[a]; run[a] += sbt[(size_t)sb * KJ_CSB_STRIDE + a]; }
    } else par([&](uint64_t c) {
        uint64_t run[KJ_MAX_ALEN]; for (int a = 0; a < alen; a++) run[a] = H.C[a] + ccount[(size_t)c * alen + a];
        uint64_t e = std::min(n, (c + 1) * CH);
        for (uint64_t b0 = c * CH; b0 < e; b0 += RB) {
            uint64_t b = b0 / RB, be = std::min(n, b0 + RB);
            for (int a = 0; a < alen; a++) H.rank[((size_t)a * nb + b) * RW] = run[a];
            for (uint64_t k = b0; k < be; k++) {
                uint32_t a = lcode[v.bwt[k]], r = (uint32_t)(k - b0);
                H.rank[((size_t)a * nb + b) * RW + 1u + (r >> 6)] |= 1ull << (r & 63);
                run[a]++;
            }
        }
        for (uint64_t k = c * CH; k < e; k++) H.letters[k / KJ_LETTERS_PER_WORD] |= (uint64_t)lcode[v.bwt[k]] << (5 * (k % KJ_LETTERS_PER_WORD));
    });
    // the record after the last letter (k == bwtlen lands there when bwtlen % RB == 0; otherwise the last partial block already exists)
    if (n % RB == 0 && H.wide != KJ_LAYOUT_COMPACT) for (int a = 0; a < alen; a++) H.rank[((size_t)a * nb + (nb - 1)) * RW] = H.C[a] + total[a];
    if (H.wide == KJ_LAYOUT_WIDE) {   // fold the in-block prefix popcounts into the header
        std::vector<std::thread> th; const size_t tot = (size_t)alen * nb;
        for (unsigned tI = 0; tI < nthr; tI++) th.emplace_back([&, tI] { for (size_t i = tI; i < tot; i += nthr) { uint64_t* B = &H.rank[i * 4];
            uint64_t p1 = (uint64_t)__builtin_popcountll(B[1]), p2 = p1 + (uint64_t)__builtin_popcountll(B[2]); B[0] = (B[0] & KJ_CNT_MASK) | (p1 << KJ_P1_SHIFT) | (p2 << KJ_P2_SHIFT); } });
        for (auto& x : th) x.join();
    }

    H.sa_tax.resize((size_t)v.ncheck); if (!H.seq_acc.empty()) H.sa_acc.resize((size_t)v.ncheck);
    {
        std::vector<std::thread> th; const uint64_t nc = (uint64_t)v.ncheck; std::atomic<bool> bad(false);
        for (unsigned tI = 0; tI < nthr; tI++) th.emplace_back([&, tI] {
            for (uint64_t e = tI; e < nc; e += nthr) {
                const uint8_t* p = v.sa + e * (uint64_t)v.nbytes; uint64_t val = 0;
                for (int b = 0; b < v.nbytes; b++) val = (val << 8) + p[b];                  // uchar2long (suffixArray.h:37-41)
                uint64_t seq = val >> v.pbits;
                if (seq >= (uint64_t)v.nseq) { bad = true; continue; }
                H.sa_tax[e] = H.seq_tax[seq];
                if (!H.seq_acc.empty()) H.sa_acc[e] = H.seq_acc[seq];
            }
        });
        for (auto& x : th) x.join();
        if (bad) { kj_err() = "corrupt suffix array (sequence number out of range)"; return KJ_ERR_IO; }
    }
    if (quirk) {
        for (int a = 0; a < alen; a++) H.quirk_d[a] = host_rank(H, (uint32_t)a, n - 65536ull) - H.C[a];
    }
    { const char* ek = getenv("KJ_KMER_K"); kj_build_kmer_table(H, ek ? atoi(ek) : kj_default_kmer_k(H.bwtlen)); }
    return KJ_OK;
}

// host-side rank on the device layout (used only to fill the k-mer table)
static inline uint64_t host_rank(const KjHostIndex& H, uint32_t c, uint64_t k) {
    if (H.wide == KJ_LAYOUT_COMPACT) {
        const uint64_t* R = &H.rank[(size_t)(k >> 7) * KJ_RANK_WORDS_COMPACT]; const uint32_t h = (uint32_t)(k >> 6) & 1u, bit = (uint32_t)k & 63u;
        uint64_t m = ~0ull; for (int b = 0; b < 5; b++) m &= ((c >> b) & 1u) ? R[5 * h + b] : ~R[5 * h + b];
        const uint64_t below = (1ull << bit) - 1ull;
        const uint64_t mid = H.letters[(size_t)(k >> KJ_CSB_SHIFT) * KJ_CSB_STRIDE + c] + ((const uint16_t*)(R + KJ_CPT_COUNT_WORD))[c];
        const uint64_t v = h ? mid + (uint64_t)__builtin_popcountll(m & below) : mid - (uint64_t)__builtin_popcountll(m & ~below);
        return k >= H.quirk_lo ? v - H.quirk_d[c] : v;
    }
    const uint32_t RB = kj_rank_rows(H.wide), RW = kj_rank_words(H.wide);
    uint64_t b = k / RB; uint32_t r = (uint32_t)(k - b * RB); const uint64_t* B = &H.rank[((size_t)c * H.nb + b) * RW];
    uint32_t wi = r >> 6, bit = r & 63u; uint64_t ww = B[1 + wi];
    uint64_t add = (H.wide && wi) ? ((B[0] >> (32 + 8 * wi)) & 0xff) : 0;
    const uint64_t v = (H.wide ? (B[0] & KJ_CNT_MASK) : B[0]) + add + (uint64_t)__builtin_popcountll(ww & ((1ull << bit) - 1ull));
    return k >= H.quirk_lo ? v - H.quirk_d[c] : v;                  // the reference's checkpoint quirk (kj_build_host_index)
}
uint64_t kj_host_rank(const KjHostIndex& H, uint32_t c, uint64_t k) { return host_rank(H, c, k); }
// index = a0*20^(k-1) + a1*20^(k-2) + ... + a(k-1), a_t = letter consumed t-th by the backward search (end of the k-mer first), letters 1..20 -> 0..19
void kj_build_kmer_table(KjHostIndex& H, int k) {
    H.kmer.clear(); H.kmer32.clear(); H.kmer_k = 0;
    if (k < 2 || k > 6 || H.alen != 21) return;
    std::vector<KjKmer> cur(20), nxt;
    for (uint32_t a = 0; a < 20; a++) { cur[a].lo = H.C[a + 1]; cur[a].hi = H.C[a + 2]; }
    unsigned nthr = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    for (int d = 1; d < k; d++) {
        nxt.assign(cur.size() * 20, KjKmer{0, 0});
        std::vector<std::thread> th; const size_t n = cur.size();
        for (unsigned t = 0; t < nthr; t++) th.emplace_back([&, t] {
            for (size_t i = t; i < n; i += nthr) {
                const KjKmer iv = cur[i];
                for (uint32_t a = 0; a < 20; a++) {
                    KjKmer o{0, 0};
                    if (iv.lo < iv.hi) { o.lo = host_rank(H, a + 1, iv.lo); o.hi = host_rank(H, a + 1, iv.hi); if (o.lo >= o.hi) { o.lo = 0; o.hi = 0; } }
                    nxt[i * 20 + a] = o;
                }
            }
        });
        for (auto& x : th) x.join();
        cur.swap(nxt);
    }
    if (H.wide) H.kmer.swap(cur); else { H.kmer32.resize(cur.size()); for (size_t i = 0; i < cur.size(); i++) { H.kmer32[i].lo = (uint32_t)cur[i].lo; H.kmer32[i].hi = (uint32_t)cur[i].hi; } }
    H.kmer_k = k;
}

// E-value gate (ConsumerThread.cpp:500-513): Evalue = db_length * query_len * 2^-bitscore(best) must not exceed min_Evalue.
// For a fixed score k the left-hand side is a monotone function of query_len in IEEE arithmetic (two multiplications by
// positive constants), so "score k passes" <=> query_len <= breaks[k], where breaks[k] is found by bisection over the
// bit patterns of the positive doubles with the reference's own expression.  The device computes query_len with the same
// IEEE divisions/additions as the reference and counts the breaks below it: an exact integer threshold, any read length.
int kj_build_evalue_breaks(const kj_params& p, double db_length, std::vector<double>& breaks) {
    breaks.clear();
    if (!(p.mode == 1 && p.use_evalue)) return KJ_OK;
    auto passes = [&](double query_len, unsigned best) {
        double bitscore = (0.3176 * best - (-2.009915479)) / 0.6931471805;                  // LAMBDA, LN_K, LN_2 (ConsumerThread.hpp:41-44)
        double Evalue = db_length * query_len * pow(2, -1 * bitscore);
        return !(Evalue > p.min_evalue);
    };
    double prev = 0.0;
    for (unsigned k = 0; k < 65536; k++) {
        uint64_t lo = 0, hi; const double top = 1e300; memcpy(&hi, &top, 8);                // passes(0) holds, passes(1e300) cannot
        if (passes(top, k)) { breaks.push_back(top); break; }
        while (hi - lo > 1) { uint64_t mid = lo + (hi - lo) / 2; double q; memcpy(&q, &mid, 8); if (passes(q, k)) lo = mid; else hi = mid; }
        double q; memcpy(&q, &lo, 8);
        if (q < prev) { kj_err() = "E-value threshold is not monotone in the score"; return KJ_ERR_UNSUPPORTED; }
        breaks.push_back(q); prev = q;
        if (q > 1e12) break;                                                                 // longer queries than any supported read
    }
    return KJ_OK;
}

void kj_fill_run_params(const kj_params& p, uint32_t max_len, KjRunParams& rp) {
    memset(&rp, 0, sizeof rp);
    rp.mode = p.mode; rp.m = p.min_fragment_length; rp.e = p.mismatches; rp.min_score = p.min_score; rp.seed_length = p.seed_length;
    rp.use_evalue = p.use_evalue; rp.seg = p.seg; rp.protein = p.input_is_protein; rp.name_mode = p.name_mode ? 1 : 0;
    if (p.input_is_protein) max_len *= 3;  // a protein read is laid out like one reading frame: residue e at array index 3e
    if (max_len < 24) max_len = 24;
    rp.max_len = (max_len + 7) / 8 * 8;
    rp.max_frag = rp.max_len / 3 + 1;
    uint32_t per_class = (rp.max_frag + 1 + rp.m) / (rp.m + 1);
    rp.item_cap = 2 * 12 * per_class + 8; rp.item_cap = (rp.item_cap + 1) & ~1u;
    rp.kept_cap_smem = KJ_KEPT_SMEM;       // 5 Greedy CTAs per SM fit with it
    rp.scratch_entries = 4 * rp.max_len + 64;
    rp.variant_cap = rp.max_len <= 160 ? 256u : rp.max_len <= 512 ? 1024u : 4096u;    // entries of the Greedy variant ring (it grows x4 and the call is repeated if a read fills it)
    if (const char* v = getenv("KJ_VARIANT_CAP")) { long x = atol(v); if (x >= 32 && x <= (1 << 20)) rp.variant_cap = (uint32_t)x; }   // test hook: provoke the overflow/retry path
}

// ------------------------------------------------------------------------------------------------
// device-native index file: "KJB200IX" | version | fixed header | raw arrays in upload order.  Little-endian, host layout of
// this build (the version changes with any layout change); replaces the load-time transcode of large indexes (mkfmi.c:63-78
// writes the reference's byte-recoded BWT + index1/index2; this file holds the one-hot rank records etc. of kj_layout.h).
// ------------------------------------------------------------------------------------------------
namespace {
const char kNativeMagic[8] = {'K', 'J', 'B', '2', '0', '0', 'I', 'X'};
const uint32_t kNativeVersion = 5;
struct NativeHeader {
    uint32_t version, sizeof_tables, sizeof_rank, alen;
    uint64_t nb, bwtlen, C[KJ_MAX_ALEN + 1], sa_check; int64_t sa_bias; int32_t sa_exp; uint32_t nseq, n_present; int32_t kmer_k, wide, pad;
    double db_length; uint64_t quirk_lo, quirk_d[KJ_MAX_ALEN];
    uint64_t n_rank, n_letters, n_sa_tax, n_seq_tax, n_tax, n_lnfact, n_kmer, n_kmer32;
    uint64_t checksum;          // over the bytes of all arrays, in file order (detects a damaged file before it reaches the GPU)
};
// order-sensitive 64-bit checksum (multiply-rotate over 8-byte words; not cryptographic)
uint64_t mix_bytes(uint64_t h, const void* p, size_t n) {
    const uint8_t* b = (const uint8_t*)p; size_t i = 0;
    for (; i + 8 <= n; i += 8) { uint64_t w; memcpy(&w, b + i, 8); h = (h ^ w) * 0x9E3779B97F4A7C15ull; h = (h << 29) | (h >> 35); }
    uint64_t w = 0; if (i < n) memcpy(&w, b + i, n - i);
    h = (h ^ w ^ (uint64_t)n) * 0x9E3779B97F4A7C15ull; return (h << 29) | (h >> 35);
}
}  // namespace
uint64_t kj_mix_bytes(uint64_t h, const void* p, size_t n) { return mix_bytes(h, p, n); }
namespace {
template <class T> uint64_t mix_vec(uint64_t h, const std::vector<T>& v) { return mix_bytes(h, v.data(), v.size() * sizeof(T)); }
uint64_t index_checksum(const KjHostIndex& H) {
    uint64_t h = 0x6b616a755f623230ull;
    h = mix_bytes(h, &H.tables, sizeof(KjTables)); h = mix_vec(h, H.rank); h = mix_vec(h, H.letters); h = mix_vec(h, H.sa_tax); h = mix_vec(h, H.seq_tax);
    h = mix_vec(h, H.tax_parent); h = mix_vec(h, H.tax_depth); h = mix_vec(h, H.tax_id); h = mix_bytes(h, H.lnfact.data(), std::min<size_t>(H.lnfact.size(), KJ_LNFACT_REF) * sizeof(double)); h = mix_vec(h, H.kmer); h = mix_vec(h, H.kmer32);
    return h;
}
template <class T> bool put(FILE* f, const std::vector<T>& v) { return v.empty() || fwrite(v.data(), sizeof(T), v.size(), f) == v.size(); }
template <class T> bool get(FILE* f, std::vector<T>& v, uint64_t n) { v.resize((size_t)n); return n == 0 || fread(v.data(), sizeof(T), (size_t)n, f) == (size_t)n; }
}  // namespace

int kj_host_index_write(const KjHostIndex& H, const char* path) {
    if (H.wide == KJ_LAYOUT_COMPACT) { kj_err() = "device-native index files hold the narrow and wide layouts only"; return KJ_ERR_UNSUPPORTED; }
    FILE* f = fopen(path, "wb"); if (!f) { kj_err() = std::string("Could not open file ") + path + " for writing"; return KJ_ERR_IO; }
    NativeHeader h; memset(&h, 0, sizeof h);
    h.version = kNativeVersion; h.sizeof_tables = (uint32_t)sizeof(KjTables); h.sizeof_rank = 8u * kj_rank_words(H.wide); h.alen = (uint32_t)H.alen;
    h.nb = H.nb; h.bwtlen = H.bwtlen; memcpy(h.C, H.C, sizeof h.C); h.sa_check = H.sa_check; h.sa_bias = H.sa_bias; h.sa_exp = H.sa_exp; h.nseq = H.nseq; h.n_present = H.n_present;
    h.kmer_k = H.kmer_k; h.wide = H.wide; h.db_length = H.db_length; h.quirk_lo = H.quirk_lo; memcpy(h.quirk_d, H.quirk_d, sizeof h.quirk_d);
    h.n_rank = H.rank.size(); h.n_letters = H.letters.size(); h.n_sa_tax = H.sa_tax.size(); h.n_seq_tax = H.seq_tax.size(); h.n_tax = H.tax_id.size(); h.n_lnfact = std::min<size_t>(H.lnfact.size(), KJ_LNFACT_REF);
    h.n_kmer = H.kmer.size(); h.n_kmer32 = H.kmer32.size(); h.checksum = index_checksum(H);
    bool ok = fwrite(kNativeMagic, 1, 8, f) == 8 && fwrite(&h, sizeof h, 1, f) == 1 && fwrite(&H.tables, sizeof(KjTables), 1, f) == 1 &&
              put(f, H.rank) && put(f, H.letters) && put(f, H.sa_tax) && put(f, H.seq_tax) && put(f, H.tax_parent) && put(f, H.tax_depth) && put(f, H.tax_id) &&
              fwrite(H.lnfact.data(), sizeof(double), h.n_lnfact, f) == h.n_lnfact && put(f, H.kmer) && put(f, H.kmer32);
    ok = (fclose(f) == 0) && ok;
    if (!ok) { kj_err() = std::string("write error on ") + path; return KJ_ERR_IO; }
    return KJ_OK;
}

int kj_host_index_read(const char* path, KjHostIndex& H) {
    FILE* f = fopen(path, "rb"); if (!f) { kj_err() = std::string("Could not open file ") + path; return KJ_ERR_IO; }
    fseeko(f, 0, SEEK_END); const uint64_t fsize = (uint64_t)ftello(f); fseeko(f, 0, SEEK_SET);
    char magic[8]; NativeHeader h;
    bool ok = fread(magic, 1, 8, f) == 8 && memcmp(magic, kNativeMagic, 8) == 0 && fread(&h, sizeof h, 1, f) == 1;
    if (!ok || h.version != kNativeVersion || h.sizeof_tables != sizeof(KjTables) || h.sizeof_rank != 8u * kj_rank_words(h.wide) || (h.wide != 0 && h.wide != 1) || h.alen < 2 || h.alen > KJ_MAX_ALEN ||
        h.n_rank != h.nb * h.alen * kj_rank_words(h.wide) || h.nb != h.bwtlen / kj_rank_rows(h.wide) + 1 || h.n_lnfact != 10001 ||
        h.n_rank > fsize / 8 || h.n_letters > fsize / 8 || h.n_sa_tax > fsize / 4 || h.n_seq_tax > fsize / 4 || h.n_tax > fsize / 16 ||
        h.n_kmer > fsize / sizeof(KjKmer) || h.n_kmer32 > fsize / sizeof(KjKmer32)) { fclose(f); kj_err() = std::string(path) + " is not a device-native index of this library version"; return KJ_ERR_IO; }
    H = KjHostIndex();
    H.alen = (int)h.alen; H.nb = h.nb; H.bwtlen = h.bwtlen; memcpy(H.C, h.C, sizeof h.C); H.sa_check = h.sa_check; H.sa_bias = h.sa_bias; H.sa_exp = h.sa_exp; H.nseq = h.nseq; H.n_present = h.n_present;
    H.kmer_k = h.kmer_k; H.wide = h.wide; H.db_length = h.db_length; H.quirk_lo = h.quirk_lo; memcpy(H.quirk_d, h.quirk_d, sizeof h.quirk_d);
    ok = fread(&H.tables, sizeof(KjTables), 1, f) == 1 && get(f, H.rank, h.n_rank) && get(f, H.letters, h.n_letters) && get(f, H.sa_tax, h.n_sa_tax) && get(f, H.seq_tax, h.n_seq_tax) &&
         get(f, H.tax_parent, h.n_tax) && get(f, H.tax_depth, h.n_tax) && get(f, H.tax_id, h.n_tax) && get(f, H.lnfact, h.n_lnfact) && get(f, H.kmer, h.n_kmer) && get(f, H.kmer32, h.n_kmer32);
    char extra; const bool at_end = fread(&extra, 1, 1, f) == 0;
    fclose(f);
    if (!ok || !at_end || h.n_present > h.n_tax || index_checksum(H) != h.checksum) { kj_err() = std::string(path) + " is truncated or corrupt"; return KJ_ERR_IO; }
    kj_lnfact_table(H.lnfact);                                          // the file holds the reference's table; Stirling's values above it
    // internal consistency (a crafted file with a recomputed checksum must not lead to out-of-bounds reads on the device)
    uint64_t nk = 1; for (int d = 0; d < H.kmer_k; d++) nk *= 20;
    bool good = H.bwtlen > 0 && H.bwtlen < (1ull << 38) && h.n_letters >= H.bwtlen / KJ_LETTERS_PER_WORD + 1 && h.n_seq_tax == H.nseq && H.sa_exp >= 0 && H.sa_exp <= 30 &&
                H.sa_check == (1ull << H.sa_exp) - 1ull && H.sa_bias == ((int64_t)((int64_t)H.nseq - 1) >> H.sa_exp) + 1 && H.kmer_k >= 0 && H.kmer_k <= 6 &&
                (H.kmer_k == 0 ? (h.n_kmer == 0 && h.n_kmer32 == 0) : (H.wide ? (h.n_kmer == nk && h.n_kmer32 == 0) : (h.n_kmer32 == nk && h.n_kmer == 0))) &&
                (H.wide || H.bwtlen < 0xffffff00ull) && H.C[0] == 0 && H.C[H.alen] == H.bwtlen &&
                (H.bwtlen >> H.sa_exp) < (uint64_t)H.sa_bias + h.n_sa_tax + 1 && (H.quirk_lo == ~0ull || (H.wide && H.quirk_lo == H.bwtlen - 128ull));
    for (int a = 0; good && a < H.alen; a++) good = H.C[a] <= H.C[a + 1];
    if (good) {
        const uint32_t nt = (uint32_t)h.n_tax; std::atomic<bool> bad(false);
        unsigned nthr = std::max(1u, std::min(16u, std::thread::hardware_concurrency())); std::vector<std::thread> th;
        for (unsigned t = 0; t < nthr; t++) th.emplace_back([&, t] {
            bool b = false;
            for (size_t i = t; i < H.sa_tax.size(); i += nthr) b |= H.sa_tax[i] >= nt && H.sa_tax[i] != KJ_TAX_BAD;
            for (size_t i = t; i < H.seq_tax.size(); i += nthr) b |= H.seq_tax[i] >= nt && H.seq_tax[i] != KJ_TAX_BAD;
            for (size_t i = t; i < H.tax_parent.size(); i += nthr) b |= H.tax_parent[i] >= nt;
            if (H.wide) { for (size_t i = t; i < H.kmer.size(); i += nthr) b |= H.kmer[i].hi > H.bwtlen || H.kmer[i].lo > H.kmer[i].hi; }
            else for (size_t i = t; i < H.kmer32.size(); i += nthr) b |= H.kmer32[i].hi > H.bwtlen || H.kmer32[i].lo > H.kmer32[i].hi;
            if (b) bad = true; });
        for (auto& x : th) x.join();
        good = !bad;
    }
    if (!good) { kj_err() = std::string(path) + " is internally inconsistent"; return KJ_ERR_IO; }
    return KJ_OK;
}

// test hook (host only): the checksums kj_debug_index_checksums() reports for a context, computed from the host transcoder's arrays
extern "C" int kj_debug_host_index_checksums(const kj_index_view* index, const kj_taxonomy_view* taxonomy, uint64_t out[8]) {
    if (!index || !taxonomy || !out) return KJ_ERR_ARG;
    KjHostIndex H; int rc = kj_build_host_index(*index, *taxonomy, H); if (rc) return rc;
    memset(out, 0, 64);
    out[0] = kj_mix_bytes(0x6b616a75ull + 0, H.rank.data(), H.rank.size() * 8);
    out[1] = kj_mix_bytes(0x6b616a75ull + 1, H.letters.data(), H.letters.size() * 8);
    out[2] = kj_mix_bytes(0x6b616a75ull + 2, H.sa_tax.data(), H.sa_tax.size() * 4);
    out[3] = kj_mix_bytes(0x6b616a75ull + 3, H.seq_tax.data(), H.seq_tax.size() * 4);
    out[4] = H.wide ? kj_mix_bytes(0x6b616a75ull + 4, H.kmer.data(), H.kmer.size() * sizeof(KjKmer)) : kj_mix_bytes(0x6b616a75ull + 4, H.kmer32.data(), H.kmer32.size() * sizeof(KjKmer32));
    out[5] = H.bwtlen; out[6] = (uint64_t)H.wide; out[7] = H.sa_tax.size();
    return KJ_OK;
}
