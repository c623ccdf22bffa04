// kj_emu.cpp -- TEST INFRASTRUCTURE ONLY: runs the product's kernel source (kaiju_b200/csrc/kj_core.h,
// compiled with -DKJ_EMU) on a CPU by emulating one warp with 32 cooperatively scheduled fibers, so the
// exact device logic can be checked against the oracle on a machine without a GPU.  The product library
// (libkaijub200.so) never contains this file and has no CPU execution path.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>
#include <atomic>
#include <algorithm>
#define KJ_EMU 1
#include "../../kaiju_b200/csrc/kj_warp.h"

namespace kjemu {
extern "C" void kjemu_ctx_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl kjemu_ctx_switch
.type kjemu_ctx_switch,@function
kjemu_ctx_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
)");

struct Sched {
    static const int NL = 32;
    void* sp[NL]; char* stack[NL]; bool done[NL]; void* main_sp;
    int cur; uint64_t slots[2][NL]; int arrived[2]; long gen[NL]; long complete; long progress; int ndone;
    void (*body)(Sched*, int, void*); void* arg;
    size_t stack_size;
    Sched() : stack_size(256 * 1024) { for (int i = 0; i < NL; i++) stack[i] = (char*)aligned_alloc(64, stack_size); }
    ~Sched() { for (int i = 0; i < NL; i++) free(stack[i]); }
    void yield_from(int lane) {
        long p0 = progress; int spins = 0;
        for (;;) {
            int nx = lane;
            for (int t = 1; t <= NL; t++) { int c = (lane + t) % NL; if (!done[c]) { nx = c; break; } }
            if (nx == lane) {   // nobody else runnable
                fprintf(stderr, "kjemu: deadlock -- lane %d waits in a collective while all other lanes have exited\n", lane); abort();
            }
            int me = lane; cur = nx; kjemu_ctx_switch(&sp[me], sp[nx]);
            // resumed
            if (progress != p0) return;
            if (++spins > 4 * NL) { fprintf(stderr, "kjemu: deadlock -- lanes diverged around a warp collective (lane %d)\n", lane); abort(); }
            return;   // let the caller re-check its condition
        }
    }
};
static thread_local Sched* tls_sched = nullptr;

static void fiber_entry() {
    Sched* s = tls_sched; int lane = s->cur;
    s->body(s, lane, s->arg);
    s->done[lane] = true; s->ndone++; s->progress++;
    if (s->ndone == Sched::NL) { void* dummy; kjemu_ctx_switch(&dummy, s->main_sp); }
    for (;;) {
        int nx = -1; for (int t = 1; t <= Sched::NL; t++) { int c = (lane + t) % Sched::NL; if (!s->done[c]) { nx = c; break; } }
        if (nx < 0) { void* dummy; kjemu_ctx_switch(&dummy, s->main_sp); }
        s->cur = nx; void* dummy; kjemu_ctx_switch(&dummy, s->sp[nx]);
    }
}

static void run_warp(Sched* s, void (*body)(Sched*, int, void*), void* arg) {
    tls_sched = s; s->body = body; s->arg = arg; s->arrived[0] = s->arrived[1] = 0; s->complete = -1; s->progress = 0; s->ndone = 0;
    for (int i = 0; i < Sched::NL; i++) {
        s->done[i] = false; s->gen[i] = 0;
        uintptr_t top = ((uintptr_t)(s->stack[i] + s->stack_size)) & ~(uintptr_t)63;
        void** p = (void**)(top - 64);
        // layout popped by kjemu_ctx_switch: r15 r14 r13 r12 rbx rbp, then ret -> fiber_entry (rsp must be 8 mod 16 at entry)
        p[-1] = nullptr;                 // fake return address of fiber_entry (never used)
        p[-2] = (void*)&fiber_entry;     // address at 16-aligned slot -> after ret rsp = &p[-1] which is 8 mod 16
        for (int k = 3; k <= 8; k++) p[-k] = nullptr;
        s->sp[i] = (void*)&p[-8];
    }
    s->cur = 0; kjemu_ctx_switch(&s->main_sp, s->sp[0]);
}

uint64_t rendezvous(Sched* s, int lane, uint64_t v, int kind, int arg) {
    long g = s->gen[lane]++; int par = (int)(g & 1);
    s->slots[par][lane] = v;
    if (++s->arrived[par] == Sched::NL) { s->arrived[par] = 0; s->complete = g; s->progress++; }
    int spins = 0;
    while (s->complete < g) { s->yield_from(lane); if (++spins > 100000) { fprintf(stderr, "kjemu: stuck collective\n"); abort(); } }
    int src = kind == 0 ? (arg & 31) : ((lane ^ arg) & 31);
    return s->slots[par][src];
}
uint32_t rendezvous_ballot(Sched* s, int lane, bool p) {
    long g = s->gen[lane]++; int par = (int)(g & 1);
    s->slots[par][lane] = p ? 1 : 0;
    if (++s->arrived[par] == Sched::NL) { s->arrived[par] = 0; s->complete = g; s->progress++; }
    int spins = 0;
    while (s->complete < g) { s->yield_from(lane); if (++spins > 100000) { fprintf(stderr, "kjemu: stuck collective\n"); abort(); } }
    uint32_t m = 0; for (int i = 0; i < Sched::NL; i++) if (s->slots[par][i]) m |= 1u << i;
    return m;
}
}  // namespace kjemu

struct KjEmuStats;
#include "../../kaiju_b200/csrc/kj_core.h"
thread_local KjEmuStats kj_emu_stats;
static KjEmuStats g_emu_total; static std::atomic<int> g_emu_lock(0);
#include "../../kaiju_b200/csrc/kj_core_greedy.h"
#include "../../kaiju_b200/csrc/kj_host.h"

struct EmuCtx {
    KjHostIndex H; KjDevIndex D; kj_params P; std::vector<double> evbreaks;
};
struct ItemArg { uint8_t* rec; char* text; uint32_t text_cap, text_len; bool want_acc; uint32_t nacc; uint32_t accs[24]; uint32_t nids; uint32_t ids[24]; EmuCtx* c; KjRunParams* rp; uint8_t* smem; KjKept* spill; void* gscratch; uint32_t* err; const uint8_t* s1; int n1; const uint8_t* s2; int n2; bool paired; uint32_t tax[32]; uint32_t best[32]; };

static void item_body(kjemu::Sched* s, int lane, void* a) {
    ItemArg* A = (ItemArg*)a;
    KjWarpCtx cx; cx.w.lane = lane; cx.w.s = s; cx.ix = &A->c->D; cx.rp = A->rp; cx.tb = &A->c->H.tables; cx.smem = A->smem;
    cx.L = kj_smem_layout(*A->rp); cx.spill = A->spill; cx.gscratch = A->gscratch; cx.err = A->err;
    cx.text = A->text; cx.text_cap = A->text_cap; cx.text_len = 0; cx.want_acc = A->want_acc;
    uint32_t best = 0;
    const bool wide = A->c->D.wide != 0;
    uint32_t t;
    if (A->rp->mode == 1 && A->rec) {
        // the two-kernel Greedy path: front end -> record -> (work space wiped) -> search
        if (wide) (void)kj_classify_item<1, uint64_t, 1>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best, A->rec); else (void)kj_classify_item<1, uint32_t, 1>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best, A->rec);
        cx.w.sync();
        for (uint32_t i = (uint32_t)lane; i < cx.L.total; i += 32) cx.smem[i] = 0xA5;
        cx.w.sync();
        t = wide ? kj_classify_item<1, uint64_t, 2>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best, A->rec) : kj_classify_item<1, uint32_t, 2>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best, A->rec);
    } else
    t = A->rp->mode == 0 ? (wide ? kj_classify_item<0, uint64_t>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best) : kj_classify_item<0, uint32_t>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best))
        : wide ? kj_classify_item<1, uint64_t>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best) : kj_classify_item<1, uint32_t>(cx, A->s1, A->n1, A->s2, A->n2, A->paired, best);
    A->tax[lane] = t; A->best[lane] = best;
    if (lane == 0) { A->nids = cx.nids; const uint32_t* ids = (const uint32_t*)(cx.smem + cx.L.ids_off); for (uint32_t u = 0; u < cx.nids && u < 24; u++) A->ids[u] = ids[u];
                     A->text_len = cx.text_len; const uint32_t* accs = (const uint32_t*)(cx.smem + cx.L.accs_off); A->nacc = (A->want_acc && t != KJ_TAX_BAD) ? accs[20] : 0; for (uint32_t u = 0; u < A->nacc && u < 20; u++) A->accs[u] = accs[u]; }
}

extern "C" {
void* kjemu_create(const char* fmi_path, const char* nodes_path, const kj_params* p) {
    kj_fmi* f = nullptr; kj_nodes* t = nullptr;
    if (kj_fmi_load(fmi_path, &f) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); return nullptr; }
    kj_index_view iv; kj_taxonomy_view tv; kj_fmi_view(f, &iv);
    std::vector<uint64_t> st, node, parent;
    if (nodes_path && *nodes_path) {
        if (kj_nodes_load(nodes_path, &t) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); return nullptr; }
        kj_nodes_view(t, &tv);
    } else {   // the name front-ends' view (kj_cli.cpp run_name_frontend): sequences numbered 2.. under the root 1
        st.resize((size_t)iv.nseq); node.resize((size_t)iv.nseq + 1); parent.assign((size_t)iv.nseq + 1, 1); node[0] = 1;
        for (int32_t i = 0; i < iv.nseq; i++) { st[(size_t)i] = (uint64_t)i + 2; node[(size_t)i + 1] = (uint64_t)i + 2; }
        iv.seq_taxon = st.data(); tv.n = node.size(); tv.node = node.data(); tv.parent = parent.data();
    }
    EmuCtx* c = new EmuCtx(); c->P = *p;
    if (kj_check_params(*p) != KJ_OK || kj_build_host_index(iv, tv, c->H) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); delete c; return nullptr; }
    kj_fmi_free(f); if (t) kj_nodes_free(t);
    if (kj_build_evalue_breaks(*p, c->H.db_length, c->evbreaks) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); delete c; return nullptr; }
    KjDevIndex& D = c->D; KjHostIndex& H = c->H; memset(&D, 0, sizeof D);
    // the guard entry the device appends (create_ctx): the last sampled row of a reference-built index may have no suffix-array entry
    const size_t n_sa = H.sa_tax.size(); H.sa_tax.push_back(KJ_TAX_BAD); if (!H.sa_acc.empty()) H.sa_acc.push_back(0xffffffffu);
    D.rank = H.rank.data(); D.nb = H.nb; D.letters = H.letters.data(); D.bwtlen = H.bwtlen; D.alen = H.alen;
    for (int a = 0; a <= H.alen; a++) D.C[a] = H.C[a];
    for (int a = 0; a < H.alen; a++) D.rank_base[a] = D.rank + (uint64_t)a * H.nb * kj_rank_words(H.wide);
    D.sa_tax = H.sa_tax.data(); D.seq_tax = H.seq_tax.data(); D.sa_acc = H.sa_acc.empty() ? nullptr : H.sa_acc.data(); D.seq_acc = H.seq_acc.empty() ? nullptr : H.seq_acc.data(); D.sa_check = H.sa_check; D.sa_exp = H.sa_exp; D.sa_bias = H.sa_bias;
    D.n_sa = n_sa; D.nseq = H.nseq;
    D.tax_parent = H.tax_parent.data(); D.tax_depth = H.tax_depth.data(); D.tax_id = H.tax_id.data(); D.n_tax = (uint32_t)H.tax_id.size();
    D.lnfact = H.lnfact.data(); D.n_lnfact = (int)H.lnfact.size(); D.kmer = H.kmer_k ? (H.wide ? (const void*)H.kmer.data() : (const void*)H.kmer32.data()) : nullptr; D.kmer_k = H.kmer_k; D.wide = H.wide; D.tables = &H.tables; D.quirk_lo = H.quirk_lo; D.quirk_d = H.quirk_d; D.mono = (H.quirk_lo == ~0ull && !getenv("KJ_EMU_NOMONO")) ? 1 : 0;
    return c;
}
void kjemu_destroy(void* h) { delete (EmuCtx*)h; }

// device-native index file: write the transcoded index of (fmi, nodes), read it back, compare every field.  0 = identical.
int kjemu_native_roundtrip(const char* fmi_path, const char* nodes_path, const char* out_path) {
    kj_fmi* f = nullptr; kj_nodes* t = nullptr;
    if (kj_fmi_load(fmi_path, &f) != KJ_OK || kj_nodes_load(nodes_path, &t) != KJ_OK) return -1;
    kj_index_view iv; kj_taxonomy_view tv; kj_fmi_view(f, &iv); kj_nodes_view(t, &tv);
    KjHostIndex A, B; int rc = kj_build_host_index(iv, tv, A); kj_fmi_free(f); kj_nodes_free(t);
    if (rc || kj_host_index_write(A, out_path) != KJ_OK || kj_host_index_read(out_path, B) != KJ_OK) { fprintf(stderr, "kjemu: %s\n", kj_last_error()); return -2; }
    auto same = [](const auto& x, const auto& y) { return x.size() == y.size() && (x.empty() || memcmp(x.data(), y.data(), x.size() * sizeof(x[0])) == 0); };
    bool ok = same(A.rank, B.rank) && same(A.letters, B.letters) && same(A.sa_tax, B.sa_tax) && same(A.seq_tax, B.seq_tax) && same(A.tax_parent, B.tax_parent) &&
              same(A.tax_depth, B.tax_depth) && same(A.tax_id, B.tax_id) && same(A.lnfact, B.lnfact) && same(A.kmer, B.kmer) && same(A.kmer32, B.kmer32) &&
              A.nb == B.nb && A.bwtlen == B.bwtlen && A.alen == B.alen && memcmp(A.C, B.C, sizeof A.C) == 0 && A.sa_check == B.sa_check && A.sa_exp == B.sa_exp &&
              A.sa_bias == B.sa_bias && A.nseq == B.nseq && A.n_present == B.n_present && A.kmer_k == B.kmer_k && A.wide == B.wide && A.db_length == B.db_length && A.quirk_lo == B.quirk_lo && memcmp(A.quirk_d, B.quirk_d, sizeof A.quirk_d) == 0 &&
              memcmp(&A.tables, &B.tables, sizeof(KjTables)) == 0;
    return ok ? 0 : 1;
}
// E-value gate: the break points (largest passing query length per score) the device counts against
int kjemu_evalue_breaks(double min_evalue, double db_length, double* out, int cap) {
    kj_params p; memset(&p, 0, sizeof p); p.mode = 1; p.use_evalue = 1; p.min_evalue = min_evalue; p.min_fragment_length = 11; p.min_score = 65; p.seed_length = 7;
    std::vector<double> b; if (kj_build_evalue_breaks(p, db_length, b) != KJ_OK) return -1;
    for (size_t i = 0; i < b.size() && (int)i < cap; i++) out[i] = b[i];
    return (int)b.size();
}
// developer counters of the chain-resolution loops (rounds, warp-steps, lane-steps, chains completed, blocks, look-aheads, pops ...)
int kjemu_stats(unsigned long long* out, int cap, int reset) {
    const unsigned long long* a = (const unsigned long long*)&g_emu_total; int n = (int)(sizeof(KjEmuStats) / 8);
    for (int k = 0; k < n && k < cap; k++) out[k] = a[k];
    if (reset) memset(&g_emu_total, 0, sizeof g_emu_total);
    return n;
}
int kjemu_native_read(const char* path) { KjHostIndex H; return kj_host_index_read(path, H); }

int kjemu_classify_v2(void* h, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n, uint64_t* taxon_out, uint32_t* best_out,
                      uint64_t* ids_out, uint8_t* nids_out, uint32_t* acc_out, uint8_t* nacc_out, char* frag_out, uint32_t frag_stride, uint32_t* frag_len_out, int nthreads);
int kjemu_classify_ids(void* h, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                       uint64_t* taxon_out, uint32_t* best_out, uint64_t* ids_out, uint8_t* nids_out, int nthreads) {
    return kjemu_classify_v2(h, seq1, off1, seq2, off2, n, taxon_out, best_out, ids_out, nids_out, nullptr, nullptr, nullptr, 0, nullptr, nthreads); }
int kjemu_classify(void* h, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                   uint64_t* taxon_out, uint32_t* best_out, int nthreads) { return kjemu_classify_ids(h, seq1, off1, seq2, off2, n, taxon_out, best_out, nullptr, nullptr, nthreads); }
// ids_out[i*21 .. +nids_out[i]): the match-id set of read i, ascending (what kj_classify_verbose delivers)
// all verbose outputs of kj_classify_verbose2 (accession ranks ascending, fragment strings)
int kjemu_classify_v2(void* h, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n, uint64_t* taxon_out, uint32_t* best_out,
                      uint64_t* ids_out, uint8_t* nids_out, uint32_t* acc_out, uint8_t* nacc_out, char* frag_out, uint32_t frag_stride, uint32_t* frag_len_out, int nthreads) {
    EmuCtx* c = (EmuCtx*)h; bool paired = seq2 != nullptr;
    uint32_t max1 = 0, max2 = 0;
    for (uint64_t i = 0; i < n; i++) { max1 = std::max<uint32_t>(max1, (uint32_t)(off1[i + 1] - off1[i])); if (paired) max2 = std::max<uint32_t>(max2, (uint32_t)(off2[i + 1] - off2[i])); }
    if (c->P.input_is_protein ? (paired || max1 > KJ_MAX_PROTEIN_LEN) : (max1 > KJ_MAX_READ_LEN || max2 > KJ_MAX_READ_LEN)) return KJ_ERR_UNSUPPORTED;
    KjRunParams rp; kj_fill_run_params(c->P, std::max(max1, max2), rp);
    rp.ev_breaks = c->evbreaks.data(); rp.n_ev_breaks = (uint32_t)c->evbreaks.size();
    rp.ws_global = 1;          // host memory either way; the device-only pointer switch is covered by the GPU tests
    KjSmemLayout L = kj_smem_layout(rp);
    std::atomic<uint64_t> next(0); std::atomic<uint32_t> errs(0);
    if (nthreads < 1) nthreads = 1;
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) th.emplace_back([&] {
        kjemu::Sched* s = new kjemu::Sched();
        std::vector<uint8_t> smem(L.total + 64); std::vector<KjKept> spill(rp.scratch_entries);
        std::vector<uint8_t> gscratch(kj_greedy_scratch_bytes(rp)); uint32_t err = 0;
        const bool split = getenv("KJ_EMU_SPLIT") != nullptr && rp.mode == 1;      // Greedy through the front-end / search pair of the two-kernel path
        std::vector<uint8_t> rec(kj_prep_stride(rp) + 64, 0xA5);
        for (;;) {
            uint64_t i = next.fetch_add(1); if (i >= n) break;
            ItemArg A; A.rec = split ? rec.data() : nullptr; A.c = c; A.rp = &rp; A.smem = smem.data(); A.spill = spill.data(); A.gscratch = gscratch.data(); A.err = &err;
            A.s1 = (const uint8_t*)seq1 + off1[i]; A.n1 = (int)(off1[i + 1] - off1[i]);
            A.s2 = paired ? (const uint8_t*)seq2 + off2[i] : nullptr; A.n2 = paired ? (int)(off2[i + 1] - off2[i]) : 0; A.paired = paired;
            A.text = frag_out ? frag_out + i * (size_t)frag_stride : nullptr; A.text_cap = frag_stride; A.text_len = 0; A.want_acc = acc_out != nullptr && c->D.sa_acc != nullptr; A.nacc = 0;
            memset(smem.data(), 0xA5, smem.size());      // poison: the kernel must not rely on zeroed shared memory
            kjemu::run_warp(s, item_body, &A);
            // the red zones between the work-space arrays must be untouched (a stray store would silently corrupt a neighbour on the GPU)
            for (uint32_t g = 0; g < L.nguard; g++) for (uint32_t b = 0; b < 64; b++) if (smem[L.guard[g] + b] != 0xA5) {
                fprintf(stderr, "kjemu: work-space red zone %u (offset %u) overwritten at read %llu\n", g, L.guard[g], (unsigned long long)i); abort(); }
            for (size_t b = L.total; b < smem.size(); b++) if (smem[b] != 0xA5) { fprintf(stderr, "kjemu: store past the work space at read %llu\n", (unsigned long long)i); abort(); }
            for (size_t b = kj_prep_stride(rp); b < rec.size(); b++) if (rec[b] != 0xA5) { fprintf(stderr, "kjemu: store past the prepared-item record at read %llu\n", (unsigned long long)i); abort(); }
            for (int l = 1; l < 32; l++) if (A.tax[l] != A.tax[0] || A.best[l] != A.best[0]) { fprintf(stderr, "kjemu: non-uniform result at read %llu\n", (unsigned long long)i); abort(); }
            taxon_out[i] = A.tax[0] == KJ_TAX_BAD ? 0 : c->H.tax_id[A.tax[0]];
            if (best_out) best_out[i] = taxon_out[i] ? A.best[0] : 0;
            if (acc_out) { std::vector<uint32_t> v(A.accs, A.accs + std::min<uint32_t>(A.nacc, 20)); std::sort(v.begin(), v.end()); for (size_t u = 0; u < v.size(); u++) acc_out[i * 20 + u] = v[u]; nacc_out[i] = (uint8_t)v.size(); }
            if (frag_len_out) frag_len_out[i] = taxon_out[i] ? A.text_len : 0;
            if (ids_out) { std::vector<uint64_t> v; if (taxon_out[i]) for (uint32_t u = 0; u < A.nids && u < 24; u++) v.push_back(c->H.tax_id[A.ids[u]]); std::sort(v.begin(), v.end());
                           for (size_t u = 0; u < v.size() && u < 21; u++) ids_out[i * 21 + u] = v[u]; nids_out[i] = (uint8_t)std::min<size_t>(v.size(), 21); }
        }
        errs |= err; delete s;
        {   // fold this thread's counters into the process-wide totals
            while (g_emu_lock.exchange(1)) {}
            unsigned long long* a = (unsigned long long*)&g_emu_total; const unsigned long long* b = (const unsigned long long*)&kj_emu_stats;
            for (size_t k = 0; k < sizeof(KjEmuStats) / 8; k++) a[k] += b[k];
            memset(&kj_emu_stats, 0, sizeof kj_emu_stats); g_emu_lock.store(0);
        }
    });
    for (auto& x : th) x.join();
    return errs.load() ? KJ_ERR_OVERFLOW - 100 * (int)errs.load() : KJ_OK;
}
}
