// kj_emu_row_tax.cpp -- TEST INFRASTRUCTURE ONLY: the CPU warp emulator (kj_emu.cpp, same translation unit) plus the dense row -> taxon
// array that the library builds on the device for narrow indexes (kj_bld_row_tax), so the taxon look-up through that array can be checked
// against the SA walk and the oracle on a machine without a GPU.  Compiled by tests/emu_row_tax.py.
#include "kj_emu.cpp"
#include <map>
#include <mutex>

static std::mutex g_row_tax_mu;
static std::map<void*, std::vector<uint32_t>> g_row_tax;      // per emulator context

extern "C" {
// on = 1: the kept rows' taxa come from the row -> taxon array (built on first use, as the device builds it: every row resolved by the walk,
// narrow indexes only); on = 0: from the SA walk.  Returns whether the array is used.
int kjemu_use_row_tax(void* h, int on) {
    EmuCtx* c = (EmuCtx*)h;
    c->D.row_tax = nullptr;
    if (!on || c->H.wide) return 0;
    std::lock_guard<std::mutex> lk(g_row_tax_mu);
    std::vector<uint32_t>& rt = g_row_tax[h];
    if (rt.empty()) {
        // the guard entry the device appends (create_ctx): the last sampled row of a reference-built index has no suffix-array entry
        c->H.sa_tax.push_back(KJ_TAX_BAD); c->D.sa_tax = c->H.sa_tax.data();
        rt.resize(c->H.bwtlen);
        for (uint64_t k = 0; k < c->H.bwtlen; k++) rt[k] = kj_row_taxon<uint32_t>(c->D, k);
    }
    c->D.row_tax = rt.data();
    return 1;
}
// kjemu_destroy plus the context's array
void kjemu_destroy_row_tax(void* h) {
    { std::lock_guard<std::mutex> lk(g_row_tax_mu); g_row_tax.erase(h); }
    kjemu_destroy(h);
}
}
