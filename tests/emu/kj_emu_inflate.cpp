// kj_emu_inflate.cpp -- TEST INFRASTRUCTURE ONLY: the BGZF inflate code of the product (kaiju_b200/csrc/kj_inflate.h, compiled with -DKJ_EMU) on
// the CPU warp emulator (kj_emu.cpp, same translation unit).  Every block runs on heap copies of exactly its payload and its ISIZE, so that an
// address sanitiser build sees any access outside them.  Compiled by tests/emu_inflate.py.
#include "kj_emu.cpp"
#include "../../kaiju_b200/csrc/kj_inflate.h"

struct InflateArg { KjInflateWarp* S; const uint32_t* crc_tab; const uint8_t* in; uint32_t in_len; uint8_t* out; uint32_t isize, crc; uint32_t res[32]; };
static void inflate_body(kjemu::Sched* s, int lane, void* a) {
    InflateArg* A = (InflateArg*)a; Warp w; w.lane = lane; w.s = s;
    A->res[lane] = kj_inflate_block(w, A->S, A->crc_tab, A->in, A->in_len, A->out, A->isize, A->crc);
}
static uint32_t run_block(const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t isize, uint32_t crc) {
    static uint32_t crc_tab[256]; static bool have = false;
    if (!have) { for (uint32_t i = 0; i < 256; i++) kj_inf_crc_table_entry(i, crc_tab); have = true; }
    std::vector<uint8_t> ci(in, in + in_len), co(isize, 0xA5);                  // exact sizes: the sanitiser's red zones follow directly
    KjInflateWarp* S = new KjInflateWarp; memset(S, 0xA5, sizeof *S);          // the decoder must not rely on a zeroed work space
    kjemu::Sched* sc = new kjemu::Sched();
    InflateArg A; A.S = S; A.crc_tab = crc_tab; A.in = ci.data(); A.in_len = in_len; A.out = co.data(); A.isize = isize; A.crc = crc;
    kjemu::run_warp(sc, inflate_body, &A);
    delete sc; delete S;
    for (int l = 1; l < 32; l++) if (A.res[l] != A.res[0]) { fprintf(stderr, "kjemu: non-uniform inflate result\n"); abort(); }
    if (A.res[0] == KJ_INF_OK && isize) memcpy(out, co.data(), isize);
    return A.res[0];
}

extern "C" {
// one payload -> KjInflateErr
int kjemu_inflate_raw(const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t isize, uint32_t crc) { return (int)run_block(in, in_len, out, isize, crc); }
// kj_bgzf_walk on buf[0, n): table entries as 8 x uint32 words (in_off lo/hi, out_off lo/hi, in_len, isize, crc, header bytes); returns the count
int kjemu_bgzf_walk(const uint8_t* buf, uint64_t n, uint64_t out_budget, uint64_t max_blocks, KjBgzfBlock* table_out, uint64_t cap, uint64_t* consumed, uint64_t* out_bytes, int* stop) {
    std::vector<KjBgzfBlock> t; const KjBgzfWalk w = kj_bgzf_walk(buf, (size_t)n, out_budget, (size_t)max_blocks, 0, 0, t);
    for (size_t i = 0; i < t.size() && i < cap; i++) table_out[i] = t[i];
    *consumed = w.consumed; *out_bytes = w.out_bytes; *stop = w.stop; return (int)t.size();
}
// a whole BGZF file: 0, or -2 with the compressed offset of the first bad block and its KjInflateErr (header trouble: error 100 + KjBgzfStop)
int kjemu_inflate_bgzf(const uint8_t* file, uint64_t n, uint8_t* out, uint64_t out_cap, uint64_t* out_n, uint64_t* bad_offset, uint32_t* bad_err) {
    std::vector<KjBgzfBlock> t; const KjBgzfWalk w = kj_bgzf_walk(file, (size_t)n, ~0ull, ~(size_t)0, 0, 0, t);
    *out_n = 0; *bad_offset = 0; *bad_err = 0;
    if (w.stop != KJ_BGZF_END && w.stop != KJ_BGZF_GARBAGE) { *bad_offset = w.consumed; *bad_err = 100u + (uint32_t)w.stop; return -2; }
    if (w.out_bytes > out_cap) return -1;
    for (const KjBgzfBlock& b : t) {
        const uint32_t e = run_block(file + b.in_off, b.in_len, out + b.out_off, b.isize, b.crc);
        if (e) { *bad_offset = b.in_off - b.hdr; *bad_err = e; return -2; }
    }
    *out_n = w.out_bytes; return 0;
}
}
