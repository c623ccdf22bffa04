// kj_inflate.h -- blocked gzip (BGZF, the container `bgzip` writes) -> text, one block per warp.
//
// A BGZF file is a series of complete gzip members of at most 64 KiB compressed and 65,536 bytes inflated; an extra subfield "BC" of each
// header holds the member's size, so the chain of blocks is walked on the host from the headers alone (kj_bgzf_walk) and every block is
// inflated independently of the others (kj_inflate_block: RFC 1951, all three block types).
//
// Inside the warp: DEFLATE symbols depend on each other bit by bit, so lane 0 alone decodes them -- through look-up tables in the warp's shared
// memory (10 bits literal/length, 8 bits distance; longer codes fall back to a canonical bit-by-bit walk) -- into a batch of up to 32 tokens
// with their output positions.  The warp then writes the batch: every lane stores one literal, and each match is copied by all lanes (a match
// may read what the same batch wrote, so matches go in order with a warp barrier between them).  The tables of a dynamic block are filled by
// all lanes from the canonical order lane 0 computed; stored blocks are a warp-wide copy.  When the block is complete its CRC-32 is taken by
// the 32 lanes over contiguous slices and combined by multiplication with x^(8 * bytes behind the slice) mod P.
//
// The input comes from outside the program: lane 0 checks every token before it enters the batch (payload end, ISIZE, distance within the
// block's own output, code validity), so the lanes that write never test anything; every loop consumes input bits or produces output bytes,
// and the outer loop carries an explicit bound besides.  A block that fails any check gets a nonzero KjInflateErr and the warp leaves it.
//
// Written in the Warp vocabulary (kj_warp.h): the same source runs on the CPU warp emulator of the tests (-DKJ_EMU).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <vector>
#include "kj_warp.h"

struct KjBgzfBlock { uint64_t in_off, out_off; uint32_t in_len, isize, crc, hdr; };     // payload in the compressed bytes, place in the text, trailer, header bytes before the payload

enum KjInflateErr {
    KJ_INF_OK = 0, KJ_INF_INPUT = 1, KJ_INF_BTYPE = 2, KJ_INF_STORED = 3, KJ_INF_LENS = 4, KJ_INF_CODE = 5, KJ_INF_DIST = 6, KJ_INF_OUTPUT = 7,
    KJ_INF_ISIZE = 8, KJ_INF_CRC = 9, KJ_INF_BOUND = 10, KJ_INF_TRAILING = 11
};
static inline const char* kj_inflate_strerror(uint32_t e) {
    static const char* const t[] = {"ok", "the deflate stream passes the end of the block", "invalid block type", "stored block length does not match its complement",
        "invalid code lengths set", "invalid literal/length or distance code", "distance reaches before the start of the block", "more data than the block's ISIZE",
        "the deflate stream ends before the block's ISIZE", "CRC-32 mismatch", "decoder step bound exceeded", "bytes left behind the deflate stream"};
    return e < sizeof t / sizeof t[0] ? t[e] : "unknown error";
}

// ------------------------------------------------------------------------------------------------
// host: the block chain
// ------------------------------------------------------------------------------------------------
enum KjBgzfStop {
    KJ_BGZF_MORE = 0,      // stopped at the budget (inflated bytes or table entries); the next block starts at `consumed`
    KJ_BGZF_END = 1,       // every byte given was consumed
    KJ_BGZF_PARTIAL = 2,   // the block at `consumed` is not complete in the bytes given
    KJ_BGZF_FOREIGN = 3,   // a gzip member that is not a BGZF block starts at `consumed`
    KJ_BGZF_GARBAGE = 4,   // no gzip member at `consumed` (zlib ignores such bytes behind the last member)
    KJ_BGZF_BAD = 5        // a BGZF header whose sizes contradict each other
};
struct KjBgzfWalk { size_t consumed = 0; uint64_t out_bytes = 0; int stop = KJ_BGZF_END; };
// Appends the whole blocks of buf[0, n) to `table` while the inflated bytes stay within out_budget (the first block is always taken) and the
// table below max_blocks.  in_base / out_base: added to the offsets the table records.
static inline KjBgzfWalk kj_bgzf_walk(const uint8_t* buf, size_t n, uint64_t out_budget, size_t max_blocks, uint64_t in_base, uint64_t out_base, std::vector<KjBgzfBlock>& table) {
    KjBgzfWalk r; size_t at = 0; const size_t first = table.size();
    for (;;) {
        r.consumed = at;
        if (at == n) { r.stop = KJ_BGZF_END; return r; }
        const uint8_t* h = buf + at; const size_t left = n - at;
        if (left < 2 || h[0] != 0x1f || h[1] != 0x8b) {
            r.stop = (left < 2 && h[0] == 0x1f) ? KJ_BGZF_PARTIAL : KJ_BGZF_GARBAGE; return r; }
        if (left < 12) { r.stop = (left >= 4 && (h[2] != 8 || h[3] != 4)) ? KJ_BGZF_FOREIGN : KJ_BGZF_PARTIAL; return r; }
        if (h[2] != 8 || h[3] != 4) { r.stop = KJ_BGZF_FOREIGN; return r; }              // BGZF: deflate, FLG = FEXTRA alone
        const size_t xlen = (size_t)h[10] | ((size_t)h[11] << 8);
        if (left < 12 + xlen) { r.stop = KJ_BGZF_PARTIAL; return r; }
        size_t bsize = 0; bool found = false;
        for (size_t x = 12; x + 4 <= 12 + xlen;) {
            const size_t slen = (size_t)h[x + 2] | ((size_t)h[x + 3] << 8);
            if (x + 4 + slen > 12 + xlen) break;
            if (h[x] == 'B' && h[x + 1] == 'C' && slen == 2) { bsize = ((size_t)h[x + 4] | ((size_t)h[x + 5] << 8)) + 1; found = true; break; }
            x += 4 + slen;
        }
        if (!found) { r.stop = KJ_BGZF_FOREIGN; return r; }
        if (bsize < 12 + xlen + 8 + 1) { r.stop = KJ_BGZF_BAD; return r; }                // header + at least one payload byte + trailer
        if (left < bsize) { r.stop = KJ_BGZF_PARTIAL; return r; }
        const uint8_t* t = h + bsize - 8;
        KjBgzfBlock b; b.in_off = in_base + at + 12 + xlen; b.in_len = (uint32_t)(bsize - 12 - xlen - 8); b.out_off = out_base + r.out_bytes; b.hdr = (uint32_t)(12 + xlen);
        b.crc = (uint32_t)t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
        b.isize = (uint32_t)t[4] | ((uint32_t)t[5] << 8) | ((uint32_t)t[6] << 16) | ((uint32_t)t[7] << 24);
        if (b.isize > 65536u) { r.stop = KJ_BGZF_BAD; return r; }
        if (table.size() > first && (r.out_bytes + b.isize > out_budget || table.size() - first >= max_blocks)) { r.stop = KJ_BGZF_MORE; return r; }
        table.push_back(b); r.out_bytes += b.isize; at += bsize;
    }
}

// ------------------------------------------------------------------------------------------------
// device (and emulator): one block per warp
// ------------------------------------------------------------------------------------------------
#define KJ_INF_LBITS 10u
#define KJ_INF_DBITS 8u
#define KJ_INF_BATCH 32u
#define KJ_INF_POLY 0xedb88320u
enum { KJ_INF_CMD_TOKENS = 0, KJ_INF_CMD_STORED = 1, KJ_INF_CMD_BUILD = 2, KJ_INF_CMD_DONE = 3, KJ_INF_CMD_ERR = 4 };

struct KjInflateWarp {      // the warp's work space (shared memory on the device)
    uint16_t llut[1u << KJ_INF_LBITS], dlut[1u << KJ_INF_DBITS];     // (symbol << 4) | code length; 0: no code of at most the table's bits
    uint16_t lsym[288], dsym[32];                                     // symbols in canonical order
    uint16_t lcnt[16], dcnt[16];                                      // codes per length
    uint8_t lens[320];                                                // code lengths: literal/length, then distance (from hlit on)
    uint32_t tok[KJ_INF_BATCH], tpos[KJ_INF_BATCH];                   // literal: bit 31 | byte; match: (length << 15) | (distance - 1); output position
    uint32_t cmd, ntok, err, hlit, copy_src, copy_len, copy_dst;
};

// bit reader of lane 0 over the block's payload; never reads outside [0, end)
struct KjInfBits {
    const uint8_t* p; uint32_t pos, end; uint64_t buf; uint32_t cnt;
    KJ_DEV void refill() { while (cnt <= 56u && pos < end) { buf |= (uint64_t)p[pos++] << cnt; cnt += 8u; } }
    KJ_DEV bool take(uint32_t n, uint32_t& v) { if (n > cnt) return false; v = (uint32_t)(buf & ((1ull << n) - 1ull)); buf >>= n; cnt -= n; return true; }
};
// canonical code from its lengths: codes per length, symbols in code order.  false: over-subscribed, or incomplete where that is not allowed
// (a single code of length 1 is; so is a distance set without any code: such a block holds literals only)
static KJ_DEV bool kj_inf_canon(const uint8_t* lens, uint32_t n, uint16_t* cnt, uint16_t* sym, bool dist) {
    uint16_t offs[16];
    for (int l = 0; l < 16; l++) cnt[l] = 0;
    for (uint32_t i = 0; i < n; i++) cnt[lens[i] & 15u]++;
    int left = 1;
    for (int l = 1; l < 16; l++) { left = (left << 1) - (int)cnt[l]; if (left < 0) return false; }
    const uint32_t used = n - cnt[0];
    if (left > 0 && !(used == 1 && cnt[1] == 1) && !(dist && used == 0)) return false;
    offs[1] = 0; for (int l = 1; l < 15; l++) offs[l + 1] = (uint16_t)(offs[l] + cnt[l]);
    for (uint32_t i = 0; i < n; i++) if (lens[i]) sym[offs[lens[i]]++] = (uint16_t)i;
    return true;
}
// one symbol; false: the bits are no code, or the payload ends inside it (err set)
static KJ_DEV bool kj_inf_symbol(KjInfBits& b, const uint16_t* lut, uint32_t bits, const uint16_t* cnt, const uint16_t* sym, uint32_t& out, uint32_t& err) {
    const uint32_t e = lut[(uint32_t)b.buf & ((1u << bits) - 1u)];
    if (e) { const uint32_t l = e & 15u; if (l > b.cnt) { err = KJ_INF_INPUT; return false; } b.buf >>= l; b.cnt -= l; out = e >> 4; return true; }
    uint32_t code = 0, first = 0, index = 0;
    for (uint32_t l = 1; l <= 15u; l++) {
        if (l > b.cnt) { err = KJ_INF_INPUT; return false; }
        code |= (uint32_t)(b.buf >> (l - 1u)) & 1u;
        const uint32_t c = cnt[l];
        if (code < first + c) { b.buf >>= l; b.cnt -= l; out = sym[index + (code - first)]; return true; }
        index += c; first = (first + c) << 1; code <<= 1;
    }
    err = KJ_INF_CODE; return false;
}
// header of a dynamic block -> lens[0, hlit + hdist), S.hlit; 0 or the error
static KJ_DEV uint32_t kj_inf_dynamic_header(KjInfBits& b, KjInflateWarp* S, uint32_t& hdist) {
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint32_t v, err = 0;
    b.refill();
    if (!b.take(14, v)) return KJ_INF_INPUT;
    const uint32_t hlit = (v & 31u) + 257u, hclen = (v >> 10) + 4u; hdist = ((v >> 5) & 31u) + 1u;
    if (hlit > 286u || hdist > 30u) return KJ_INF_LENS;
    uint8_t cl[19];
    for (int i = 0; i < 19; i++) cl[i] = 0;
    for (uint32_t i = 0; i < hclen; i++) { b.refill(); if (!b.take(3, v)) return KJ_INF_INPUT; cl[order[i]] = (uint8_t)v; }
    // the code-length code has no table: its symbols are decoded by the canonical walk (an all-zero table never matches)
    uint16_t* ccnt = S->dcnt; uint16_t* csym = S->dsym;
    if (!kj_inf_canon(cl, 19, ccnt, csym, false) || ccnt[0] == 19) return KJ_INF_LENS;
    { int left = 1; for (int l = 1; l < 16; l++) left = (left << 1) - (int)ccnt[l]; if (left != 0) return KJ_INF_LENS; }      // this one must be complete
    const uint32_t total = hlit + hdist; uint32_t i = 0;
    while (i < total) {
        uint32_t s = 0; b.refill();
        const uint16_t none = 0;
        if (!kj_inf_symbol(b, &none, 0, ccnt, csym, s, err)) return err == KJ_INF_CODE ? (uint32_t)KJ_INF_LENS : err;
        if (s < 16u) { S->lens[i++] = (uint8_t)s; continue; }
        uint32_t rep, val = 0;
        if (s == 16u) { if (i == 0) return KJ_INF_LENS; val = S->lens[i - 1]; if (!b.take(2, v)) return KJ_INF_INPUT; rep = 3u + v; }
        else if (s == 17u) { if (!b.take(3, v)) return KJ_INF_INPUT; rep = 3u + v; }
        else { if (!b.take(7, v)) return KJ_INF_INPUT; rep = 11u + v; }
        if (i + rep > total) return KJ_INF_LENS;
        while (rep--) S->lens[i++] = (uint8_t)val;
    }
    if (S->lens[256] == 0) return KJ_INF_LENS;                       // no end-of-block code
    S->hlit = hlit; return 0;
}
// all lanes: look-up table of a canonical code (cnt, sym)
static KJ_DEV void kj_inf_fill_lut(const Warp& w, uint16_t* lut, uint32_t bits, const uint16_t* cnt, const uint16_t* sym) {
    for (uint32_t k = (uint32_t)w.lane; k < (1u << bits); k += 32u) lut[k] = 0;
    w.sync();
    uint32_t total = 0; for (uint32_t l = 1; l <= bits; l++) total += cnt[l];
    uint32_t len = 1, start = 0, first = 0;
    for (uint32_t i = (uint32_t)w.lane; i < total; i += 32u) {
        while (i >= start + cnt[len]) { start += cnt[len]; first = (first + cnt[len]) << 1; len++; }
        const uint32_t s = sym[i], code = first + (i - start);
        uint32_t rev = 0; for (uint32_t k = 0; k < len; k++) rev |= ((code >> k) & 1u) << (len - 1u - k);
        for (uint32_t k = rev; k < (1u << bits); k += 1u << len) lut[k] = (uint16_t)((s << 4) | len);
    }
}
static KJ_DEV uint32_t kj_inf_mulmod(uint32_t a, uint32_t b) {       // a * b mod P, bit 31 = x^0
    uint32_t p = 0;
    for (uint32_t m = 0x80000000u; m; m >>= 1) { if (a & m) p ^= b; b = (b & 1u) ? (b >> 1) ^ KJ_INF_POLY : b >> 1; }
    return p;
}
static KJ_HD void kj_inf_crc_table_entry(uint32_t i, uint32_t* tab) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ KJ_INF_POLY : c >> 1; tab[i] = c; }

// Inflates payload in[0, in_len) into out[0, isize) and checks length and CRC-32.  Every lane returns the block's KjInflateErr.
static KJ_DEV uint32_t kj_inflate_block(const Warp& w, KjInflateWarp* S, const uint32_t* crc_tab, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t isize, uint32_t crc) {
    // lane 0's decoder state
    KjInfBits b; b.p = in; b.pos = 0; b.end = in_len; b.buf = 0; b.cnt = 0;
    uint32_t opos = 0; bool in_block = false, last_block = false, ended = false;
    uint32_t result = KJ_INF_BOUND;
    // every round consumes at least one bit or yields at least one byte
    const uint64_t max_rounds = (uint64_t)in_len * 8u + isize + 8u;
    for (uint64_t round = 0; round < max_rounds; round++) {
        if (w.lane == 0) {
            uint32_t n = 0, cmd = KJ_INF_CMD_TOKENS, err = 0, v;
            while (n < KJ_INF_BATCH && cmd == KJ_INF_CMD_TOKENS) {
                b.refill();
                if (!in_block) {
                    if (ended) {
                        if (opos != isize) { err = KJ_INF_ISIZE; break; }
                        if (b.pos - b.cnt / 8u != b.end) { err = KJ_INF_TRAILING; break; }
                        cmd = KJ_INF_CMD_DONE; break;
                    }
                    if (!b.take(3, v)) { err = KJ_INF_INPUT; break; }
                    last_block = (v & 1u) != 0; const uint32_t type = v >> 1;
                    if (type == 0) {
                        (void)b.take(b.cnt & 7u, v);                                          // to the byte boundary
                        if (!b.take(32, v)) { err = KJ_INF_INPUT; break; }
                        const uint32_t len = v & 0xffffu;
                        if (len != ((v >> 16) ^ 0xffffu)) { err = KJ_INF_STORED; break; }
                        const uint32_t src = b.pos - b.cnt / 8u;
                        if (len > b.end - src) { err = KJ_INF_INPUT; break; }
                        if (len > isize - opos) { err = KJ_INF_OUTPUT; break; }
                        S->copy_src = src; S->copy_len = len; S->copy_dst = opos; opos += len;
                        b.pos = src + len; b.buf = 0; b.cnt = 0; ended = last_block; cmd = KJ_INF_CMD_STORED;
                    } else if (type == 1) {
                        for (uint32_t i = 0; i < 288u; i++) S->lens[i] = (uint8_t)(i < 144u ? 8 : i < 256u ? 9 : i < 280u ? 7 : 8);
                        for (uint32_t i = 288u; i < 320u; i++) S->lens[i] = 5;
                        S->hlit = 288u;
                        (void)kj_inf_canon(S->lens, 288u, S->lcnt, S->lsym, false); (void)kj_inf_canon(S->lens + 288, 32u, S->dcnt, S->dsym, true);
                        in_block = true; cmd = KJ_INF_CMD_BUILD;
                    } else if (type == 2) {
                        uint32_t hdist = 0;
                        if ((err = kj_inf_dynamic_header(b, S, hdist))) break;
                        if (!kj_inf_canon(S->lens, S->hlit, S->lcnt, S->lsym, false) || !kj_inf_canon(S->lens + S->hlit, hdist, S->dcnt, S->dsym, true)) { err = KJ_INF_LENS; break; }
                        in_block = true; cmd = KJ_INF_CMD_BUILD;
                    } else { err = KJ_INF_BTYPE; break; }
                } else {
                    uint32_t s = 0;
                    if (!kj_inf_symbol(b, S->llut, KJ_INF_LBITS, S->lcnt, S->lsym, s, err)) break;
                    if (s < 256u) {
                        if (opos >= isize) { err = KJ_INF_OUTPUT; break; }
                        S->tok[n] = 0x80000000u | s; S->tpos[n] = opos; n++; opos++;
                    } else if (s == 256u) { in_block = false; ended = last_block; }
                    else {
                        const uint32_t c = s - 257u; uint32_t len, dist, d = 0;
                        if (c >= 29u) { err = KJ_INF_CODE; break; }
                        if (c < 8u) len = 3u + c; else if (c == 28u) len = 258u;
                        else { const uint32_t eb = (c >> 2) - 1u; if (!b.take(eb, v)) { err = KJ_INF_INPUT; break; } len = 3u + ((4u + (c & 3u)) << eb) + v; }
                        if (!kj_inf_symbol(b, S->dlut, KJ_INF_DBITS, S->dcnt, S->dsym, d, err)) break;
                        if (d >= 30u) { err = KJ_INF_CODE; break; }
                        if (d < 4u) dist = 1u + d;
                        else { const uint32_t eb = (d >> 1) - 1u; if (!b.take(eb, v)) { err = KJ_INF_INPUT; break; } dist = 1u + ((2u + (d & 1u)) << eb) + v; }
                        if (dist > opos) { err = KJ_INF_DIST; break; }                       // no preset dictionary: nothing before the block's own output
                        if (len > isize - opos) { err = KJ_INF_OUTPUT; break; }
                        S->tok[n] = (len << 15) | (dist - 1u); S->tpos[n] = opos; n++; opos += len;
                    }
                }
            }
            S->ntok = err ? 0u : n; S->err = err; S->cmd = err ? (uint32_t)KJ_INF_CMD_ERR : cmd;
        }
        w.sync();
        const uint32_t n = S->ntok, cmd = S->cmd;
        // the batch: literals side by side, then the matches in order (a match may read what the batch wrote before it)
        const uint32_t t = (uint32_t)w.lane < n ? S->tok[w.lane] : 0x80000000u;
        if ((uint32_t)w.lane < n && (t >> 31)) out[S->tpos[w.lane]] = (uint8_t)t;
        uint32_t mm = w.ballot(!(t >> 31));
        while (mm) {
            const int i = kj_ffs(mm) - 1; mm &= mm - 1u;
            const uint32_t ti = S->tok[i], len = ti >> 15, d = (ti & 0x7fffu) + 1u, o = S->tpos[i];
            w.sync();
            for (uint32_t k = (uint32_t)w.lane; k < len; k += 32u) out[o + k] = out[o - d + (d >= len ? k : k % d)];
        }
        if (cmd == KJ_INF_CMD_STORED) {
            const uint32_t src = S->copy_src, len = S->copy_len, dst = S->copy_dst;
            for (uint32_t k = (uint32_t)w.lane; k < len; k += 32u) out[dst + k] = in[src + k];
        } else if (cmd == KJ_INF_CMD_BUILD) {
            kj_inf_fill_lut(w, S->llut, KJ_INF_LBITS, S->lcnt, S->lsym);
            kj_inf_fill_lut(w, S->dlut, KJ_INF_DBITS, S->dcnt, S->dsym);
        }
        const uint32_t err = S->err;
        w.sync();                                                    // the batch is in memory, the work space may be rewritten
        if (cmd == KJ_INF_CMD_ERR) { result = err; break; }
        if (cmd == KJ_INF_CMD_DONE) { result = KJ_INF_OK; break; }
    }
    if (result != KJ_INF_OK) return result;
    // CRC-32 of out[0, isize): a contiguous slice per lane, each moved to its place by x^(8 * bytes behind it)
    const uint32_t per = (isize + 31u) / 32u, lo = (uint32_t)w.lane * per < isize ? (uint32_t)w.lane * per : isize, hi = lo + per < isize ? lo + per : isize;
    uint32_t c = 0xffffffffu;
    for (uint32_t p = lo; p < hi; p++) c = crc_tab[(c ^ out[p]) & 0xffu] ^ (c >> 8);
    c = ~c;
    uint32_t xn = 0x80000000u, base = 0x00800000u;                   // x^0, x^8
    for (uint32_t e = isize - hi; e; e >>= 1) { if (e & 1u) xn = kj_inf_mulmod(xn, base); base = kj_inf_mulmod(base, base); }
    c = kj_inf_mulmod(xn, c);
    for (int m = 16; m > 0; m >>= 1) c ^= w.shfl_xor(c, m);
    return c == crc ? (uint32_t)KJ_INF_OK : (uint32_t)KJ_INF_CRC;
}

#if !defined(KJ_EMU)
#define KJ_INF_WARPS 4
// One warp per table entry: comp + in_off -> text + out_off; status[i] = KjInflateErr of block i.
__global__ void __launch_bounds__(KJ_INF_WARPS * 32) kj_inflate_kernel(const uint8_t* __restrict__ comp, const KjBgzfBlock* __restrict__ table, uint32_t nblocks, uint8_t* text, uint32_t* __restrict__ status) {
    __shared__ KjInflateWarp ws[KJ_INF_WARPS]; __shared__ uint32_t crc_tab[256];
    for (uint32_t i = threadIdx.x; i < 256u; i += blockDim.x) kj_inf_crc_table_entry(i, crc_tab);
    __syncthreads();
    const uint32_t blk = blockIdx.x * KJ_INF_WARPS + (threadIdx.x >> 5);
    if (blk >= nblocks) return;
    Warp w; w.lane = (int)(threadIdx.x & 31u);
    const KjBgzfBlock b = table[blk];
    const uint32_t e = kj_inflate_block(w, &ws[threadIdx.x >> 5], crc_tab, comp + b.in_off, b.in_len, text + b.out_off, b.isize, b.crc);
    if (w.lane == 0) status[blk] = e;
}
#endif
