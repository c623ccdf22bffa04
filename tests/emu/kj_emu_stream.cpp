// kj_emu_stream.cpp -- TEST INFRASTRUCTURE ONLY: the stream side of the file pipeline's reader (kaiju_b200/csrc/kj_stream.h) on the CPU, driven
// as KjFileReader::run drives it: the probe, then plain chunks, BGZF rounds (two round buffers, the carry moved from one to the other, the blocks
// through the inflate emulator of kj_emu_inflate.cpp) or zlib -- over whatever descriptor the test passes, a real pipe or FIFO.  Also gzread over
// a file, the path other gzip takes from a regular file.  Compiled by tests/emu_stream.py.
#include "kj_emu_inflate.cpp"
#include "../../kaiju_b200/csrc/kj_stream.h"

// the text of s: 0, 1 with *err (the message the reader would give), KJ_STREAM_HALTED.  chunks: the chunks the reader would stage
static int read_all(KjStream& s, size_t chunk, const std::string& path, std::string& text, uint64_t& inflated, uint64_t& chunks, std::string& err) {
    std::vector<char> head(65536); size_t got = 0; bool eof = false;
    int r = s.fill(head.data(), head.size(), got, eof);
    if (r) { err = "read error in file " + path; return r; }
    const int format = kj_input_format((const uint8_t*)head.data(), got);
    s.unread(head.data(), got);
    if (format == KJ_INPUT_BGZF) {
        const size_t rchunk = std::max<size_t>(chunk, 65536), max_blocks = rchunk / 1024 + 64;
        std::vector<char> buf[2] = {std::vector<char>(rchunk), std::vector<char>(rchunk)};
        std::vector<KjBgzfBlock> table; size_t at = 0, left = 0; uint64_t off = 0;
        for (int it = 0;; it++) {
            char* b = buf[it & 1].data(); bool ceof = false;
            if ((r = kj_bgzf_top_up(s, b, rchunk, buf[(it & 1) ^ 1].data(), at, left, got, ceof))) { err = "read error in file " + path; return r; }
            const KjBgzfRound plan = kj_bgzf_plan((const uint8_t*)b, got, ceof, rchunk, max_blocks, off, path, table);
            if (!plan.error.empty()) { err = plan.error; return 1; }
            const size_t base = text.size(); text.resize(base + plan.w.out_bytes); chunks++;
            for (const KjBgzfBlock& k : table) {
                const uint32_t st = run_block((const uint8_t*)b + k.in_off, k.in_len, (uint8_t*)&text[base + k.out_off], k.isize, k.crc);
                if (st) { err = kj_bgzf_block_error(path, off, k, st); return 1; }
            }
            inflated += plan.w.out_bytes; off += plan.w.consumed; at = plan.w.consumed; left = got - at;
            if (plan.eof) return 0;
            if (plan.to_zlib) { s.unread(b + at, left); break; }
        }
    }
    KjGzStream gz;
    if (format != KJ_INPUT_PLAIN && !gz.start()) { err = "inflateInit2"; return 1; }
    std::vector<char> b(chunk);
    for (;;) {
        r = gz.on ? gz.read(s, b.data(), chunk, got, eof) : s.fill(b.data(), chunk, got, eof);
        if (r) { gz.end(); err = "read error in file " + path; return r; }
        text.append(b.data(), got); chunks++;
        if (eof) break;
    }
    gz.end(); return 0;
}

extern "C" {
void* kjemu_stream_new(int fd) { KjStream* s = new KjStream(); if (!s->open(fd)) { s->close(); delete s; return nullptr; } return s; }
void kjemu_stream_halt(void* s) { ((KjStream*)s)->halt(); }
void kjemu_stream_free(void* s) { ((KjStream*)s)->close(); delete (KjStream*)s; }
// 0 (text in out[0, *out_n)), 1 (msg), -1 (out too small), KJ_STREAM_ERROR / KJ_STREAM_HALTED (msg)
int kjemu_stream_read(void* sp, uint64_t chunk, const char* path, uint8_t* out, uint64_t cap, uint64_t* out_n, uint64_t* inflated, uint64_t* chunks, char* msg, uint64_t msg_cap) {
    std::string text, err; *out_n = 0; *inflated = 0; *chunks = 0;
    const int r = read_all(*(KjStream*)sp, (size_t)chunk, path, text, *inflated, *chunks, err);
    snprintf(msg, (size_t)msg_cap, "%s", err.c_str());
    if (r) return r;
    if (text.size() > cap) return -1;
    memcpy(out, text.data(), text.size()); *out_n = text.size(); return 0;
}
// what the reader does with other gzip from a regular file: gzread until it returns 0 (the text) or -1 (returns 1: "read error")
int kjemu_gzread_file(const char* path, uint8_t* out, uint64_t cap, uint64_t* out_n) {
    gzFile fp = gzopen(path, "rb"); *out_n = 0; if (!fp) return 1;
    for (;;) {
        const int r = gzread(fp, out + *out_n, (unsigned)std::min<uint64_t>(cap - *out_n, 1u << 20));
        if (r < 0) { gzclose(fp); return 1; }
        if (r == 0) break;
        *out_n += (uint64_t)r;
        if (*out_n == cap) { gzclose(fp); return -1; }
    }
    gzclose(fp); return 0;
}
}
