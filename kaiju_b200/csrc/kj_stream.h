// kj_stream.h -- the host side of the file pipeline's reader (KjFileReader, kj_ingest.h) that needs no device: how the format of an input is
// told from its first bytes, how a round of BGZF blocks is planned, and input that cannot seek (a FIFO, a pipe, /dev/stdin or /dev/fd/N, a
// character device), which is read once, front to back:
//   KjStream       fills a buffer from the descriptor.  Bytes taken from the stream but not used yet (the format probe; what a BGZF round left
//                  over when the rest goes to zlib) are put back in front of it, so no byte is read twice.  Every wait is a poll() that halt()
//                  ends: a call that fails never waits for a stalled writer.
//   kj_bgzf_top_up the BGZF carry: what the last round did not consume (blocks whose text did not fit the ring slot, a block cut by the round's
//                  end) goes to the front of the next round's buffer, and the stream fills the rest.
//   KjGzStream     other gzip through a z_stream, read as gzread reads a file.
// No CUDA here: the CPU tests drive all of it over a real pipe (tests/emu/kj_emu_stream.cpp, the BGZF blocks on the inflate emulator).
#pragma once
#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <sys/eventfd.h>
#include <unistd.h>
#include <zlib.h>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>
#include "kj_inflate.h"

enum { KJ_INPUT_PLAIN = 0, KJ_INPUT_BGZF = 1, KJ_INPUT_GZIP = 2 };
// The format of an input from its first bytes (up to 64 KiB): BGZF is what the first member says it is, a gzip header with the "BC" subfield
// (its whole block lies within the first 64 KiB); other gzip goes to zlib; everything else is read as it is.
static inline int kj_input_format(const uint8_t* head, size_t got) {
    std::vector<KjBgzfBlock> table; const int st = got > 0 ? kj_bgzf_walk(head, got, 0, 1, 0, 0, table).stop : KJ_BGZF_GARBAGE;
    if (!table.empty() || st == KJ_BGZF_PARTIAL) return KJ_INPUT_BGZF;
    return got >= 2 && head[0] == 0x1f && head[1] == 0x8b ? KJ_INPUT_GZIP : KJ_INPUT_PLAIN;
}

// One round of BGZF blocks: buf[0, got) are the compressed bytes at input offset `off`, ceof = the input ends behind them.  The whole blocks
// whose text fits text_cap (at most max_blocks) go to `table`; eof: this round holds the last text; to_zlib: a gzip member that is no BGZF block
// starts at w.consumed; error: a bad header or a truncated block, with its offset from the start of the input.
struct KjBgzfRound { KjBgzfWalk w; bool eof = false, to_zlib = false; std::string error; };
static inline KjBgzfRound kj_bgzf_plan(const uint8_t* buf, size_t got, bool ceof, uint64_t text_cap, size_t max_blocks, uint64_t off, const std::string& path,
                                       std::vector<KjBgzfBlock>& table) {
    KjBgzfRound r; table.clear();
    r.w = kj_bgzf_walk(buf, got, text_cap, max_blocks, 0, 0, table); const KjBgzfWalk& w = r.w;
    if (w.stop == KJ_BGZF_END) r.eof = ceof;
    else if (w.stop == KJ_BGZF_GARBAGE) r.eof = true;                  // zlib, too, ignores what follows the last member
    else if (w.stop == KJ_BGZF_FOREIGN) r.to_zlib = true;
    else if (w.stop == KJ_BGZF_BAD) r.error = "corrupt BGZF header in file " + path + " at compressed offset " + std::to_string(off + w.consumed);
    else if (w.stop == KJ_BGZF_PARTIAL && (ceof || w.consumed == 0)) r.error = "truncated BGZF block in file " + path + " at compressed offset " + std::to_string(off + w.consumed);
    return r;
}
// the message for block b of a round at input offset `off` whose inflate status is st
static inline std::string kj_bgzf_block_error(const std::string& path, uint64_t off, const KjBgzfBlock& b, uint32_t st) {
    return "corrupt BGZF block in file " + path + " at compressed offset " + std::to_string(off + b.in_off - b.hdr) + ": " + kj_inflate_strerror(st);
}

enum { KJ_STREAM_ERROR = -1, KJ_STREAM_HALTED = -2 };
struct KjStream {
    int fd = -1, wake = -1;                       // the input, opened with O_NONBLOCK; an eventfd that halt() makes readable
    uint64_t pos = 0;                             // bytes handed out: the offset of the next byte from the start of the stream
    std::vector<char> back; size_t back_at = 0;   // bytes put back, handed out before the descriptor's
    bool ended = false;                           // read() returned 0
    // takes fd; false: no eventfd
    bool open(int fd_) {
        fd = fd_; pos = 0; back.clear(); back_at = 0; ended = false;
        wake = eventfd(0, EFD_CLOEXEC | EFD_NONBLOCK);
        (void)fcntl(fd, F_SETPIPE_SZ, 1 << 20);  // a pipe: 1 MiB in flight instead of 64 KiB (fewer wake-ups of writer and reader); fails harmlessly otherwise
        return wake >= 0;
    }
    void close() { if (fd >= 0) ::close(fd); if (wake >= 0) ::close(wake); fd = wake = -1; back.clear(); back_at = 0; }
    void halt() { if (wake >= 0) { const uint64_t one = 1; (void)!::write(wake, &one, sizeof one); } }      // any thread; every later wait returns HALTED
    void unread(const char* p, size_t n) { back.erase(back.begin(), back.begin() + (long)back_at); back.insert(back.begin(), p, p + n); back_at = 0; pos -= n; }
    // 1 to n bytes into b (0 only where the stream has ended): *got; 0, KJ_STREAM_ERROR or KJ_STREAM_HALTED
    int some(char* b, size_t n, size_t& got) {
        got = 0;
        if (back_at < back.size()) {
            got = std::min(n, back.size() - back_at); memcpy(b, back.data() + back_at, got); back_at += got; pos += got;
            if (back_at == back.size()) { back.clear(); back_at = 0; }
            return 0;
        }
        if (ended || n == 0) return 0;
        for (;;) {
            // poll first: a FIFO opened with O_NONBLOCK reads 0 bytes until its first writer opens it, and poll() waits for that writer
            pollfd p[2] = {{fd, POLLIN, 0}, {wake, POLLIN, 0}};
            if (::poll(p, 2, -1) < 0) { if (errno == EINTR) continue; return KJ_STREAM_ERROR; }
            if (p[1].revents) return KJ_STREAM_HALTED;
            if (!p[0].revents) continue;
            const ssize_t k = ::read(fd, b, n);
            if (k > 0) { got = (size_t)k; pos += got; return 0; }
            if (k == 0) { ended = true; return 0; }
            if (errno != EINTR && errno != EAGAIN && errno != EWOULDBLOCK) return KJ_STREAM_ERROR;
        }
    }
    // n bytes into b, fewer only where the stream ends (eof); 0, KJ_STREAM_ERROR or KJ_STREAM_HALTED
    int fill(char* b, size_t n, size_t& got, bool& eof) {
        got = 0; eof = false;
        while (got < n) { size_t k = 0; const int r = some(b + got, n - got, k); if (r) return r; if (!k) { eof = true; break; } got += k; }
        return 0;
    }
};

// The next BGZF round's compressed bytes into b[0, cap): prev[at, at + left) (what the last round did not consume), then the stream.
// *got: bytes in b; ceof: the stream ended.  0, KJ_STREAM_ERROR or KJ_STREAM_HALTED
static inline int kj_bgzf_top_up(KjStream& s, char* b, size_t cap, const char* prev, size_t at, size_t left, size_t& got, bool& ceof) {
    if (left) memcpy(b, prev + at, left);
    size_t more = 0; const int r = s.fill(b + left, cap - left, more, ceof);
    got = left + more; return r;
}

// Other gzip over a stream, read as zlib's gzread reads a file (inflateInit2 with gzip framing, so a damaged member and a wrong CRC-32 or length
// are data errors): a member that ends is followed by another when the next two bytes are the gzip magic, and anything else behind a member is
// ignored; a member cut short by the end of the stream ends the text without an error.
struct KjGzStream {
    z_stream z; bool on = false, look = false, done = false; std::vector<unsigned char> in;
    bool start() {
        memset(&z, 0, sizeof z); look = done = false; in.resize(1u << 20);
        on = inflateInit2(&z, 15 + 16) == Z_OK; return on;
    }
    void end() { if (on) inflateEnd(&z); on = false; }
    // n bytes of text into b, fewer only at its end (eof); 0, 1 (a data error), KJ_STREAM_ERROR or KJ_STREAM_HALTED
    int read(KjStream& s, char* b, size_t n, size_t& got, bool& eof) {
        got = 0; eof = false;
        while (got < n) {
            if (done) { eof = true; break; }
            if (z.avail_in == 0 || (look && z.avail_in < 2)) {        // more input, behind what is left
                if (z.avail_in) memmove(in.data(), z.next_in, z.avail_in);
                size_t k = 0; const int r = s.some((char*)in.data() + z.avail_in, in.size() - z.avail_in, k); if (r) return r;
                z.next_in = in.data(); z.avail_in += (uInt)k;
                if (!k) done = true;                                  // the end of the stream: after a member, or inside one
                continue;
            }
            if (look) { if (z.next_in[0] == 0x1f && z.next_in[1] == 0x8b) { inflateReset(&z); look = false; } else done = true; continue; }
            z.next_out = (Bytef*)b + got; z.avail_out = (uInt)std::min<size_t>(n - got, 1u << 30);
            const int r = inflate(&z, Z_NO_FLUSH);
            got = (size_t)((char*)z.next_out - b);
            if (r == Z_STREAM_END) look = true;
            else if (r != Z_OK && r != Z_BUF_ERROR) return 1;
        }
        return 0;
    }
};
