// kj_ingest.h -- FASTA/FASTQ text -> packed reads -> classification -> output text, all on the device (SURVEY.md 8f-1).
//
// Replaces the reader loop of the reference's front end (src/kaiju.cpp:288-394: file-type detection by the first
// character, name = header line without its first character cut at the first of " /\t\r", FASTQ = 4-line records,
// FASTA = header + all lines up to the next '>' line, strip() of non-letters, util.cpp:25-33; kaijup.cpp:227-262 for a name-mode protein context) and
// the output formatting of ConsumerThread::doWork / ConsumerThreadx / ConsumerThreadp (every KJ_OUT_* format, kj_format.h) for whole chunks of text:
//   newline positions (count + scan + scatter) -> per-line classification (header / sequence / ignored), letters and
//   trimmed-name lengths (one warp per line) -> scans over lines -> packed sequences + offsets + names blob ->
//   [kj_name_gate] -> kj_classify_kernel (formats with fragment strings: in launches of at most KJ_FRAG_BUDGET) -> per-record output line lengths -> scan ->
//   formatted "C\tname\ttaxid..." text.
// The host only moves bytes (kj_classify_files): reader threads (one per file: page cache -> two pinned buffers -> ring of device staging buffers;
// blocked gzip (BGZF) is inflated on the way by kj_inflate_kernel, other gzip by zlib on the reader thread),
// a parser thread (staged chunks -> batches of device text -> the kernels above on a high-priority stream; the incomplete record at the end of a batch is
// carried over on the device), one classifying thread per context (two classification lanes: launch batch k+1 while batch k runs, count / format / copy
// out batch k-1; kj_classify_files_multi deals the batches to several contexts, on one device or several) and a writer thread that writes the batches
// in input order.  Record rules beyond the happy path (kaiju.cpp:288-404): file type = first character of the first non-empty line, empty lines between
// FASTQ records are skipped (phases from an automaton scan when a batch has any), last line without newline, the loop ends with file 1.
// Included by kj_device.cu (one translation unit: it uses kj_ctx and launch()).
#pragma once
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <set>
#include "kj_inflate.h"
#include "kj_stream.h"
#include "kj_format.h"

// ------------------------------------------------------------------------------------------------
// device-wide exclusive scan of uint32 (in place); total -> *total.  Tile = 256 threads x 8 elements.
// ------------------------------------------------------------------------------------------------
#define KJ_SCAN_TILE 2048u
static __device__ __forceinline__ uint32_t kj_block_excl_scan(uint32_t v, uint32_t* smem_warp, uint32_t& block_total) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += o; }
    if (lane == 31) smem_warp[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < (blockDim.x >> 5) ? smem_warp[lane] : 0u, y = w;
        for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, y, d); if (lane >= (uint32_t)d) y += o; }
        smem_warp[32 + lane] = y - w;                       // exclusive warp bases
        if (lane == 31) smem_warp[64] = y;                  // block total
    }
    __syncthreads();
    block_total = smem_warp[64];
    const uint32_t r = smem_warp[32 + wid] + x - v;
    __syncthreads();
    return r;
}
__global__ void kj_scan_reduce(const uint32_t* __restrict__ in, uint64_t n, uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t sw[80];
    const uint64_t base = (uint64_t)blockIdx.x * KJ_SCAN_TILE + (uint64_t)threadIdx.x * 8u; uint32_t s = 0;
    for (int k = 0; k < 8; k++) if (base + k < n) s += in[base + k];
    uint32_t tot; (void)kj_block_excl_scan(s, sw, tot);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}
__global__ void kj_scan_blocks(uint32_t* __restrict__ block_sums, uint32_t nblocks, uint32_t* __restrict__ total) {   // one block of 1024 threads
    __shared__ uint32_t sw[80];
    uint32_t carry = 0;
    for (uint32_t b = 0; b < nblocks; b += blockDim.x) {
        const uint32_t i = b + threadIdx.x; const uint32_t v = i < nblocks ? block_sums[i] : 0u;
        uint32_t tot; const uint32_t e = kj_block_excl_scan(v, sw, tot);
        if (i < nblocks) block_sums[i] = carry + e;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}
__global__ void kj_scan_apply(uint32_t* __restrict__ data, uint64_t n, const uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t sw[80];
    const uint64_t base = (uint64_t)blockIdx.x * KJ_SCAN_TILE + (uint64_t)threadIdx.x * 8u;
    uint32_t v[8], s = 0;
    for (int k = 0; k < 8; k++) { v[k] = base + k < n ? data[base + k] : 0u; s += v[k]; }
    uint32_t tot; uint32_t e = kj_block_excl_scan(s, sw, tot) + block_sums[blockIdx.x];
    for (int k = 0; k < 8; k++) { if (base + k < n) data[base + k] = e; e += v[k]; }
}

// ------------------------------------------------------------------------------------------------
// text -> lines
// ------------------------------------------------------------------------------------------------
#define KJ_NL_TILE 4096u            // bytes per block: 256 threads x 16 bytes
static __device__ __forceinline__ uint32_t kj_nl_mask16(const char* __restrict__ text, uint64_t n, uint64_t p) {   // bit k set <=> text[p+k] == '\n'
    uint32_t m = 0;
    if (p + 16 <= n && ((uintptr_t)(text + p) & 15u) == 0) {
        const uint4 q = *(const uint4*)(text + p); const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        #pragma unroll
        for (int k = 0; k < 16; k++) if (((w[k >> 2] >> (8 * (k & 3))) & 0xffu) == '\n') m |= 1u << k;
    } else for (int k = 0; k < 16; k++) if (p + k < n && text[p + k] == '\n') m |= 1u << k;
    return m;
}
__global__ void kj_nl_count(const char* __restrict__ text, uint64_t n, uint32_t* __restrict__ tile_counts) {
    __shared__ uint32_t sw[80];
    const uint64_t p = (uint64_t)blockIdx.x * KJ_NL_TILE + (uint64_t)threadIdx.x * 16u;
    const uint32_t c = p < n ? (uint32_t)__popc(kj_nl_mask16(text, n, p)) : 0u;
    uint32_t tot; (void)kj_block_excl_scan(c, sw, tot);
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = tot;
}
// line_start[0] = 0, line_start[k] = position after the k-th newline
__global__ void kj_nl_scatter(const char* __restrict__ text, uint64_t n, const uint32_t* __restrict__ tile_base, uint64_t* __restrict__ line_start) {
    __shared__ uint32_t sw[80];
    const uint64_t p = (uint64_t)blockIdx.x * KJ_NL_TILE + (uint64_t)threadIdx.x * 16u;
    uint32_t m = p < n ? kj_nl_mask16(text, n, p) : 0u;
    uint32_t tot; uint32_t e = kj_block_excl_scan((uint32_t)__popc(m), sw, tot) + tile_base[blockIdx.x];
    while (m) { const int k = __ffs((int)m) - 1; m &= m - 1; line_start[++e] = p + (uint64_t)k + 1u; }
    if (blockIdx.x == 0 && threadIdx.x == 0) line_start[0] = 0;
}

// FASTQ records when blank lines occur between them (kaiju.cpp:288-289 skips empty lines while it looks for the next header, and only there):
// the phase of a line (0 = header expected, 1 = sequence, 2 = '+', 3 = qualities) is a four-state automaton over the lines; its transition
// functions compose associatively, so the phases come out of a scan.  A map is 4 x 2 bits: bits [2s+1:2s] = next phase from phase s.
#define KJ_FQ_MAP_LINE  0x39u      // 0->1 1->2 2->3 3->0
#define KJ_FQ_MAP_BLANK 0x38u      // 0->0 (skipped) 1->2 2->3 3->0
#define KJ_FQ_MAP_ID    0xE4u
static __device__ __forceinline__ uint32_t kj_fq_compose(uint32_t a, uint32_t b) {     // a first, then b
    uint32_t r = 0;
    #pragma unroll
    for (int st = 0; st < 4; st++) r |= ((b >> (2u * ((a >> (2 * st)) & 3u))) & 3u) << (2 * st);
    return r;
}
static __device__ __forceinline__ uint32_t kj_fq_line_map(const uint64_t* __restrict__ line_start, uint64_t i, uint64_t n_lines) {
    if (i >= n_lines) return KJ_FQ_MAP_ID;
    return line_start[i + 1] - 1 == line_start[i] ? KJ_FQ_MAP_BLANK : KJ_FQ_MAP_LINE;
}
// block-wide exclusive scan of maps under composition (256 threads); total = composition of the whole block
static __device__ __forceinline__ uint32_t kj_fq_block_scan(uint32_t v, uint32_t* sm, uint32_t& total) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x = kj_fq_compose(o, x); }
    if (lane == 31) sm[wid] = x;
    __syncthreads();
    if (wid == 0) {
        const uint32_t w = lane < (blockDim.x >> 5) ? sm[lane] : KJ_FQ_MAP_ID; uint32_t y = w;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, y, d); if (lane >= (uint32_t)d) y = kj_fq_compose(o, y); }
        const uint32_t ex = __shfl_up_sync(0xffffffffu, y, 1);
        sm[32 + lane] = lane ? ex : KJ_FQ_MAP_ID;
        if (lane == 31) sm[64] = y;
    }
    __syncthreads();
    total = sm[64];
    uint32_t ex = __shfl_up_sync(0xffffffffu, x, 1); if (lane == 0) ex = KJ_FQ_MAP_ID;
    const uint32_t r = kj_fq_compose(sm[32 + wid], ex);
    __syncthreads();
    return r;
}
#define KJ_FQ_TILE 2048u            // lines per block: 256 threads x 8
__global__ void kj_fq_tile_maps(const uint64_t* __restrict__ line_start, uint64_t n_lines, uint32_t* __restrict__ tile_map) {
    __shared__ uint32_t sm[80];
    const uint64_t base = (uint64_t)blockIdx.x * KJ_FQ_TILE + (uint64_t)threadIdx.x * 8u; uint32_t m = KJ_FQ_MAP_ID;
    for (int k = 0; k < 8; k++) m = kj_fq_compose(m, kj_fq_line_map(line_start, base + k, n_lines));
    uint32_t tot; (void)kj_fq_block_scan(m, sm, tot);
    if (threadIdx.x == 0) tile_map[blockIdx.x] = tot;
}
__global__ void kj_fq_tile_prefix(uint32_t* __restrict__ tile_map, uint32_t ntiles) {     // one thread: a few hundred tiles per chunk
    if (blockIdx.x || threadIdx.x) return;
    uint32_t acc = KJ_FQ_MAP_ID;
    for (uint32_t t = 0; t < ntiles; t++) { const uint32_t m = tile_map[t]; tile_map[t] = acc; acc = kj_fq_compose(acc, m); }
}
// phase[i] = phase before line i, for i in [0, n_lines] (the chunk starts at a record boundary: phase 0)
__global__ void kj_fq_phases(const uint64_t* __restrict__ line_start, uint64_t n_lines, const uint32_t* __restrict__ tile_map, uint8_t* __restrict__ phase) {
    __shared__ uint32_t sm[80];
    const uint64_t base = (uint64_t)blockIdx.x * KJ_FQ_TILE + (uint64_t)threadIdx.x * 8u; uint32_t mk[8], m = KJ_FQ_MAP_ID;
    for (int k = 0; k < 8; k++) { mk[k] = kj_fq_line_map(line_start, base + k, n_lines); m = kj_fq_compose(m, mk[k]); }
    uint32_t tot; uint32_t pre = kj_fq_compose(tile_map[blockIdx.x], kj_fq_block_scan(m, sm, tot));
    for (int k = 0; k < 8; k++) { if (base + k <= n_lines) phase[base + k] = (uint8_t)(pre & 3u); pre = kj_fq_compose(pre, mk[k]); }
}

struct KjParseDims { uint32_t fastq; uint32_t n_lines; uint32_t whole_names; };    // whole_names: kaijup keeps the header line whole
static __device__ __forceinline__ bool kj_is_letter(uint32_t c) { const uint32_t u = c & 0xDFu; return u >= 'A' && u <= 'Z'; }    // util.cpp:21-23
// what line i is: header / sequence line / neither.  FASTQ without a phase array: four lines per record from the start of the chunk; an empty
// line where a header is expected raises flag 64 (the chunk is then parsed again with the phases)
static __device__ __forceinline__ void kj_line_kind(const char* __restrict__ text, KjParseDims d, const uint8_t* __restrict__ phase, uint64_t i, uint64_t s, uint64_t e, bool& is_hdr, bool& is_seq, bool& blank) {
    blank = false;
    if (d.fastq) { const uint32_t ph = phase ? phase[i] : (uint32_t)(i & 3u); blank = ph == 0 && e == s; is_hdr = ph == 0 && !(phase && blank); is_seq = ph == 1; }
    else { is_hdr = e > s && text[s] == '>'; is_seq = !is_hdr; }
}
// one warp per complete line: cnt = letters of a sequence line, hdr = 1 for a header line, nlen = trimmed name length
__global__ void kj_line_info(const char* __restrict__ text, const uint64_t* __restrict__ line_start, KjParseDims d, const uint8_t* __restrict__ phase,
                             uint32_t* __restrict__ cnt, uint32_t* __restrict__ hdr, uint32_t* __restrict__ nlen, uint32_t* __restrict__ err) {
    const uint32_t lane = threadIdx.x & 31; const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t i = warp; i <= d.n_lines; i += nwarps) {
        if (i == d.n_lines) { if (lane == 0) { cnt[i] = 0; hdr[i] = 0; nlen[i] = 0; } continue; }     // virtual line: the scans deliver the totals here
        const uint64_t s = line_start[i], e = line_start[i + 1] - 1;                                  // [s, e) without the newline
        bool is_hdr, is_seq, blank; kj_line_kind(text, d, phase, i, s, e, is_hdr, is_seq, blank);
        if (d.fastq && lane == 0) { if (blank && !phase) atomicOr(err, 64u); if (is_hdr && e > s && text[s] != '@') atomicOr(err, 16u); }
        uint32_t c = 0, nl = 0;
        if (is_seq) {
            for (uint64_t p = s + lane; p < e; p += 32) c += kj_is_letter((uint8_t)text[p]) ? 1u : 0u;
            for (int m = 16; m > 0; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
        } else if (is_hdr) {
            // name = line without its first character, cut at the first of " /\t\r" (kaiju.cpp:279, 303-307); kaijup keeps it whole (kaijup.cpp:241, 253)
            nl = e > s ? (uint32_t)(e - (s + 1)) : 0u;
            for (uint64_t p0 = s + 1; !d.whole_names && p0 < e; p0 += 32) {
                const uint64_t p = p0 + lane; const uint32_t ch = p < e ? (uint8_t)text[p] : 0u;
                const uint32_t stop = __ballot_sync(0xffffffffu, p < e && (ch == ' ' || ch == '/' || ch == '\t' || ch == '\r'));
                if (stop) { nl = (uint32_t)(p0 - (s + 1)) + (uint32_t)(__ffs((int)stop) - 1); break; }
            }
        }
        if (lane == 0) { cnt[i] = c; hdr[i] = is_hdr ? 1u : 0u; nlen[i] = nl; }
    }
}
// after the scans: S = letters before line i, R = headers before line i, NS = name bytes before line i
__global__ void kj_line_emit(const char* __restrict__ text, const uint64_t* __restrict__ line_start, KjParseDims d, const uint8_t* __restrict__ phase,
                             const uint32_t* __restrict__ S, const uint32_t* __restrict__ R, const uint32_t* __restrict__ NS,
                             char* __restrict__ seq, uint64_t* __restrict__ off, char* __restrict__ names, uint32_t* __restrict__ name_off, uint64_t* __restrict__ rec_pos) {
    const uint32_t lane = threadIdx.x & 31; const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t i = warp; i <= d.n_lines; i += nwarps) {
        if (i == d.n_lines) { if (lane == 0) { const uint32_t r = R[i]; off[r] = S[i]; name_off[r] = NS[i]; rec_pos[r] = line_start[i]; } continue; }
        const uint64_t s = line_start[i], e = line_start[i + 1] - 1;
        bool is_hdr, is_seq, blank; kj_line_kind(text, d, phase, i, s, e, is_hdr, is_seq, blank);
        if (is_hdr) {
            const uint32_t r = R[i], nl = NS[i + 1] - NS[i];
            if (lane == 0) { off[r] = S[i]; name_off[r] = NS[i]; rec_pos[r] = s; }
            for (uint32_t k = lane; k < nl; k += 32) names[NS[i] + k] = text[s + 1 + k];
        } else if (is_seq) {
            uint64_t dst = S[i];
            for (uint64_t p0 = s; p0 < e; p0 += 32) {
                const uint64_t p = p0 + lane; const char ch = p < e ? text[p] : 0; const bool l = p < e && kj_is_letter((uint8_t)ch);
                const uint32_t m = __ballot_sync(0xffffffffu, l);
                if (l) seq[dst + (uint32_t)__popc(m & ((1u << lane) - 1u))] = ch;
                dst += (uint32_t)__popc(m);
            }
        }
    }
}
// paired input: names of both files must be identical record by record (kaiju.cpp:359-362, 377-380)
__global__ void kj_names_equal(const char* __restrict__ na, const uint32_t* __restrict__ oa, const char* __restrict__ nb, const uint32_t* __restrict__ ob, uint64_t n, uint32_t* __restrict__ err) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t la = oa[r + 1] - oa[r], lb = ob[r + 1] - ob[r]; bool same = la == lb;
        for (uint32_t k = 0; same && k < la; k++) same = na[oa[r] + k] == nb[ob[r] + k];
        if (!same) atomicOr(err, 32u);
    }
}

// ------------------------------------------------------------------------------------------------
// output lines: one length pass, one scan, one write pass over the lines of kj_format.h
// ------------------------------------------------------------------------------------------------
// length of every line (one thread per read: the columns' lengths are a few loads each); n_classified counts the "C" lines
__global__ void kj_fmt_len(const __grid_constant__ KjFmtIn in, uint64_t n, uint32_t* __restrict__ len, unsigned long long* __restrict__ n_classified) {
    uint32_t ccount = 0;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (uint64_t)gridDim.x * blockDim.x) {
        if (r == n) { len[r] = 0; continue; }
        if (kj_fmt_status(in, r) == 2) ccount++;
        len[r] = kj_fmt_line(in, r, nullptr, 0, 1);
    }
    for (int m = 16; m > 0; m >>= 1) ccount += __shfl_xor_sync(0xffffffffu, ccount, m);
    if ((threadIdx.x & 31) == 0 && ccount) atomicAdd(n_classified, (unsigned long long)ccount);
}
// the lines at their scanned positions: formats 0 and 1 (a name and a few numbers) one thread per read; the formats with string columns
// (accessions, labels, fragment strings of up to kilobytes) one warp per read, the strings copied lane-strided
__global__ void kj_fmt_write(const __grid_constant__ KjFmtIn in, uint64_t n, const uint32_t* __restrict__ pos, char* __restrict__ out) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (uint64_t)gridDim.x * blockDim.x;
    if (in.fmt <= KJ_OUT_KAIJU_IDS) { for (uint64_t r = tid; r < n; r += nthr) kj_fmt_line(in, r, out + pos[r], 0, 1); return; }
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t r = tid >> 5; r < n; r += nthr >> 5) kj_fmt_line(in, r, out + pos[r], lane, 32);
}

// The front-end gate of kaijux / kaijup, one warp per read (gate[r] = 1: the line is "U\t<name>\t0"):
//   DNA (ConsumerThreadx.cpp:202-207): every mate shorter than 3 m;
//   protein (ConsumerThreadp.cpp:16-20, 22-70): shorter than m, or no piece between letters outside the 20 residues (upper-cased) of at least m
//   residues -- in Greedy also with a BLOSUM62 self-score of at least min_score.
// A piece is closed at each splitting letter: the window's inclusive prefix sums of the scores give its score, the piece that runs into the next
// window is carried.
__global__ void kj_name_gate(const char* __restrict__ seq, const uint64_t* __restrict__ off1, const uint64_t* __restrict__ off2, uint64_t n, uint32_t m,
                             int protein, int greedy, uint32_t min_score, uint8_t* __restrict__ gate) {
    const uint32_t lane = threadIdx.x & 31; const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t r = warp; r < n; r += nwarps) {
        const uint64_t b = off1[r], e = off1[r + 1], l1 = e - b;
        if (!protein) {
            if (lane == 0) gate[r] = off2 ? (l1 < 3u * m && off2[r + 1] - off2[r] < 3u * m) : l1 < 3u * m;
            continue;
        }
        bool any = false; uint64_t clen = 0, cscore = 0;      // the open piece
        auto piece = [&](uint64_t len, uint64_t score) { return len >= m && (!greedy || score >= min_score); };
        for (uint64_t p0 = b; l1 >= m && p0 < e && !any; p0 += 32) {
            const uint64_t p = p0 + lane; const uint32_t wl = e - p0 < 32 ? (uint32_t)(e - p0) : 32u;
            const uint32_t c = p < e ? ((uint32_t)(uint8_t)seq[p] & 0xDFu) : 0u, sc = p < e ? kj_fmt_self_score(c) : 0u;
            const uint32_t brk = __ballot_sync(0xffffffffu, p < e && sc == 0);
            uint32_t ps = sc;      // inclusive prefix sum of the scores in the window
            for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, ps, d); if (lane >= (uint32_t)d) ps += o; }
            const uint32_t tot = __shfl_sync(0xffffffffu, ps, wl - 1);
            const uint32_t below = brk & ((1u << lane) - 1u); const int q = below ? 31 - __clz((int)below) : 0;     // the previous splitting letter
            const uint32_t psq = __shfl_sync(0xffffffffu, ps, q);
            bool mine = false;
            if ((brk >> lane) & 1u) mine = below ? piece((uint64_t)(lane - q - 1), ps - psq) : piece(clen + lane, cscore + ps);
            any = __any_sync(0xffffffffu, mine);
            if (brk) { const int q = 31 - __clz((int)brk); clen = wl - 1 - (uint32_t)q; cscore = tot - __shfl_sync(0xffffffffu, ps, q); }
            else { clen += wl; cscore += tot; }
        }
        if (!any && l1 >= m) any = piece(clen, cscore);
        if (lane == 0) gate[r] = any ? 0 : 1;
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Room for `bytes` in an ingest buffer, grown with slack; boost: allocate for a batch that many times as large (cudaFree waits for every
// running kernel: avoid regrowth while the batches ramp up)
static int kj_need(KjDevBuf& b, size_t bytes, float boost = 1.f) { return b.grow(bytes, (size_t)((double)bytes * boost) + bytes / 4 + 4096); }
static int kj_scan_u32(uint32_t* d, uint64_t n, KjDevBuf& tmp, float boost, uint32_t* d_total, cudaStream_t st) {
    const uint32_t nb = (uint32_t)((n + KJ_SCAN_TILE - 1) / KJ_SCAN_TILE);
    int rc = kj_need(tmp, (size_t)(nb + 1) * sizeof(uint32_t), boost); if (rc) return rc;
    kj_scan_reduce<<<nb, 256, 0, st>>>(d, n, tmp.as<uint32_t>());
    kj_scan_blocks<<<1, 1024, 0, st>>>(tmp.as<uint32_t>(), nb, d_total);
    kj_scan_apply<<<nb, 256, 0, st>>>(d, n, tmp.as<uint32_t>());
    CK(cudaGetLastError());
    return KJ_OK;
}

// Pinned host buffers outlive one kj_classify_files call (allocation and release cost ~0.3 ms per MB).  Portable: the output buffers of
// kj_classify_files_multi take device-to-host copies from the contexts of every device.
struct KjPinnedPool {
    std::mutex mu; std::vector<std::pair<char*, size_t>> idle;
    char* get(size_t bytes) {
        { std::lock_guard<std::mutex> lk(mu); for (size_t k = 0; k < idle.size(); k++) if (idle[k].second == bytes) { char* b = idle[k].first; idle.erase(idle.begin() + k); return b; } }
        char* b = nullptr; return cudaHostAlloc((void**)&b, bytes, cudaHostAllocPortable) == cudaSuccess ? b : nullptr;
    }
    void put(char* b, size_t bytes) { std::lock_guard<std::mutex> lk(mu); idle.push_back({b, bytes}); }
    void release() { std::lock_guard<std::mutex> lk(mu); for (auto& e : idle) cudaFreeHost(e.first); idle.clear(); }
};

struct KjBatchSide {     // what the parser hands to the classifier for one input file
    KjDevBuf seq, off, names, name_off;
    size_t bytes[4] = {0, 0, 0, 0};       // the bytes of the four buffers the parse wrote (what a context on another device copies)
};
struct KjParsed {   // one side (file) of a chunk while it is parsed
    KjDevBuf text[2]; int cur = 0; uint64_t nbytes = 0;         // device text (ping-pong for the carry), valid bytes
    KjDevBuf line_start, cnt, hdr, nlen, tiles, scan_tmp, rec_pos, totals, phase, phase_tiles;
    int fastq = -1;                                              // file type, fixed by the first byte of the file
    bool whole_names = false;                                    // kaijup's reader: names not trimmed, the file type from the first line as it is
    uint64_t n_lines = 0, n_rec = 0, consumed = 0; bool eof = false, skip_all = false;
};

// Parse the complete records in P.text[P.cur][0, P.nbytes) into O.  Sets P.n_rec; *launches counts the kernels.
// exact: FASTQ with blank lines between records (phases from the automaton scan instead of line number mod 4).  boost: the batch's (kj_need).
// Both files of a pair go through the three stages together: the parser's stream synchronises three times per batch (line count, totals, end), not
// three times per file -- each host round trip is a gap in which the persistent classify grid of the other pipeline stage takes every free SM slot.
static int kj_parse_sides(int sm_count, KjParsed* Ps, KjBatchSide* Os, int nfiles, const std::string* fn, cudaStream_t st, uint32_t* d_perr, uint64_t* launches, bool exact, float boost) {
    int rc; bool on[2] = {false, false}; uint32_t ntiles[2] = {0, 0}, nl[2] = {0, 0}, h[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}}; uint8_t end_phase[2] = {0, 0}; const uint8_t* phase[2] = {nullptr, nullptr};
    const int blocks = sm_count * 8;
    // stage 0: file type (first batch of a file only), newline counts
    for (int f = 0; f < nfiles; f++) {
        KjParsed& P = Ps[f];
        P.n_rec = 0; P.consumed = 0; P.n_lines = 0; P.skip_all = false;
        if (P.nbytes == 0) continue;
        if (P.nbytes >= (1ull << 31)) { kj_err() = "kj_classify_files: a single record larger than 2 GB"; return KJ_ERR_UNSUPPORTED; }
        const char* text = P.text[P.cur].as<char>();
        if (P.fastq < 0) {
            // the file type is the first character of the first non-empty line (kaiju.cpp:289-299: empty lines are skipped before it is looked at)
            char first = '\n', first_byte = 0; std::vector<char> head;
            for (uint64_t at = 0, win = 256; first == '\n' && at < P.nbytes; at += head.size(), win *= 4) {
                head.resize((size_t)std::min<uint64_t>(win, P.nbytes - at));
                CK(cudaMemcpyAsync(head.data(), text + at, head.size(), cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
                if (at == 0) first_byte = head[0];
                for (char ch : head) if (ch != '\n') { first = ch; break; }
            }
            if (P.whole_names) first = first_byte;                                    // kaijup.cpp:228-236: the first line, even an empty one
            else if (first == '\n') { P.skip_all = true; continue; }                  // nothing but empty lines so far: they are dropped
            if (first == '@') P.fastq = 1; else if (first == '>') P.fastq = 0;
            else { kj_err() = "Auto-detection of file type for file " + fn[f] + " failed."; return KJ_ERR_IO; }                 // kaiju.cpp:296-299
        }
        ntiles[f] = (uint32_t)((P.nbytes + KJ_NL_TILE - 1) / KJ_NL_TILE);
        if ((rc = kj_need(P.tiles, (size_t)(ntiles[f] + 1) * 4, boost)) || (rc = kj_need(P.totals, 64))) return rc;
        kj_nl_count<<<ntiles[f], 256, 0, st>>>(text, P.nbytes, P.tiles.as<uint32_t>());
        if ((rc = kj_scan_u32(P.tiles.as<uint32_t>(), ntiles[f], P.scan_tmp, boost, P.totals.as<uint32_t>() + 0, st))) return rc;
        CK(cudaMemcpyAsync(&nl[f], P.totals.as<uint32_t>() + 0, 4, cudaMemcpyDeviceToHost, st));
        on[f] = true; *launches += 4;
    }
    CK(cudaStreamSynchronize(st));
    // stage 1: line starts, per-line classes, the three scans
    for (int f = 0; f < nfiles; f++) {
        KjParsed& P = Ps[f];
        if (!on[f]) continue;
        P.n_lines = nl[f];
        if (nl[f] == 0) { on[f] = false; continue; }                                  // not even one complete line yet
        const char* text = P.text[P.cur].as<char>(); uint32_t* tot = P.totals.as<uint32_t>();
        const size_t L1 = (size_t)nl[f] + 1;
        if ((rc = kj_need(P.line_start, (L1 + 1) * 8, boost)) || (rc = kj_need(P.cnt, (L1 + 1) * 4, boost)) || (rc = kj_need(P.hdr, (L1 + 1) * 4, boost)) ||
            (rc = kj_need(P.nlen, (L1 + 1) * 4, boost))) return rc;
        kj_nl_scatter<<<ntiles[f], 256, 0, st>>>(text, P.nbytes, P.tiles.as<uint32_t>(), P.line_start.as<uint64_t>());
        KjParseDims d; d.fastq = (uint32_t)P.fastq; d.n_lines = nl[f]; d.whole_names = P.whole_names ? 1u : 0u;
        if (P.fastq && exact) {
            const uint32_t nt = (uint32_t)((L1 + KJ_FQ_TILE - 1) / KJ_FQ_TILE);
            if ((rc = kj_need(P.phase, L1 + 8, boost)) || (rc = kj_need(P.phase_tiles, (size_t)(nt + 1) * 4, boost))) return rc;
            kj_fq_tile_maps<<<nt, 256, 0, st>>>(P.line_start.as<uint64_t>(), nl[f], P.phase_tiles.as<uint32_t>());
            kj_fq_tile_prefix<<<1, 32, 0, st>>>(P.phase_tiles.as<uint32_t>(), nt);
            kj_fq_phases<<<nt, 256, 0, st>>>(P.line_start.as<uint64_t>(), nl[f], P.phase_tiles.as<uint32_t>(), P.phase.as<uint8_t>());
            phase[f] = P.phase.as<uint8_t>(); *launches += 3;
        }
        kj_line_info<<<blocks, 256, 0, st>>>(text, P.line_start.as<uint64_t>(), d, phase[f], P.cnt.as<uint32_t>(), P.hdr.as<uint32_t>(), P.nlen.as<uint32_t>(), d_perr);
        if ((rc = kj_scan_u32(P.cnt.as<uint32_t>(), L1, P.scan_tmp, boost, tot + 1, st)) || (rc = kj_scan_u32(P.hdr.as<uint32_t>(), L1, P.scan_tmp, boost, tot + 2, st)) ||
            (rc = kj_scan_u32(P.nlen.as<uint32_t>(), L1, P.scan_tmp, boost, tot + 3, st))) return rc;
        CK(cudaMemcpyAsync(h[f], tot, 16, cudaMemcpyDeviceToHost, st));
        if (phase[f]) CK(cudaMemcpyAsync(&end_phase[f], phase[f] + nl[f], 1, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    // stage 2: packed sequences, offsets, names (the caller synchronises once more after its own kernels)
    for (int f = 0; f < nfiles; f++) {
        KjParsed& P = Ps[f]; KjBatchSide& O = Os[f];
        if (!on[f]) continue;
        const char* text = P.text[P.cur].as<char>();
        const uint64_t letters = h[f][1], headers = h[f][2], name_bytes = h[f][3];
        O.bytes[0] = letters + 64; O.bytes[1] = (headers + 2) * 8; O.bytes[2] = name_bytes + 64; O.bytes[3] = (headers + 2) * 4;
        if ((rc = kj_need(O.seq, O.bytes[0], boost)) || (rc = kj_need(O.off, O.bytes[1], boost)) || (rc = kj_need(O.names, O.bytes[2], boost)) ||
            (rc = kj_need(O.name_off, O.bytes[3], boost)) || (rc = kj_need(P.rec_pos, (headers + 2) * 8, boost))) return rc;
        KjParseDims d; d.fastq = (uint32_t)P.fastq; d.n_lines = nl[f]; d.whole_names = P.whole_names ? 1u : 0u;
        kj_line_emit<<<blocks, 256, 0, st>>>(text, P.line_start.as<uint64_t>(), d, phase[f], P.cnt.as<uint32_t>(), P.hdr.as<uint32_t>(), P.nlen.as<uint32_t>(),
                                            O.seq.as<char>(), O.off.as<uint64_t>(), O.names.as<char>(), O.name_off.as<uint32_t>(), P.rec_pos.as<uint64_t>());
        CK(cudaGetLastError()); *launches += 12;
        // complete records: FASTQ = whole groups of four lines; FASTA = every header that is followed by another header (or by the end of the file)
        if (P.fastq) { P.n_rec = phase[f] ? (end_phase[f] == 0 ? headers : (headers ? headers - 1 : 0)) : nl[f] / 4; }       // a record is complete with its fourth line
        else { P.n_rec = P.eof ? headers : (headers ? headers - 1 : 0); }
    }
    return KJ_OK;
}

static inline double kj_ms_since(std::chrono::steady_clock::time_point& t) { const auto n = std::chrono::steady_clock::now(); const double d = std::chrono::duration<double, std::milli>(n - t).count(); t = n; return d; }
// One I/O chunk of an input file, already on its way to the device: slot of the reader's staging ring + the event of its copy
struct KjStaged { int slot = -1; size_t n = 0; bool eof = false; char last = 0; cudaEvent_t ev = nullptr; std::string error; };
// Per input file: gz (zlib, one thread) or plain (a pool of pread() threads) -> two alternating pinned buffers -> host-to-device copies on the
// reader's own stream into a ring of device staging buffers.  The parser only ever sees device memory; the pinned footprint is two chunks.
// BGZF (a gzip file whose first member carries the "BC" extra subfield): the compressed bytes are read like a plain file's, the block chain is
// walked on the host and the blocks are inflated on the device straight into the ring slot a plain chunk would have been copied to; a later
// member that is no BGZF block sends the rest of the file to zlib.
// Input that cannot seek (fstat: not a regular file -- a FIFO, a pipe, /dev/stdin, a character device) is read once, front to back, by the
// reader thread alone (KjStream, kj_stream.h): its first 64 KiB are the format probe and then the start of the first chunk, BGZF round or zlib
// input; a BGZF round carries what it did not consume to the front of the next round's buffer; other gzip goes through a z_stream.  The
// descriptor is opened with O_NONBLOCK, so the two files of a pair are open before either has a writer, and every wait of the thread is a poll()
// that halt() ends.
// A pair of streams from one writer (samtools fastq -1 a -2 b): the parser fills side 0 up to its target (at most batch_max + chunk bytes of
// text) before side 1, so file 2's reader must hold what the writer puts into file 2 meanwhile: its ring of `depth` = min(64, batch_max / chunk + 4)
// chunks plus the chunk in its pinned buffer (and the pipe's own buffer).  That covers records of file 2 up to (depth + 1) * chunk /
// (batch_max + chunk) times as long as file 1's -- 1.44 with the default 16 MB chunks and 128 MB batches, 3 with KJ_INGEST_CHUNK alone -- and, while
// side 1 is filled, records of file 1 up to ((depth + 1) * chunk + batch_max) / (batch_max + chunk) times as long as file 2's (2.33, 3.5).  Mates
// of 150 and 100 bases (about 1.47 : 1 in FASTQ bytes with short names) lie within both bounds with 150-base mates in file 1; a skew beyond them
// stalls the writer and with it the call.
struct KjFileReader {
    gzFile fp = nullptr; int fd = -1; uint64_t file_off = 0; std::string path; size_t chunk = 0; int device = 0; KjPinnedPool* pinned = nullptr;
    bool is_stream = false; KjStream src; KjGzStream gz; size_t left_at = 0, left_n = 0;     // input that cannot seek; a BGZF round's unconsumed bytes
    // Pairs: file 1's reader (follower = file 2's) hands its error to file 2's as lead_error.  The parser takes file 1's chunks before file 2's
    // and ends only at the end of file 1, so that error ends the call whatever file 2 still holds; a wait for the next chunk of a file-2 stream
    // returns it at once (the stream's writer may be waiting for file 1 to be read).
    KjFileReader* follower = nullptr; std::string lead_error;
    char* pin[2] = {nullptr, nullptr}; cudaEvent_t pin_ev[2] = {nullptr, nullptr}; bool pin_busy[2] = {false, false}; cudaStream_t stream = nullptr;
    std::vector<KjDevBuf> ring; std::vector<cudaEvent_t> ring_ev; std::deque<int> free_slots; std::deque<KjStaged> ready;
    std::mutex mu; std::condition_variable cv; std::thread th; bool stop = false;
    // plain files: NT worker threads copy 1 MB slices of the current chunk out of the page cache in parallel (a single thread moves ~1-3 GB/s)
    static constexpr size_t SLICE = 1u << 20;
    std::vector<std::thread> workers; std::mutex wmu; std::condition_variable wcv, wdone; char* wbuf = nullptr; size_t wnext = 0, wslices = 0, wleft = 0; uint64_t wgen = 0; bool wstop = false, werr = false;
    std::vector<size_t> wgot;
    // BGZF: bytes read per round (a whole block always fits), size of a ring slot, most blocks per round; the compressed bytes, the block table
    // and the blocks' status words of a round share one pinned buffer and one device buffer (two of each: one round is in flight while the next is read)
    bool bgzf = false; size_t rchunk = 0, slot_bytes = 0, max_blocks = 0, tab_off = 0, st_off = 0, last_off = 0, zbytes = 0;
    char* zpin[2] = {nullptr, nullptr}; KjDevBuf zdev[2]; cudaStream_t zstream = nullptr; std::vector<KjBgzfBlock> table;
    uint64_t inflated = 0; char last_byte = 0; double tm_read = 0, tm_inflate = 0;
    void worker() {
        uint64_t seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> lk(wmu);
            wcv.wait(lk, [&] { return wstop || (wgen != seen && wnext < wslices); });
            if (wstop) return;
            const uint64_t gen = wgen;
            while (wgen == gen && wnext < wslices) {
                const size_t sl = wnext++; char* b = wbuf; const uint64_t base = file_off;
                lk.unlock();
                const size_t o = sl * SLICE, want = std::min(SLICE, rchunk - o); size_t g = 0; bool bad = false;
                while (g < want) { const ssize_t r = ::pread(fd, b + o + g, want - g, (off_t)(base + o + g)); if (r < 0) { bad = true; break; } if (r == 0) break; g += (size_t)r; }
                lk.lock();
                wgot[sl] = g; if (bad) werr = true;
                if (--wleft == 0) wdone.notify_all();
            }
            seen = gen;
        }
    }
    int open(const std::string& p, size_t chunk_bytes, int depth, int device_, KjPinnedPool* pp) {
        path = p; chunk = chunk_bytes; device = device_; pinned = pp; stop = false; wstop = false; file_off = 0; inflated = 0; last_byte = 0; tm_read = tm_inflate = 0;
        left_at = left_n = 0;
        fd = ::open(p.c_str(), O_RDONLY | O_NONBLOCK);           // a FIFO opens at once, with or without a writer
        struct stat sb;
        if (fd < 0 || fstat(fd, &sb) != 0) { if (fd >= 0) ::close(fd); fd = -1; kj_err() = "Could not open file " + p; return KJ_ERR_IO; }
        is_stream = !S_ISREG(sb.st_mode);
        if (is_stream) {      // the format is probed on the reader thread: the first read may wait for the writer
            const int sfd = fd; fd = -1;
            if (!src.open(sfd)) { src.close(); kj_err() = "Could not open file " + p + " (eventfd)"; return KJ_ERR_IO; }
            return start(depth);
        }
        (void)fcntl(fd, F_SETFL, fcntl(fd, F_GETFL) & ~O_NONBLOCK);
        std::vector<uint8_t> head(65536); const ssize_t got = ::pread(fd, head.data(), head.size(), 0);
        const int format = kj_input_format(head.data(), got > 0 ? (size_t)got : 0);
        bgzf = format == KJ_INPUT_BGZF; layout();
        if (format == KJ_INPUT_GZIP) {             // other gzip: inflate through zlib; everything else is read as it is
            ::close(fd); fd = -1; fp = gzopen(p.c_str(), "rb");
            if (!fp) { kj_err() = "Could not open file " + p; return KJ_ERR_IO; }
            gzbuffer(fp, 1 << 20);
        } else {
            posix_fadvise(fd, 0, 0, POSIX_FADV_SEQUENTIAL);
            unsigned nt = std::max(2u, std::min(8u, std::thread::hardware_concurrency() / 4u));
            if (const char* v = getenv("KJ_IO_THREADS")) { const long x = atol(v); if (x >= 1 && x <= 64) nt = (unsigned)x; }      // tuning hook
            wgot.assign((rchunk + SLICE - 1) / SLICE, 0);
            for (unsigned t = 0; t < nt; t++) workers.emplace_back([this] { worker(); });
        }
        return start(depth);
    }
    int start(int depth) {
        if ((int)ring.size() != depth) { ring.clear(); ring.resize((size_t)depth); }
        free_slots.clear(); ready.clear(); for (int k = 0; k < depth; k++) free_slots.push_back(k);
        th = std::thread([this] { run(); });
        return KJ_OK;
    }
    void layout() {        // the sizes of a round and of a ring slot, once the format is known
        rchunk = bgzf ? std::max<size_t>(chunk, 65536) : chunk; slot_bytes = rchunk + 16;
        max_blocks = rchunk / 1024 + 64; tab_off = (rchunk + 63) & ~(size_t)63; st_off = tab_off + max_blocks * sizeof(KjBgzfBlock); last_off = st_off + max_blocks * 4; zbytes = last_off + 16;
    }
    // a stream's first bytes (up to 64 KiB) decide its format as a file's do; they are put back in front of the stream.  false: the call is over
    bool probe() {
        std::vector<char> head(65536); size_t got = 0; bool eof = false;
        const int r = src.fill(head.data(), head.size(), got, eof);
        if (r) { if (r != KJ_STREAM_HALTED) fail("read error in file " + path); return false; }
        const int format = kj_input_format((const uint8_t*)head.data(), got);
        src.unread(head.data(), got);
        bgzf = format == KJ_INPUT_BGZF; layout();
        if (format == KJ_INPUT_GZIP && !gz.start()) { fail("Could not open file " + path + " (inflateInit2)"); return false; }
        return true;
    }
    // one round of the worker pool: the rchunk bytes at file_off (fewer at the end of the file) into b.  false: read error
    bool read_round(char* b, size_t& got, bool& eof) {
        const size_t ns = (rchunk + SLICE - 1) / SLICE; got = 0; eof = false;
        {
            std::unique_lock<std::mutex> lk(wmu);
            wbuf = b; wnext = 0; wslices = ns; wleft = ns; werr = false; wgen++;
            wcv.notify_all();
            wdone.wait(lk, [&] { return wleft == 0; });
            wslices = 0;
        }
        if (werr) return false;
        for (size_t sl = 0; sl < ns; sl++) {
            got += wgot[sl];
            if (wgot[sl] < std::min(SLICE, rchunk - sl * SLICE)) { eof = true; break; }          // short slice = end of file (later slices read nothing)
        }
        if (got == rchunk && !eof) { char probe; if (::pread(fd, &probe, 1, (off_t)(file_off + rchunk)) == 0) eof = true; }
        return true;
    }
    // The BGZF blocks of the file, round by round.  false: the file is done (its last chunk or an error is queued); true: a gzip member that is no
    // BGZF block starts at file_off, and zlib (fp) reads the rest.
    bool run_bgzf() {
        struct Flight { KjStaged ck; int pb = 0; size_t nblk = 0; uint64_t off = 0; bool on = false; } prev, cur;
        auto finish = [&](Flight& f) -> bool {      // the round's blocks are inflated and good: its chunk goes to the parser
            if (!f.on) return true;
            auto t0 = std::chrono::steady_clock::now();
            if (cudaEventSynchronize(f.ck.ev) != cudaSuccess) { fail("inflating " + path + " failed on the device"); return false; }
            tm_inflate += kj_ms_since(t0);
            const uint32_t* st = (const uint32_t*)(zpin[f.pb] + st_off); const KjBgzfBlock* tb = (const KjBgzfBlock*)(zpin[f.pb] + tab_off);
            for (size_t i = 0; i < f.nblk; i++) if (st[i]) { fail(kj_bgzf_block_error(path, f.off, tb[i], st[i])); return false; }
            if (f.ck.n) last_byte = zpin[f.pb][last_off];
            f.ck.last = last_byte; f.on = false;
            { std::lock_guard<std::mutex> lk(mu); ready.push_back(f.ck); }
            cv.notify_all(); return true;
        };
        if (!zstream) { int lo = 0, hi = 0;      // beside the parse stream: the inflate kernel, too, has to find room next to the persistent classify grid
            if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess || cudaStreamCreateWithPriority(&zstream, cudaStreamNonBlocking, hi) != cudaSuccess) { fail("cudaStreamCreate failed"); return false; } }
        for (uint64_t it = 0;; it++) {
            const int pb = (int)(it & 1);          // the round that used this pair of buffers has been finished one round ago
            if (!zpin[pb]) { zpin[pb] = pinned->get(zbytes); if (!zpin[pb]) { fail("cudaMallocHost failed"); return false; } }
            if (zdev[pb].grow(zbytes) != KJ_OK) { fail("cudaMalloc failed (compressed staging)"); return false; }
            char* b = zpin[pb]; size_t got = 0; bool ceof = false;
            auto t0 = std::chrono::steady_clock::now();
            if (is_stream) {         // the other buffer's unconsumed bytes (that round is in flight: its copy reads only the bytes it consumed), then the stream
                const int r = kj_bgzf_top_up(src, b, rchunk, zpin[pb ^ 1], left_at, left_n, got, ceof);
                if (r) { if (r != KJ_STREAM_HALTED) fail("read error in file " + path); return false; }
            } else if (!read_round(b, got, ceof)) { fail("read error in file " + path); return false; }
            tm_read += kj_ms_since(t0);
            const KjBgzfRound plan = kj_bgzf_plan((const uint8_t*)b, got, ceof, slot_bytes - 16, max_blocks, file_off, path, table);
            if (!plan.error.empty()) { fail(plan.error); return false; }
            const KjBgzfWalk w = plan.w; const bool eof = plan.eof, to_zlib = plan.to_zlib;
            left_at = w.consumed; left_n = got - w.consumed;
            cur = Flight(); cur.pb = pb; cur.nblk = table.size(); cur.off = file_off; cur.on = true; cur.ck.n = (size_t)w.out_bytes; cur.ck.eof = eof;
            {   // a free staging buffer on the device
                std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return stop || !free_slots.empty(); }); if (stop) return false;
                cur.ck.slot = free_slots.front(); free_slots.pop_front();
            }
            if (kj_need(ring[cur.ck.slot], slot_bytes) != KJ_OK) { fail("cudaMalloc failed (staging ring)"); return false; }
            if (cur.nblk) {
                memcpy(b + tab_off, table.data(), cur.nblk * sizeof(KjBgzfBlock));
                char* d = zdev[pb].as<char>(); bool ok = true;
                ok = ok && cudaMemcpyAsync(d, b, w.consumed, cudaMemcpyHostToDevice, zstream) == cudaSuccess;
                ok = ok && cudaMemcpyAsync(d + tab_off, b + tab_off, cur.nblk * sizeof(KjBgzfBlock), cudaMemcpyHostToDevice, zstream) == cudaSuccess;
                if (ok) kj_inflate_kernel<<<(unsigned)((cur.nblk + KJ_INF_WARPS - 1) / KJ_INF_WARPS), KJ_INF_WARPS * 32, 0, zstream>>>((const uint8_t*)d, (const KjBgzfBlock*)(d + tab_off), (uint32_t)cur.nblk,
                                                                                                                                      ring[cur.ck.slot].as<uint8_t>(), (uint32_t*)(d + st_off));
                ok = ok && cudaGetLastError() == cudaSuccess;
                ok = ok && cudaMemcpyAsync(b + st_off, d + st_off, cur.nblk * 4, cudaMemcpyDeviceToHost, zstream) == cudaSuccess;
                if (cur.ck.n) ok = ok && cudaMemcpyAsync(b + last_off, ring[cur.ck.slot].as<char>() + cur.ck.n - 1, 1, cudaMemcpyDeviceToHost, zstream) == cudaSuccess;
                if (!ok) { fail("launching the inflate kernel failed"); return false; }
            }
            cudaEventRecord(ring_ev[cur.ck.slot], zstream); cur.ck.ev = ring_ev[cur.ck.slot];
            file_off += w.consumed; inflated += w.out_bytes;
            if (!finish(prev)) return false;
            prev = cur;
            if (!eof && !to_zlib) continue;
            if (!finish(prev) || eof) return false;
            if (is_stream) {         // zlib takes the unconsumed bytes, then the rest of the stream
                src.unread(b + left_at, left_n);
                if (!gz.start()) { fail("Could not open file " + path + " (inflateInit2)"); return false; }
                return true;
            }
            if (::lseek(fd, (off_t)file_off, SEEK_SET) < 0 || !(fp = gzdopen(fd, "rb"))) { fail("Could not open file " + path); return false; }
            fd = -1; gzbuffer(fp, 1 << 20);
            return true;
        }
    }
    void fail(const std::string& what) {
        KjStaged e; e.error = what; { std::lock_guard<std::mutex> lk(mu); ready.push_back(e); } cv.notify_all();
        if (follower) { { std::lock_guard<std::mutex> lk(follower->mu); follower->lead_error = what; } follower->cv.notify_all(); }
    }
    void run() {
        if (cudaSetDevice(device) != cudaSuccess) { fail("cudaSetDevice failed"); return; }
        if (!stream && cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) { fail("cudaStreamCreate failed"); return; }
        while (ring_ev.size() < ring.size()) { cudaEvent_t e; if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) { fail("cudaEventCreate failed"); return; } ring_ev.push_back(e); }
        if (is_stream && !probe()) return;
        if (bgzf && !run_bgzf()) return;
        char prev_last = last_byte;
        for (uint64_t it = 0;; it++) {
            const int pb = (int)(it & 1);
            if (!pin[pb]) {       // allocated here, next to the running pipeline, not before it starts
                pin[pb] = pinned->get(chunk);
                if (!pin[pb] || cudaEventCreateWithFlags(&pin_ev[pb], cudaEventDisableTiming) != cudaSuccess) { fail("cudaMallocHost failed"); return; }
            }
            if (pin_busy[pb]) { cudaEventSynchronize(pin_ev[pb]); pin_busy[pb] = false; }     // the copy that read this buffer two chunks ago
            char* b = pin[pb]; KjStaged ck; size_t got = 0;
            if (fd >= 0) {
                if (!read_round(b, got, ck.eof)) ck.error = "read error in file " + path;
                file_off += got;
            } else if (is_stream) {
                const int r = gz.on ? gz.read(src, b, chunk, got, ck.eof) : src.fill(b, chunk, got, ck.eof);
                if (r == KJ_STREAM_HALTED) return;
                if (r) ck.error = "read error in file " + path;
            } else while (got < chunk) {
                const ssize_t r = (ssize_t)gzread(fp, b + got, (unsigned)std::min<size_t>(chunk - got, 1u << 30));
                if (r < 0) { ck.error = "read error in file " + path; break; }
                if (r == 0) { ck.eof = true; break; }
                got += (size_t)r;
            }
            if (!ck.error.empty()) { fail(ck.error); return; }
            ck.n = got; if (got) prev_last = b[got - 1]; ck.last = prev_last;
            {   // a free staging buffer on the device
                std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return stop || !free_slots.empty(); }); if (stop) return;
                ck.slot = free_slots.front(); free_slots.pop_front();
            }
            if (kj_need(ring[ck.slot], slot_bytes) != KJ_OK) { fail("cudaMalloc failed (staging ring)"); return; }
            if (got && cudaMemcpyAsync(ring[ck.slot].p, b, got, cudaMemcpyHostToDevice, stream) != cudaSuccess) { fail("cudaMemcpyAsync failed"); return; }
            cudaEventRecord(ring_ev[ck.slot], stream); cudaEventRecord(pin_ev[pb], stream); pin_busy[pb] = true; ck.ev = ring_ev[ck.slot];
            const bool last = ck.eof;
            { std::lock_guard<std::mutex> lk(mu); ready.push_back(ck); }
            cv.notify_all();
            if (last) return;
        }
    }
    KjStaged next() {
        std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return stop || !ready.empty() || (is_stream && !lead_error.empty()); });
        if (ready.empty()) { KjStaged e; e.error = stop ? "the call was stopped" : lead_error; return e; }      // halt(): the call is failing elsewhere
        KjStaged ck = ready.front(); ready.pop_front(); return ck;
    }
    void release_slot(int slot) { { std::lock_guard<std::mutex> lk(mu); free_slots.push_back(slot); } cv.notify_all(); }
    // ends every wait of the reader thread and of next(), a read from a stream included
    void halt() { { std::lock_guard<std::mutex> lk(mu); stop = true; } cv.notify_all(); src.halt(); }
    void close() {
        halt();
        if (th.joinable()) th.join();
        { std::lock_guard<std::mutex> lk(wmu); wstop = true; } wcv.notify_all();
        for (auto& w : workers) if (w.joinable()) w.join();
        workers.clear();
        if (stream) cudaStreamSynchronize(stream);
        if (zstream) cudaStreamSynchronize(zstream);
        for (int k = 0; k < 2; k++) { if (zpin[k]) pinned->put(zpin[k], zbytes); zpin[k] = nullptr; }
        if (fp) gzclose(fp); fp = nullptr;
        if (fd >= 0) ::close(fd); fd = -1;
        gz.end(); src.close(); is_stream = false;
        for (int k = 0; k < 2; k++) { if (pin[k]) pinned->put(pin[k], chunk); pin[k] = nullptr; pin_busy[k] = false; if (pin_ev[k]) cudaEventDestroy(pin_ev[k]); pin_ev[k] = nullptr; }
        ready.clear(); free_slots.clear(); wgen = 0; wslices = 0; wnext = 0; wleft = 0;
    }
    void release() { for (auto e : ring_ev) cudaEventDestroy(e); ring_ev.clear(); if (stream) cudaStreamDestroy(stream); stream = nullptr; if (zstream) cudaStreamDestroy(zstream); zstream = nullptr; }
};
// Output in batch order: pinned buffers filled by device-to-host copies (from the lanes of any context), written by one thread.  A batch is
// written in one or more pieces, the last one flagged; one context produces the pieces of a batch, in order.  The pieces of a batch wait here
// until every earlier batch has been written.
// No deadlock: `open_min`, the oldest batch whose last piece is not in yet, may take any buffer; every other batch leaves one buffer free (or
// not yet allocated), so later batches hold at most nbuf - 1 buffers.  The batches before open_min are complete and get written, which frees
// their buffers, so the context of open_min always gets one.  A context finishes its batches in order, so with one context every get() is
// open_min's and the reserve never holds anything back.
struct KjWriter {
    struct Piece { char* b; size_t n; bool last; };
    FILE* out = nullptr; bool own = false; std::vector<char*> pool; size_t cap = 0; int nbuf = 3, made = 0; std::deque<char*> free_;
    std::map<uint64_t, std::deque<Piece>> ready; std::set<uint64_t> complete;       // pieces by batch; batches whose last piece is in, not yet written
    uint64_t next = 0, open_min = 0; size_t held_max = 0;                            // the batch being written; the most complete batches held back
    std::mutex mu; std::condition_variable cv; std::thread th; bool done = false, failed = false, cancelled = false; KjPinnedPool* pinned = nullptr;
    int open(const char* path, size_t cap_bytes, int nbuf_, KjPinnedPool* pp) {
        if (path && *path) { out = fopen(path, "w"); own = true; if (!out) { kj_err() = std::string("Could not open file ") + path + " for writing"; return KJ_ERR_IO; } } else { out = stdout; own = false; }
        cap = cap_bytes; nbuf = nbuf_; made = 0; pinned = pp; done = false; failed = false; cancelled = false; next = open_min = 0; held_max = 0;
        th = std::thread([this] {
            for (;;) {
                Piece job;
                {
                    std::unique_lock<std::mutex> lk(mu);
                    auto writable = [&] { const auto it = ready.find(next); return it != ready.end() && !it->second.empty(); };
                    cv.wait(lk, [&] { return done || writable(); }); if (!writable()) return;
                    std::deque<Piece>& q = ready[next]; job = q.front(); q.pop_front();
                    if (job.last) { ready.erase(next); complete.erase(next); next++; }
                }
                if (job.n && fwrite(job.b, 1, job.n, out) != job.n) failed = true;
                { std::lock_guard<std::mutex> lk(mu); if (job.b) free_.push_back(job.b); } cv.notify_all();
            }
        });
        return KJ_OK;
    }
    char* get(uint64_t batch) {      // nullptr: out of pinned memory, or the call was cancelled
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return cancelled || (int)free_.size() + (nbuf - made) > (batch == open_min ? 0 : 1); });
        if (cancelled) return nullptr;
        if (!free_.empty()) { char* b = free_.front(); free_.pop_front(); return b; }
        made++; lk.unlock(); char* b = pinned->get(cap); lk.lock();
        if (b) pool.push_back(b); else made--;
        return b;
    }
    // b = nullptr, n = 0: a piece without bytes (the end of a batch)
    void put(uint64_t batch, char* b, size_t n, bool last) {
        {
            std::lock_guard<std::mutex> lk(mu);
            ready[batch].push_back({b, n, last});
            if (last) {
                complete.insert(batch); held_max = std::max(held_max, complete.size() - complete.count(next));
                while (complete.count(open_min)) open_min++;
            }
        }
        cv.notify_all();
    }
    void cancel() { { std::lock_guard<std::mutex> lk(mu); cancelled = true; } cv.notify_all(); }      // after an error: no get() waits any more
    int close() {
        { std::lock_guard<std::mutex> lk(mu); done = true; } cv.notify_all();
        if (th.joinable()) th.join();
        if (out) { fflush(out); if (own) fclose(out); } out = nullptr;
        for (char* b : pool) pinned->put(b, cap); pool.clear(); ready.clear(); complete.clear(); free_.clear();
        if (failed) { kj_err() = "write error on the output file"; return KJ_ERR_IO; }
        return KJ_OK;
    }
};

// One parsed batch on its way from the parser thread to a classifying thread
struct KjBatch { KjBatchSide s[2]; uint64_t n = 0; unsigned int maxlen[2] = {0, 0}; bool last = false; float boost = 1.f; uint64_t seq = 0; };   // seq: 0, 1, ... in file order
// One of the two classification lanes of a context's classifying thread: while the kernel of batch k runs on one lane, batch k+1 is launched on the other
// (its CTAs fill the SMs as the first kernel's CTAs retire), and batch k-1 is formatted and written
// (formats with fragment strings: rows [b0, b0 + sub) of the batch are classified per launch, then formatted, then the next rows are launched)
// A lane of the parser's context classifies the parser's batch slot in place (batch = the slot); a lane of another context classifies its own
// copy of the batch (batch = -1).
struct KjLane {
    KjDevBuf tax, best, ids, nids, acc, nacc, frag, fraglen, gate, len, out, scan_tmp, totals; int batch = -1; bool busy = false;
    uint64_t b0 = 0, sub = 0; uint32_t stride = 0;        // the launch in flight: its first row, rows per launch, fragment-string bytes per read
    KjBatch* B = nullptr; KjBatch copy;                   // the batch being classified; the copy of it (contexts other than the parser's)
};
// Fragment strings of one launch, per lane: 512 MB hold the strings of ~300 k PE150 reads (1,728 bytes each), so a full batch of short reads
// takes one or two launches, each long enough to fill the persistent grid; the two lanes' 1 GB stays well inside the 4 GB of HBM that a tiered
// context keeps free for classification (KJ_TIER_HEADROOM), next to the batch buffers.  A batch of long reads (about 11 MB per 1 Mb read) gets
// launches of fewer reads, and the long-read kernels size their scratch from the HBM that is left.
#define KJ_FRAG_BUDGET (512ull << 20)
#define KJ_FILE_SLOTS 4
// Everything kj_classify_files needs besides the context; kept in the context between calls (device buffers and pinned memory are reused).
// In kj_classify_files_multi, the state of ctxs[0] holds the readers, the parser, its batch slots and the writer; that of every other context
// only its lanes and its second pending-count vector.
struct KjFilesState {
    KjParsed side[2]; KjFileReader rd[2]; KjWriter wr; int nfiles = 1; bool rd_open[2] = {false, false}, wr_open = false;
    KjBatch slot[KJ_FILE_SLOTS]; KjLane lane[2]; KjPinnedPool pinned; cudaStream_t sp = nullptr; KjDevBuf pstat, pending2;
    // parser thread -> classifying threads: filled slots in file order; a slot comes back (free_slot) when its batch has been classified and
    // written from it, or copied to another context
    std::mutex mu; std::condition_variable cv; std::deque<int> filled, free_slot; bool abort = false; std::thread parser;
    std::string fn[2], perr; int prc = KJ_OK;                 // input names; the parser thread's error
    uint64_t dev_inflated = 0;                                // bytes of text the inflate kernel produced in the last call
    uint64_t parse_launches = 0; double tm[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; uint64_t nbatches = 0;
    void reset_slots() { free_slot.clear(); for (int k = 0; k < KJ_FILE_SLOTS; k++) free_slot.push_back(k); }
    void end_call() {      // threads, files and in-flight copies of one call
        { std::lock_guard<std::mutex> lk(mu); abort = true; } cv.notify_all();
        for (int f = 0; f < 2; f++) if (rd_open[f]) rd[f].halt();      // a parser waiting for a stream's next chunk returns too
        if (parser.joinable()) parser.join();
        for (int f = 0; f < 2; f++) {
            if (rd_open[f]) rd[f].close(); rd_open[f] = false;
            KjParsed& P = side[f]; P.cur = 0; P.nbytes = 0; P.fastq = -1; P.n_lines = P.n_rec = P.consumed = 0; P.eof = false;
        }
        if (wr_open) wr.close(); wr_open = false;
        filled.clear(); reset_slots(); abort = false; lane[0].busy = lane[1].busy = false;
    }
    void release() {       // with the context; the device buffers go with their owners
        for (int f = 0; f < 2; f++) rd[f].release();
        if (sp) cudaStreamDestroy(sp); sp = nullptr;
        pinned.release();
    }
};
static void kj_files_state_free(KjFilesState* S) { if (!S) return; S->end_call(); S->release(); delete S; }

// Parser thread: staged file chunks -> device text -> packed reads, names and offsets of the complete records, one KjBatch per round.
// Stage 1 of the pipeline: while the caller's thread classifies and formats earlier batches on its streams, this thread assembles and parses the
// next ones on another; the carry (the incomplete record at the end of a batch) only depends on the parse.  A batch is `target` bytes of text
// per file: one I/O chunk at first (the pipeline starts after the first 16 MB), doubling up to batch_max (fewer, longer classify launches).
static int kj_parse_chunks(int device, int sm_count, KjFilesState& S, size_t chunk, size_t batch_max, bool paired) {
    CK(cudaSetDevice(device));
    const std::string* fn = S.fn;
    cudaStream_t st = S.sp; int rc; auto t = std::chrono::steady_clock::now();
    uint32_t* d_stat = S.pstat.as<uint32_t>();       // [0,1] longest read of each side, [2] error bits of the parse kernels
    size_t target = chunk; std::vector<int> used[2];
    for (;;) {
        int si;
        { std::unique_lock<std::mutex> lk(S.mu); S.cv.wait(lk, [&] { return S.abort || !S.free_slot.empty(); }); if (S.abort) return KJ_OK; si = S.free_slot.front(); S.free_slot.pop_front(); }
        KjBatch& B = S.slot[si]; B.seq = S.nbatches++;
        S.tm[0] += kj_ms_since(t);
        B.boost = target < batch_max ? (float)batch_max / (float)target : 1.f;      // buffers of the first, small batches are allocated for the final batch size
        // 1. top up both sides to `target` bytes: the carry is already at the front of the device text, staged chunks are appended behind it
        for (int f = 0; f < S.nfiles; f++) {
            KjParsed& P = S.side[f];
            while (!P.eof && P.nbytes < target) {
                KjStaged ck = S.rd[f].next();
                if (!ck.error.empty()) { kj_err() = ck.error; return KJ_ERR_IO; }
                if ((P.nbytes + ck.n + 1) > P.text[P.cur].cap) {           // grow: move what is there into the larger buffer
                    KjDevBuf nb; if ((rc = kj_need(nb, P.nbytes + ck.n + std::max(target, batch_max) + chunk + 1))) return rc;
                    if (P.nbytes) CK(cudaMemcpyAsync(nb.p, P.text[P.cur].p, P.nbytes, cudaMemcpyDeviceToDevice, st));
                    CK(cudaStreamSynchronize(st)); P.text[P.cur] = std::move(nb);
                }
                CK(cudaStreamWaitEvent(st, ck.ev, 0));
                if (ck.n) CK(cudaMemcpyAsync(P.text[P.cur].as<char>() + P.nbytes, S.rd[f].ring[ck.slot].p, ck.n, cudaMemcpyDeviceToDevice, st));
                used[f].push_back(ck.slot);
                if ((int)used[f].size() + 2 >= (int)S.rd[f].ring.size()) {   // never hold the whole ring: the reader needs free staging buffers to get ahead
                    CK(cudaStreamSynchronize(st)); for (int sl : used[f]) S.rd[f].release_slot(sl); used[f].clear();
                }
                P.nbytes += ck.n;
                if (ck.eof) {
                    P.eof = true;
                    if (P.nbytes && ck.last != '\n') { CK(cudaMemsetAsync(P.text[P.cur].as<char>() + P.nbytes, '\n', 1, st)); P.nbytes += 1; }      // the last line of a file may lack its newline
                }
            }
        }
        S.tm[1] += kj_ms_since(t);
        // 2. parse; a FASTQ batch with an empty line where a header was expected (flag 64) is parsed again with the record phases from the automaton scan
        uint64_t n = 0; bool all_eof = false; uint64_t pos[2] = {0, 0}; uint32_t hstat[4] = {0, 0, 0, 0};
        for (int pass = 0; pass < 2; pass++) {
            CK(cudaMemsetAsync(d_stat, 0, 16, st));
            if ((rc = kj_parse_sides(sm_count, S.side, B.s, S.nfiles, fn, st, d_stat + 2, &S.parse_launches, pass == 1, B.boost))) return rc;
            // (kj_parse_sides synchronises the stream: the staging buffers appended above are free again)
            for (int f = 0; f < S.nfiles; f++) { for (int sl : used[f]) S.rd[f].release_slot(sl); used[f].clear(); }
            n = S.side[0].n_rec; if (paired) n = std::min(n, S.side[1].n_rec);
            all_eof = S.side[0].eof && (!paired || S.side[1].eof);
            if (n >= (1ull << 31)) { kj_err() = "kj_classify_files: batch with too many records"; return KJ_ERR_UNSUPPORTED; }
            if (n) {
                if (paired) kj_names_equal<<<sm_count * 4, 256, 0, st>>>(B.s[0].names.as<char>(), B.s[0].name_off.as<uint32_t>(), B.s[1].names.as<char>(), B.s[1].name_off.as<uint32_t>(), n, d_stat + 2);
                kj_maxlen_kernel<<<256, 256, 0, st>>>(B.s[0].off.as<uint64_t>(), n, d_stat);
                if (paired) kj_maxlen_kernel<<<256, 256, 0, st>>>(B.s[1].off.as<uint64_t>(), n, d_stat + 1);
                S.parse_launches += paired ? 3 : 1;
            }
            // where the first n records end: the rest is carried over
            for (int f = 0; f < S.nfiles; f++) if (S.side[f].n_lines) CK(cudaMemcpyAsync(&pos[f], S.side[f].rec_pos.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(hstat, d_stat, 16, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));       // the batch is complete in device memory from here on
            if (!(hstat[2] & 64u)) break;
        }
        for (int f = 0; f < S.nfiles; f++) { for (int sl : used[f]) S.rd[f].release_slot(sl); used[f].clear(); }      // (a side without bytes does not synchronise in kj_parse_side)
        if (paired && all_eof && S.side[0].n_rec > S.side[1].n_rec) { kj_err() = "File " + fn[0] + " contains more reads then file " + fn[1]; return KJ_ERR_IO; }   // kaiju.cpp:337-340
        if (hstat[2] & 16u) { kj_err() = "malformed FASTQ record (a header line does not start with '@') in the input"; return KJ_ERR_IO; }
        if (n && (hstat[2] & 32u)) { kj_err() = "Read names are not identical between the two input files. Probably reads are not in the same order in both files."; return KJ_ERR_IO; }
        B.n = n; B.maxlen[0] = hstat[0]; B.maxlen[1] = hstat[1];
        // 3. carry the unconsumed tail to the front of the other text buffer
        if (target < batch_max) target = std::min(batch_max, target * 2);
        for (int f = 0; f < S.nfiles; f++) {
            KjParsed& P = S.side[f]; const uint64_t consumed = P.skip_all ? P.nbytes : (P.n_lines ? pos[f] : 0);
            const uint64_t tail = P.nbytes - consumed; const int other = P.cur ^ 1;
            if ((rc = kj_need(P.text[other], tail + std::max(target, batch_max) + chunk + 1))) return rc;
            if (tail) CK(cudaMemcpyAsync(P.text[other].p, P.text[P.cur].as<char>() + consumed, tail, cudaMemcpyDeviceToDevice, st));
            P.cur = other; P.nbytes = tail;
        }
        // a side whose carry alone reaches the target cannot make progress by itself (a record longer than the batch, or the other file lagging):
        // let the next round read more
        for (int f = 0; f < S.nfiles; f++) if (!S.side[f].eof && S.side[f].nbytes >= target) target = S.side[f].nbytes + chunk;
        bool last = false;
        if (all_eof) {
            if (paired && S.side[1].n_rec > n) fprintf(stderr, "Warning: File %s has more reads then file %s\n", fn[1].c_str(), fn[0].c_str());        // kaiju.cpp:400-404
            last = true;
        } else if (paired && S.side[0].eof && S.side[0].nbytes == 0) {
            // file 1 is exhausted (end of file, nothing carried over): the reference's loop ends here, whatever file 2 still holds (kaiju.cpp:288, 396-404)
            if (S.side[1].nbytes > 0 || !S.side[1].eof) fprintf(stderr, "Warning: File %s has more reads then file %s\n", fn[1].c_str(), fn[0].c_str());
            last = true;
        }
        B.last = last;
        S.tm[3] += kj_ms_since(t);
        { std::lock_guard<std::mutex> lk(S.mu); S.filled.push_back(si); } S.cv.notify_all();
        if (last) return KJ_OK;
    }
}

// One kj_classify_files_multi call (kj_classify_files: one context): what its classifying threads share.  P is the state of ctxs[0]: the
// readers, the parser's batch slots, the queue of parsed batches and the writer.
struct KjFilesRun {
    kj_ctx** ctxs = nullptr; int n_ctx = 1; KjFilesState* P = nullptr;
    int fmt = 0; bool paired = false, want_ids = false, want_acc = false, want_frag = false, want_gate = false;
    uint64_t frag_budget = KJ_FRAG_BUDGET; uint32_t frag_stride_fix = 0; size_t out_cap = 16u << 20; int hold_ms = 0;
    bool ended = false;                                   // the last batch has been taken (under P->mu)
    std::mutex mu; int rc = KJ_OK; std::string msg;       // the first error of any thread
    std::vector<uint64_t> n_reads, n_batches;             // per context
    // the first error wins; every thread then stops: the parser and the waiting classifiers through P->abort, a wait for an output buffer
    // through the writer's cancel
    void fail(int i, int r, const std::string& m) {
        {
            std::lock_guard<std::mutex> lk(mu); if (rc != KJ_OK) return;
            rc = r; msg = n_ctx > 1 ? "device " + std::to_string(ctxs[i]->device) + ": " + m : m;
        }
        { std::lock_guard<std::mutex> lk(P->mu); P->abort = true; } P->cv.notify_all();
        P->wr.cancel();
    }
};

// The classifying thread of context i: two classification lanes on the context's own streams.  Each batch goes to whichever context next has a
// free lane.  ctxs[0] classifies from the parser's slot in place; any other context copies the slot's four buffers per file into its lane's own
// (cudaMemcpyPeerAsync: over NVLink or PCIe between devices, staged through the host where there is no peer access) and gives the slot back.
static int kj_files_classify(KjFilesRun& R, int i) {
    kj_ctx* c = R.ctxs[i]; KjFilesState& S = *c->files; KjFilesState& P = *R.P;
    const int fmt = R.fmt; const bool paired = R.paired, want_ids = R.want_ids, want_acc = R.want_acc, want_frag = R.want_frag, want_gate = R.want_gate;
    const size_t out_cap = R.out_cap; int rc;
    CK(cudaSetDevice(c->device));
    if ((rc = kj_need(S.pending2, (size_t)c->n_counts * 8 + 64))) return rc;
    unsigned long long* pend[2] = {c->counts_pending.as<unsigned long long>(), S.pending2.as<unsigned long long>()};
    for (int l = 0; l < 2; l++) {
        if ((rc = kj_need(S.lane[l].totals, 64))) return rc;
        cudaStream_t st = c->slot[l].stream;
        CK(cudaMemsetAsync(S.lane[l].totals.p, 0, 64, st)); CK(cudaMemsetAsync(pend[l], 0, (size_t)c->n_counts * 8, st)); CK(cudaStreamSynchronize(st));
        S.lane[l].busy = false; S.lane[l].batch = -1; S.lane[l].B = nullptr;
    }
    uint64_t& n_reads = R.n_reads[(size_t)i];
    auto t = std::chrono::steady_clock::now();
    auto give_back = [&](int si) { { std::lock_guard<std::mutex> lk(P.mu); P.free_slot.push_back(si); } P.cv.notify_all(); };   // the parser may overwrite the slot now
    // launch the classification of rows [b0, b0 + sub) of lane l's batch (outputs at their rows; the fragment strings at the start of the lane's buffer)
    auto launch_sub = [&](int l) -> int {
        KjLane& Ln = S.lane[l]; KjBatch& B = *Ln.B; const uint64_t b0 = Ln.b0, m = std::min(B.n, b0 + Ln.sub) - b0;
        KjOut o; o.tax = Ln.tax.as<uint64_t>() + b0; o.best = Ln.best.as<uint32_t>() + b0; o.counts = pend[l];
        if (want_ids) { o.ids = Ln.ids.as<uint64_t>() + b0 * KJ_MAX_IDS; o.nids = Ln.nids.as<uint8_t>() + b0; }
        if (want_acc) { o.acc = Ln.acc.as<uint32_t>() + b0 * KJ_MAX_MATCH_ACC; o.nacc = Ln.nacc.as<uint8_t>() + b0; }
        if (want_frag) { o.frag = Ln.frag.as<char>(); o.frag_stride = Ln.stride; o.fraglen = Ln.fraglen.as<uint32_t>() + b0; }
        return launch(c, l, B.s[0].seq.as<uint8_t>(), B.s[0].off.as<uint64_t>() + b0, paired ? B.s[1].seq.as<uint8_t>() : nullptr, paired ? B.s[1].off.as<uint64_t>() + b0 : nullptr, 0, 0, m,
                      B.maxlen[0], B.maxlen[1], o, c->slot[l].stream, false);
    };
    auto take = [&](int l, int si) -> int {           // lane l's batch: the parser's slot si, or (another context) a copy of it
        KjLane& Ln = S.lane[l]; KjBatch& Bp = P.slot[si];
        if (i == 0) { Ln.batch = si; Ln.B = &Bp; return KJ_OK; }
        KjBatch& B = Ln.copy; int r;
        B.n = Bp.n; B.maxlen[0] = Bp.maxlen[0]; B.maxlen[1] = Bp.maxlen[1]; B.last = Bp.last; B.boost = Bp.boost; B.seq = Bp.seq;
        cudaStream_t st = c->slot[l].stream;
        for (int f = 0; B.n && f < (paired ? 2 : 1); f++) {
            const KjBatchSide& from = Bp.s[f]; KjBatchSide& to = B.s[f];
            KjDevBuf* dst[4] = {&to.seq, &to.off, &to.names, &to.name_off}; const KjDevBuf* src[4] = {&from.seq, &from.off, &from.names, &from.name_off};
            for (int b = 0; b < 4; b++) {
                to.bytes[b] = from.bytes[b];
                if ((r = kj_need(*dst[b], from.bytes[b], B.boost))) return r;
                CK(cudaMemcpyPeerAsync(dst[b]->p, c->device, src[b]->p, R.ctxs[0]->device, from.bytes[b], st));
            }
        }
        CK(cudaStreamSynchronize(st));
        give_back(si);
        Ln.batch = -1; Ln.B = &B; return KJ_OK;
    };
    auto start = [&](int l, int si) -> int {          // launch the classification of batch si on lane l (its first rows, with fragment strings)
        int r; if ((r = take(l, si))) return r;
        KjLane& Ln = S.lane[l]; KjBatch& B = *Ln.B; const uint64_t n = B.n;
        Ln.busy = true; Ln.b0 = 0; Ln.sub = n;
        if (!n) return KJ_OK;
        if ((r = kj_need(Ln.tax, n * 8, B.boost)) || (r = kj_need(Ln.best, n * 4, B.boost)) || (r = kj_need(Ln.len, (n + 2) * 4, B.boost))) return r;
        if (want_ids && ((r = kj_need(Ln.ids, n * KJ_MAX_IDS * 8, B.boost)) || (r = kj_need(Ln.nids, n, B.boost)))) return r;
        if (want_acc && ((r = kj_need(Ln.acc, n * KJ_MAX_MATCH_ACC * 4, B.boost)) || (r = kj_need(Ln.nacc, n, B.boost)))) return r;
        if (want_frag) {      // the stride kj_classify_verbose2's callers use: 32 x (residues of the longest mate + 2) + 64
            const uint32_t mx = std::max(B.maxlen[0], B.maxlen[1]), res = c->params.input_is_protein ? mx : mx / 3u;
            Ln.stride = R.frag_stride_fix ? R.frag_stride_fix : 32u * (res + 2u) + 64u;
            Ln.sub = std::min<uint64_t>(n, std::max<uint64_t>(1, R.frag_budget / Ln.stride));
            if ((r = kj_need(Ln.frag, (size_t)Ln.sub * Ln.stride)) || (r = kj_need(Ln.fraglen, n * 4, B.boost))) return r;
        }
        if (want_gate) {
            if ((r = kj_need(Ln.gate, n, B.boost))) return r;
            kj_name_gate<<<c->sm_count * 8, 256, 0, c->slot[l].stream>>>(B.s[0].seq.as<char>(), B.s[0].off.as<uint64_t>(), paired ? B.s[1].off.as<uint64_t>() : nullptr, n,
                                                                         c->params.min_fragment_length, c->params.input_is_protein, c->params.mode == 1, c->params.min_score, Ln.gate.as<uint8_t>());
            CK(cudaGetLastError()); c->launches++;
        }
        return launch_sub(l);
    };
    auto finish = [&](int l) -> int {                 // per launch of lane l's batch: wait, check, count, format, write, launch the next rows; the slot goes back to the parser
        KjLane& Ln = S.lane[l]; KjBatch& B = *Ln.B; const uint64_t n = B.n, seq = B.seq; cudaStream_t st = c->slot[l].stream; int r;
        if (i == 0 && R.hold_ms) std::this_thread::sleep_for(std::chrono::milliseconds(R.hold_ms));      // test hook KJ_FILES_HOLD_MS
        while (n) {
            CK(cudaStreamSynchronize(st));
            uint32_t e = 0; CK(cudaMemcpy(&e, c->err.p, sizeof e, cudaMemcpyDeviceToHost));
            if (e) {
                // the error word is shared by the two lanes: let the other kernel finish, then repeat what was in flight, one launch at a time
                // (only a full Greedy variant ring is repaired by a repeat: the ring grows)
                const int o = l ^ 1; const bool other = S.lane[o].busy && S.lane[o].B->n > 0;
                if (other) CK(cudaStreamSynchronize(c->slot[o].stream));
                const uint32_t boost = c->variant_boost;
                r = check_err_flag(c);
                for (int k = 0; k < 2; k++) CK(cudaMemset(pend[k], 0, (size_t)c->n_counts * 8));      // failed launches do not count
                if (!(r == KJ_ERR_OVERFLOW && c->variant_boost != boost)) return r ? r : KJ_ERR_CUDA;
                for (int k = 0; k < 2; k++) {
                    const int ll = k == 0 ? l : o; if (k == 1 && !other) break;
                    for (;;) {
                        if ((r = launch_sub(ll))) return r;
                        CK(cudaStreamSynchronize(c->slot[ll].stream));
                        const uint32_t b2 = c->variant_boost; r = check_err_flag(c);
                        if (r) CK(cudaMemset(pend[ll], 0, (size_t)c->n_counts * 8));
                        if (r == KJ_ERR_OVERFLOW && c->variant_boost != b2) continue;
                        if (r) return r;
                        break;
                    }
                }
            }
            S.tm[6] += kj_ms_since(t);
            const uint64_t b0 = Ln.b0, m = std::min(n, b0 + Ln.sub) - b0;
            unsigned long long* d_nclass = (unsigned long long*)((char*)Ln.totals.p + 16);
            kj_count_commit<<<c->sm_count, 256, 0, st>>>(c->counts.as<unsigned long long>(), pend[l], c->n_counts); c->launches++;     // these rows succeeded: they join the per-taxon counts
            KjFmtIn in{}; in.fmt = fmt; in.tax = Ln.tax.as<uint64_t>() + b0; in.best = Ln.best.as<uint32_t>() + b0;
            if (want_ids) { in.ids = Ln.ids.as<uint64_t>() + b0 * KJ_MAX_IDS; in.nids = Ln.nids.as<uint8_t>() + b0; }
            if (want_acc) { in.acc = Ln.acc.as<uint32_t>() + b0 * KJ_MAX_MATCH_ACC; in.nacc = Ln.nacc.as<uint8_t>() + b0; }
            if (want_frag) { in.frag = Ln.frag.as<char>(); in.frag_stride = Ln.stride; in.fraglen = Ln.fraglen.as<uint32_t>() + b0; }
            if (want_gate) in.gate = Ln.gate.as<uint8_t>() + b0;
            in.names = B.s[0].names.as<char>(); in.name_off = B.s[0].name_off.as<uint32_t>() + b0;
            in.acc_str = c->out_str[KJ_STR_ACCESSION].as<char>(); in.acc_off = c->out_off[KJ_STR_ACCESSION].as<uint64_t>(); in.n_acc = c->out_n[KJ_STR_ACCESSION];
            in.lab_str = c->out_str[KJ_STR_TAXON].as<char>(); in.lab_off = c->out_off[KJ_STR_TAXON].as<uint64_t>(); in.n_lab = c->out_n[KJ_STR_TAXON];
            in.tax_id = c->tax_id.as<uint64_t>(); in.n_present = c->n_present; in.n_tax = c->n_counts - 1u;
            kj_fmt_len<<<c->sm_count * 4, 256, 0, st>>>(in, m, Ln.len.as<uint32_t>(), d_nclass);
            if ((r = kj_scan_u32(Ln.len.as<uint32_t>(), m + 1, Ln.scan_tmp, B.boost, (uint32_t*)Ln.totals.p, st))) return r;
            uint32_t out_bytes = 0; CK(cudaMemcpyAsync(&out_bytes, Ln.totals.p, 4, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
            if ((r = kj_need(Ln.out, out_bytes + 64, B.boost))) return r;
            kj_fmt_write<<<c->sm_count * 4, 256, 0, st>>>(in, m, Ln.len.as<uint32_t>(), Ln.out.as<char>());
            CK(cudaGetLastError()); c->launches += 6;
            for (size_t o = 0; o < out_bytes; o += out_cap) {
                const size_t q = std::min<size_t>(out_cap, out_bytes - o); char* hb = P.wr.get(seq);
                if (!hb) { kj_err() = "cudaMallocHost failed"; return KJ_ERR_NOMEM; }
                CK(cudaMemcpyAsync(hb, Ln.out.as<char>() + o, q, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
                P.wr.put(seq, hb, q, false);
            }
            CK(cudaStreamSynchronize(st));
            n_reads += m; S.tm[7] += kj_ms_since(t);
            Ln.b0 += m;
            if (Ln.b0 >= n) break;
            if ((r = launch_sub(l))) return r;        // the next rows: the fragment-string buffer has been formatted
        }
        Ln.busy = false; R.n_batches[(size_t)i]++;
        P.wr.put(seq, nullptr, 0, true);                 // the batch is complete
        if (Ln.batch >= 0) give_back(Ln.batch);
        Ln.batch = -1;
        return KJ_OK;
    };
    // batch k of this thread goes to lane k & 1; that lane still holds batch k - 2, the older one, when both lanes are busy
    uint64_t k = 0;
    for (;; k++) {
        const int l = (int)(k & 1);
        if (S.lane[l].busy && (rc = finish(l))) return rc;
        int si = -2;
        for (;;) {   // the next parsed batch; while none is there, complete the running lane instead of waiting
            bool took_last = false;
            {
                std::unique_lock<std::mutex> lk(P.mu);
                if (P.filled.empty() && !R.ended && !P.abort && S.lane[l ^ 1].busy) si = -3;
                else {
                    P.cv.wait(lk, [&] { return P.abort || R.ended || !P.filled.empty(); });
                    if (P.abort) return KJ_OK;                  // another thread failed (its error is the call's)
                    if (P.filled.empty()) si = -4;              // every batch has been taken
                    else { si = P.filled.front(); P.filled.pop_front(); if (si >= 0 && P.slot[si].last) R.ended = took_last = true; }
                }
            }
            if (took_last) P.cv.notify_all();
            if (si != -3) break;
            if ((rc = finish(l ^ 1))) return rc;
        }
        if (si == -1) { R.fail(0, P.prc, P.perr); return KJ_OK; }       // the parser's error (it runs on ctxs[0]'s device)
        if (si == -4) break;
        S.tm[5] += kj_ms_since(t);
        if ((rc = start(l, si))) return rc;
    }
    for (int q = 0; q < 2; q++) { const int l = (int)((k + q) & 1); if (S.lane[l].busy && (rc = finish(l))) return rc; }       // older lane first
    return KJ_OK;
}

static int kj_classify_files_impl(KjFilesRun& R, const char* in1, const char* in2, const char* out_path, uint64_t* n_reads_out, uint64_t* n_class_out) {
    kj_ctx* c = R.ctxs[0]; KjFilesState& S = *R.P;
    // developer hook KJ_FILES_TRACE: host time of each stage of the parser and of ctxs[0]'s thread (ms, summed over the batches; waits included)
    const bool ftrace = getenv("KJ_FILES_TRACE") != nullptr;
    size_t chunk = 16u << 20, batch_max = 128u << 20;
    if (const char* v = getenv("KJ_INGEST_CHUNK")) { long x = atol(v); if (x >= 256 && x <= (1l << 30)) { chunk = (size_t)x; batch_max = chunk; } }       // test hook: many small batches
    if (const char* v = getenv("KJ_INGEST_BATCH")) { long x = atol(v); if (x >= 256 && x <= (1l << 30)) batch_max = std::max((size_t)x, chunk); }
    const bool paired = in2 && *in2; S.nfiles = paired ? 2 : 1; R.paired = paired;
    for (int f = 0; f < 2; f++) S.side[f].whole_names = c->params.name_mode && c->params.input_is_protein;
    // what the format needs from the classify kernels: id sets (1-4), accession sets (2), fragment strings (2, 4), the front-end gate (3, 4)
    const int fmt = R.fmt;
    R.want_ids = fmt >= KJ_OUT_KAIJU_IDS; R.want_acc = fmt == KJ_OUT_KAIJU_V; R.want_frag = fmt == KJ_OUT_KAIJU_V || fmt == KJ_OUT_NAMES_V; R.want_gate = fmt >= KJ_OUT_NAMES;
    if (const char* v = getenv("KJ_FRAG_BUDGET")) { const long long x = atoll(v); if (x >= 1) R.frag_budget = (uint64_t)x; }      // test hook: several launches per batch
    if (const char* v = getenv("KJ_FRAG_STRIDE")) { const long long x = atoll(v); if (x >= 16 && x < (1ll << 31)) R.frag_stride_fix = (uint32_t)x; }   // test hook: a stride too small
    if (const char* v = getenv("KJ_FILES_HOLD_MS")) { const long x = atol(v); if (x >= 1 && x <= 60000) R.hold_ms = (int)x; }   // test hook: ctxs[0] formats late, batches finish out of order
    S.fn[0] = in1; S.fn[1] = paired ? in2 : ""; S.perr.clear(); S.prc = KJ_OK;
    const std::string* fn = S.fn;
    int rc;
    if (!S.sp) { int lo = 0, hi = 0; CK(cudaDeviceGetStreamPriorityRange(&lo, &hi)); CK(cudaStreamCreateWithPriority(&S.sp, cudaStreamNonBlocking, hi)); }    // the short parse kernels go first when SM slots free up
    const int depth = (int)std::min<size_t>(64, batch_max / chunk + 4);
    for (int f = 0; f < 2; f++) S.rd[f].lead_error.clear();
    S.rd[0].follower = paired ? &S.rd[1] : nullptr;
    for (int f = 0; f < S.nfiles; f++) { if ((rc = S.rd[f].open(fn[f], chunk, depth, c->device, &S.pinned))) return rc; S.rd_open[f] = true; }
    // output buffers: two per lane of every context, one more for the oldest batch (KjWriter)
    if ((rc = S.wr.open(out_path, R.out_cap, 1 + 2 * R.n_ctx, &S.pinned))) return rc; S.wr_open = true;
    if ((rc = kj_need(S.pstat, 64))) return rc;
    S.parse_launches = 0; S.nbatches = 0; for (double& x : S.tm) x = 0;
    S.reset_slots(); R.n_reads.assign((size_t)R.n_ctx, 0); R.n_batches.assign((size_t)R.n_ctx, 0);
    {   // the thread only touches S (which outlives this call) and its own copies
        KjFilesState* Sp = &S; const int dev = c->device, sms = c->sm_count;
        S.parser = std::thread([Sp, dev, sms, chunk, batch_max, paired] {
            const int r = kj_parse_chunks(dev, sms, *Sp, chunk, batch_max, paired);
            if (r) { std::lock_guard<std::mutex> lk(Sp->mu); Sp->prc = r; Sp->perr = kj_err(); Sp->filled.push_back(-1); }
            Sp->cv.notify_all();
        });
    }
    {   // one classifying thread per context; ctxs[0]'s is the calling thread
        std::vector<std::thread> th;
        for (int i = 1; i < R.n_ctx; i++) th.emplace_back([&R, i] { const int r = kj_files_classify(R, i); if (r) R.fail(i, r, kj_err()); });
        const int r = kj_files_classify(R, 0); if (r) R.fail(0, r, kj_err());
        for (auto& x : th) x.join();
    }
    CK(cudaSetDevice(c->device));
    if (R.rc) { kj_err() = R.msg; return R.rc; }
    S.parser.join();
    c->launches += S.parse_launches;
    unsigned long long n_class = 0; uint64_t n_reads = 0;
    for (int i = 0; i < R.n_ctx; i++) {
        kj_ctx* x = R.ctxs[i]; CK(cudaSetDevice(x->device)); n_reads += R.n_reads[(size_t)i];
        for (int l = 0; l < 2; l++) { unsigned long long v = 0; CK(cudaMemcpy(&v, (char*)x->files->lane[l].totals.p + 16, 8, cudaMemcpyDeviceToHost)); n_class += v; }
    }
    CK(cudaSetDevice(c->device));
    if (ftrace) fprintf(stderr, "KJ_FILES_TRACE batches %llu  parser: slot-wait %.1f  chunk-wait+append %.1f  parse+carry %.1f | classifier: batch-wait %.1f  classify-wait %.1f  format+d2h %.1f ms\n",
                        (unsigned long long)S.nbatches, S.tm[0], S.tm[1], S.tm[3], S.tm[5], S.tm[6], S.tm[7]);
    if (ftrace) for (int f = 0; f < S.nfiles; f++) if (S.rd[f].bgzf)
        fprintf(stderr, "KJ_FILES_TRACE reader %d (BGZF): read %.1f  inflate-wait %.1f ms  inflated %llu bytes on the device\n", f, S.rd[f].tm_read, S.rd[f].tm_inflate, (unsigned long long)S.rd[f].inflated);
    if (ftrace) {
        std::string per; for (int i = 0; i < R.n_ctx; i++) per += (i ? "," : "") + std::to_string(R.n_batches[(size_t)i]);
        size_t held; { std::lock_guard<std::mutex> lk(S.wr.mu); held = S.wr.held_max; }
        fprintf(stderr, "KJ_FILES_TRACE contexts %d  batches per context %s  writer held back at most %zu complete batches\n", R.n_ctx, per.c_str(), held);
    }
    if (n_reads_out) *n_reads_out = n_reads; if (n_class_out) *n_class_out = n_class;
    return KJ_OK;
}

// What format needs from context c (the messages of kj_classify_files)
static int kj_files_check(const kj_ctx* c, const char* in2, int format) {
    if (format < KJ_OUT_KAIJU || format > KJ_OUT_NAMES_V) { kj_err() = "kj_classify_files: unknown output format " + std::to_string(format); return KJ_ERR_ARG; }
    if (format >= KJ_OUT_NAMES && !c->params.name_mode) { kj_err() = "kj_classify_files: the name formats (KJ_OUT_NAMES, KJ_OUT_NAMES_V) need a context in name_mode"; return KJ_ERR_ARG; }
    if (format >= KJ_OUT_NAMES && !c->out_have[KJ_STR_TAXON]) { kj_err() = "kj_classify_files: the name formats need the KJ_STR_TAXON table (kj_set_output_strings)"; return KJ_ERR_ARG; }
    if (format == KJ_OUT_KAIJU_V && !c->dix.sa_acc) { kj_err() = "kj_classify_files: KJ_OUT_KAIJU_V needs a context created with kj_index_view.seq_accession"; return KJ_ERR_ARG; }
    if (format == KJ_OUT_KAIJU_V && !c->out_have[KJ_STR_ACCESSION]) { kj_err() = "kj_classify_files: KJ_OUT_KAIJU_V needs the KJ_STR_ACCESSION table (kj_set_output_strings)"; return KJ_ERR_ARG; }
    if (c->params.input_is_protein && in2 && *in2) { kj_err() = "Protein input only supports one input file."; return KJ_ERR_ARG; }
    return KJ_OK;
}

// The call on checked arguments: the threads of the pipeline run and are joined; afterwards no stream of any context has work in flight, and
// after an error every context's error word is clear.
static int kj_classify_files_run(kj_ctx** ctxs, int n_ctx, const char* in1, const char* in2, const char* out_path, int format, uint64_t* n_reads, uint64_t* n_classified) {
    for (int i = n_ctx - 1; i >= 0; i--) { CK(cudaSetDevice(ctxs[i]->device)); if (!ctxs[i]->files) ctxs[i]->files.reset(new KjFilesState()); }
    kj_ctx* c = ctxs[0]; KjFilesState* S = c->files.get();
    S->dev_inflated = 0;
    KjFilesRun R; R.ctxs = ctxs; R.n_ctx = n_ctx; R.P = S; R.fmt = format;
    int rc = kj_classify_files_impl(R, in1, in2, out_path, n_reads, n_classified);
    const std::string keep = kj_err();
    for (int f = 0; f < 2; f++) if (S->rd_open[f]) S->dev_inflated += S->rd[f].inflated;
    for (int i = n_ctx - 1; i >= 0; i--) { cudaSetDevice(ctxs[i]->device); cudaStreamSynchronize(ctxs[i]->slot[0].stream); cudaStreamSynchronize(ctxs[i]->slot[1].stream); }
    S->end_call();
    for (int i = 1; i < n_ctx; i++) ctxs[i]->files->end_call();
    if (rc) { for (int i = n_ctx - 1; i >= 0; i--) { cudaSetDevice(ctxs[i]->device); cudaMemset(ctxs[i]->err.p, 0, 4); } kj_err() = keep; }
    else if (S->wr.failed) { kj_err() = "write error on the output file"; rc = KJ_ERR_IO; }
    return rc;
}

extern "C" int kj_classify_files(kj_ctx* c, const char* in1, const char* in2, const char* out_path, int format, uint64_t* n_reads, uint64_t* n_classified) {
    if (!c || !in1 || !*in1) { kj_err() = "kj_classify_files: null argument"; return KJ_ERR_ARG; }
    int rc = kj_files_check(c, in2, format); if (rc) return rc;
    CK(cudaSetDevice(c->device));
    return kj_classify_files_run(&c, 1, in1, in2, out_path, format, n_reads, n_classified);
}

// One input through the contexts of several devices (or several contexts of one device): one reader set and parser on ctxs[0]'s device, each
// context classifies whole batches on its own thread, the output is written in input order -- byte for byte what kj_classify_files(ctxs[0])
// writes.
extern "C" int kj_classify_files_multi(kj_ctx** ctxs, int n_ctx, const char* in1, const char* in2, const char* out_path, int format, uint64_t* n_reads, uint64_t* n_classified) {
    if (!ctxs || n_ctx < 1 || n_ctx > KJ_MAX_GROUP || !in1 || !*in1) { kj_err() = "kj_classify_files_multi: null argument or n_ctx outside 1.." + std::to_string(KJ_MAX_GROUP); return KJ_ERR_ARG; }
    for (int i = 0; i < n_ctx; i++) {
        const kj_ctx* a = ctxs[i]; const kj_ctx* b = ctxs[0];
        if (!a) { kj_err() = "kj_classify_files_multi: null context"; return KJ_ERR_ARG; }
        for (int j = 0; j < i; j++) if (ctxs[j] == a) { kj_err() = "kj_classify_files_multi: context " + std::to_string(i) + " is listed twice"; return KJ_ERR_ARG; }
        const kj_params &p = a->params, &q = b->params;
        const bool same_params = p.mode == q.mode && p.min_fragment_length == q.min_fragment_length && p.mismatches == q.mismatches && p.min_score == q.min_score &&
                                 p.seed_length == q.seed_length && p.use_evalue == q.use_evalue && p.min_evalue == q.min_evalue && p.seg == q.seg &&
                                 p.input_is_protein == q.input_is_protein && p.name_mode == q.name_mode;
        if (!same_params) { kj_err() = "kj_classify_files_multi: context " + std::to_string(i) + " has other kj_params than context 0"; return KJ_ERR_ARG; }
        if (a->max_read_len != b->max_read_len) { kj_err() = "kj_classify_files_multi: context " + std::to_string(i) + " has another read-length limit (kj_set_max_read_len) than context 0"; return KJ_ERR_ARG; }
        if (a->H.bwtlen != b->H.bwtlen || a->H.nseq != b->H.nseq || a->n_counts != b->n_counts) {
            kj_err() = "kj_classify_files_multi: context " + std::to_string(i) + " holds another index than context 0 (BWT length, sequence count or taxa)"; return KJ_ERR_ARG; }
    }
    for (int i = 0; i < n_ctx; i++) { const int rc = kj_files_check(ctxs[i], in2, format); if (rc) return rc; }
    if (n_ctx == 1) return kj_classify_files(ctxs[0], in1, in2, out_path, format, n_reads, n_classified);
    CK(cudaSetDevice(ctxs[0]->device));
    return kj_classify_files_run(ctxs, n_ctx, in1, in2, out_path, format, n_reads, n_classified);
}

extern "C" uint64_t kj_files_device_inflated_bytes(const kj_ctx* c) { return c && c->files ? c->files->dev_inflated : 0; }

// test hook: a whole BGZF file in host memory through the header walk and the inflate kernel of the file pipeline
extern "C" int kj_debug_inflate_bgzf(kj_ctx* c, const uint8_t* file_bytes, uint64_t n, uint8_t* out, uint64_t out_cap, uint64_t* out_n, uint64_t* first_bad_offset) {
    if (!c || (!file_bytes && n) || !out_n || !first_bad_offset) { kj_err() = "kj_debug_inflate_bgzf: null argument"; return KJ_ERR_ARG; }
    CK(cudaSetDevice(c->device));
    *out_n = 0; *first_bad_offset = 0;
    std::vector<KjBgzfBlock> table; const KjBgzfWalk w = kj_bgzf_walk(file_bytes, (size_t)n, ~0ull, ~(size_t)0, 0, 0, table);
    if (w.stop != KJ_BGZF_END && w.stop != KJ_BGZF_GARBAGE) {
        *first_bad_offset = w.consumed; kj_err() = std::string(w.stop == KJ_BGZF_PARTIAL ? "truncated BGZF block" : w.stop == KJ_BGZF_FOREIGN ? "not a BGZF block" : "corrupt BGZF header") + " at compressed offset " + std::to_string(w.consumed);
        return KJ_ERR_IO;
    }
    if (w.out_bytes > out_cap || (w.out_bytes && !out)) { kj_err() = "kj_debug_inflate_bgzf: the output buffer is too small"; return KJ_ERR_ARG; }
    if (table.empty()) return KJ_OK;
    if (table.size() >= (1ull << 32)) { kj_err() = "kj_debug_inflate_bgzf: too many blocks"; return KJ_ERR_UNSUPPORTED; }
    KjDevBuf comp, tab, text, status; int rc; const uint32_t nblk = (uint32_t)table.size(); std::vector<uint32_t> st(nblk);
    if ((rc = comp.grow(w.consumed)) || (rc = tab.grow(nblk * sizeof(KjBgzfBlock))) || (rc = text.grow(w.out_bytes + 16)) || (rc = status.grow((size_t)nblk * 4))) return rc;
    cudaStream_t s = c->slot[0].stream;
    CK(cudaMemcpyAsync(comp.p, file_bytes, w.consumed, cudaMemcpyHostToDevice, s)); CK(cudaMemcpyAsync(tab.p, table.data(), nblk * sizeof(KjBgzfBlock), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(c->ev_a, s));
    kj_inflate_kernel<<<(nblk + KJ_INF_WARPS - 1) / KJ_INF_WARPS, KJ_INF_WARPS * 32, 0, s>>>(comp.as<uint8_t>(), tab.as<KjBgzfBlock>(), nblk, text.as<uint8_t>(), status.as<uint32_t>());
    CK(cudaGetLastError()); c->launches++;
    CK(cudaEventRecord(c->ev_b, s));
    CK(cudaMemcpyAsync(st.data(), status.p, (size_t)nblk * 4, cudaMemcpyDeviceToHost, s));
    if (w.out_bytes) CK(cudaMemcpyAsync(out, text.p, w.out_bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (uint32_t i = 0; i < nblk; i++) if (st[i]) {
        *first_bad_offset = table[i].in_off - table[i].hdr;
        kj_err() = "corrupt BGZF block at compressed offset " + std::to_string(*first_bad_offset) + ": " + kj_inflate_strerror(st[i]); return KJ_ERR_IO;
    }
    *out_n = w.out_bytes; return KJ_OK;
}
