// kj_build.h -- index construction on the device (SURVEY.md 8f-4): from the reference's in-memory index (BWT byte codes + sampled suffix
// array, the output of kaiju-mkfmi / readFMI: mkfmi.c:63-78, fmicommon.h:104-184) straight to the device layout of kj_layout.h.
//
// The host only uploads the raw bytes; the one-hot rank records, the packed letters, the taxon-reduced suffix array and the k-mer
// interval table are produced by the kernels below (the host transcoder of kj_host.cpp stays as the writer of device-native index
// files and as the CPU reference these kernels are tested against, array for array).
//
// `copies` > 1 builds the index of the collection in which every sequence occurs `copies` times in a row (kj_create_scaled).  That
// index follows from the base index without a suffix sort: identical suffixes are ordered by sequence number, so every suffix-array
// row of the base index becomes `copies` consecutive rows, BWT'[K r + c] = BWT[r], SA'[K r + c] = (K seq + c, pos) -- pinned against
// kaiju-mkbwt/-mkfmi run on the K-fold FASTA (tests/test_scaled_index.py).  It is how a refseq_ref-scale index (2.7e10 rows) is
// brought into HBM on a box that cannot run the reference's index builder at that size within a benchmark.
// Included by kj_device.cu (one translation unit).
#pragma once

#define KJ_BLD_THREADS 256
struct KjBuildLcode { uint8_t v[256]; };

// ---- pass 1: letter counts per tile of 256 rank blocks
template <int RB>
__global__ void __launch_bounds__(KJ_BLD_THREADS) kj_bld_count(const uint8_t* __restrict__ bwt, const __grid_constant__ KjBuildLcode lc, uint64_t n, uint32_t rep, int alen,
                                                                uint32_t* __restrict__ tile_counts) {
    __shared__ uint32_t tot[KJ_MAX_ALEN];
    __shared__ uint8_t lcs[256];
    __shared__ uint8_t cnt[KJ_MAX_ALEN * KJ_BLD_THREADS];             // per-thread counters (a thread sees RB <= 192 rows)
    if (threadIdx.x < KJ_MAX_ALEN) tot[threadIdx.x] = 0;
    lcs[threadIdx.x] = lc.v[threadIdx.x];
    for (int a = 0; a < KJ_MAX_ALEN; a++) cnt[a * KJ_BLD_THREADS + threadIdx.x] = 0;
    __syncthreads();
    const uint64_t tile_rows = (uint64_t)KJ_BLD_THREADS * RB, start = (uint64_t)blockIdx.x * tile_rows;
    for (uint32_t i = threadIdx.x; i < tile_rows; i += KJ_BLD_THREADS) {
        const uint64_t row = start + i;
        if (row < n) cnt[(uint32_t)lcs[bwt[rep == 1 ? row : row / rep]] * KJ_BLD_THREADS + threadIdx.x]++;
    }
    for (int a = 0; a < alen; a++) {
        uint32_t v = cnt[a * KJ_BLD_THREADS + threadIdx.x];
        for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(&tot[a], v);
    }
    __syncthreads();
    if (threadIdx.x < KJ_MAX_ALEN) tile_counts[(uint64_t)blockIdx.x * KJ_MAX_ALEN + threadIdx.x] = threadIdx.x < (uint32_t)alen ? tot[threadIdx.x] : 0u;
}
// exclusive scan of the tile counts per letter (one warp per letter); totals[a] = number of rows holding letter a
__global__ void kj_bld_scan_tiles(const uint32_t* __restrict__ tile_counts, uint64_t ntiles, uint64_t* __restrict__ tile_prefix, uint64_t* __restrict__ totals) {
    const uint32_t a = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t carry = 0;
    for (uint64_t t0 = 0; t0 < ntiles; t0 += 32) {
        const uint64_t t = t0 + lane; const uint64_t v = t < ntiles ? tile_counts[t * KJ_MAX_ALEN + a] : 0ull; uint64_t x = v;
        for (int d = 1; d < 32; d <<= 1) { const uint64_t o = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += o; }
        if (t < ntiles) tile_prefix[t * KJ_MAX_ALEN + a] = carry + x - v;
        carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) totals[a] = carry;
}

// ---- pass 2: rank records.  One thread per rank block (RB rows); the tile's letters are staged through shared memory (coalesced reads),
// each thread then builds, letter by letter, the one-hot words of its block with byte-wise SIMD compares; a block-wide scan of the
// per-block letter counts gives the header counts.
template <int RB, int RW>
__global__ void __launch_bounds__(KJ_BLD_THREADS) kj_bld_records(const uint8_t* __restrict__ bwt, const __grid_constant__ KjBuildLcode lc, uint64_t n, uint32_t rep, int alen, uint64_t nb,
                                                                  const uint64_t* __restrict__ tile_prefix, const uint64_t* __restrict__ Cdev, uint64_t* __restrict__ rank) {
    extern __shared__ __align__(16) uint8_t sm_raw[];
    constexpr int STR = RB + 4;                                          // row stride of a block's letters: odd number of words -> conflict-free word reads
    uint8_t* let = sm_raw;                                               // [256][STR]
    uint32_t* wsum = (uint32_t*)(sm_raw + (size_t)KJ_BLD_THREADS * STR); // [8] warp totals
    __shared__ uint8_t lcs[256];
    lcs[threadIdx.x] = lc.v[threadIdx.x];
    __syncthreads();
    const uint64_t tile_rows = (uint64_t)KJ_BLD_THREADS * RB, start = (uint64_t)blockIdx.x * tile_rows;
    for (uint32_t i = threadIdx.x; i < tile_rows; i += KJ_BLD_THREADS) {
        const uint64_t row = start + i;
        let[(i / RB) * STR + (i % RB)] = row < n ? lcs[bwt[rep == 1 ? row : row / rep]] : (uint8_t)0xff;
    }
    __syncthreads();
    const uint64_t b = (uint64_t)blockIdx.x * KJ_BLD_THREADS + threadIdx.x;
    const uint32_t* mine = (const uint32_t*)(let + (size_t)threadIdx.x * STR);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int a = 0; a < alen; a++) {
        uint64_t w[RB / 64]; uint32_t c = 0;
        const uint32_t a4 = (uint32_t)a * 0x01010101u;
        #pragma unroll
        for (int q = 0; q < RB / 64; q++) {
            uint64_t bits = 0;
            #pragma unroll
            for (int x = 0; x < 16; x++) {
                const uint32_t m = __vcmpeq4(mine[q * 16 + x], a4) & 0x01010101u;
                bits |= (uint64_t)((m * 0x01020408u) >> 24) << (4 * x);
            }
            w[q] = bits; c += (uint32_t)__popcll(bits);
        }
        // exclusive scan of c over the 256 blocks of the tile
        uint32_t x = c;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += o; }
        if (lane == 31) wsum[wid] = x;
        __syncthreads();
        uint32_t base = 0;
        for (uint32_t k = 0; k < wid; k++) base += wsum[k];
        __syncthreads();
        if (b < nb) {
            uint64_t hdr = Cdev[a] + tile_prefix[(uint64_t)blockIdx.x * KJ_MAX_ALEN + a] + (uint64_t)(base + x - c);
            uint64_t* rec = rank + ((uint64_t)a * nb + b) * RW;
            if (RW == 2) { *(ulonglong2*)rec = make_ulonglong2(hdr, w[0]); }
            else {
                const uint64_t p1 = (uint64_t)__popcll(w[0]), p2 = p1 + (uint64_t)__popcll(w[RB / 64 > 1 ? 1 : 0]);
                hdr = (hdr & KJ_CNT_MASK) | (p1 << KJ_P1_SHIFT) | (p2 << KJ_P2_SHIFT);
                *(ulonglong2*)rec = make_ulonglong2(hdr, w[0]);
                *(ulonglong2*)(rec + 2) = make_ulonglong2(w[RB / 64 > 1 ? 1 : 0], w[RB / 64 > 2 ? 2 : 0]);
            }
        }
    }
}
// packed letters: 12 per 64-bit word
__global__ void kj_bld_letters(const uint8_t* __restrict__ bwt, const __grid_constant__ KjBuildLcode lc, uint64_t n, uint32_t rep, uint64_t nwords, uint64_t* __restrict__ letters) {
    __shared__ uint8_t lcs[256];
    lcs[threadIdx.x] = lc.v[threadIdx.x];
    __syncthreads();
    for (uint64_t wd = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; wd < nwords; wd += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t v = 0;
        for (int t = 0; t < KJ_LETTERS_PER_WORD; t++) { const uint64_t row = wd * KJ_LETTERS_PER_WORD + t; if (row < n) v |= (uint64_t)lcs[bwt[rep == 1 ? row : row / rep]] << (5 * t); }
        letters[wd] = v;
    }
}
// sampled suffix array (big-endian packed (seq,pos), suffixArray.h:37-51) -> compact taxon of the sequence
__global__ void kj_bld_sa_tax(const uint8_t* __restrict__ sa, uint64_t n_entries, uint64_t first, int nbytes, int pbits, uint32_t nseq, const uint32_t* __restrict__ seq_tax,
                              uint32_t* __restrict__ sa_tax, uint32_t* __restrict__ err) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_entries; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* p = sa + e * (uint64_t)nbytes; uint64_t val = 0;
        for (int b = 0; b < nbytes; b++) val = (val << 8) + p[b];
        const uint64_t seq = val >> pbits;
        if (seq >= nseq) { atomicOr(err, 64u); continue; }
        sa_tax[first + e] = seq_tax[seq];
    }
}
// scaled index: the sampled row k' = (e + bias') << exp of the K-fold collection is copy k' % K of base row k' / K
template <class IdxT>
__global__ void kj_bld_sa_tax_scaled(const KjDevIndex* __restrict__ base_ix, uint64_t n_entries, int64_t bias, int exp, uint64_t n_rows, uint32_t rep, uint32_t* __restrict__ sa_tax) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_entries; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k = (uint64_t)((int64_t)e + bias) << exp;
        sa_tax[e] = k < n_rows ? kj_sa_taxon<IdxT>(*base_ix, k / rep) : KJ_TAX_BAD;
    }
}
// dense row -> taxon array: every row resolved by the classify kernels' own walk (kj_row_taxon), so the array equals the walk by construction,
// the guard entry of the sampled suffix array and the walks that end on a terminator included.  Narrow indexes only.
__global__ void kj_bld_row_tax(const KjDevIndex* __restrict__ ix, uint64_t n_rows, uint32_t* __restrict__ row_tax) {
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_rows; k += (uint64_t)gridDim.x * blockDim.x) row_tax[k] = kj_row_taxon<uint32_t>(*ix, k);
}
__global__ void kj_bld_repeat_u32(const uint32_t* __restrict__ src, uint64_t n_out, uint32_t rep, uint32_t* __restrict__ dst) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (uint64_t)gridDim.x * blockDim.x) dst[i] = src[i / rep];
}
// FMindex with the reference's checkpoint quirk applied (host_rank of kj_host.cpp)
template <class IdxT>
static __device__ __forceinline__ uint64_t kj_bld_rank(const KjDevIndex& ix, uint32_t c, uint64_t k) {
    uint64_t v = (uint64_t)kj_rank<IdxT>(ix, c, (IdxT)k);
    if (k >= ix.quirk_lo) v -= ix.quirk_d[c];
    return v;
}
template <class IdxT>
__global__ void kj_bld_quirk(const KjDevIndex* __restrict__ ix, uint64_t k, uint64_t* __restrict__ quirk_d) {
    const uint32_t a = threadIdx.x;
    if (a < (uint32_t)ix->alen) quirk_d[a] = (uint64_t)kj_rank<IdxT>(*ix, a, (IdxT)k) - ix->C[a];
}
// one level of the k-mer interval table: nxt[i*20 + a] = interval of cur[i] extended to the left by letter a+1
template <class IdxT>
__global__ void kj_bld_kmer_level(const KjDevIndex* __restrict__ ix, const KjKmer* __restrict__ cur, uint64_t n_cur, KjKmer* __restrict__ nxt) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_cur * 20u; t += (uint64_t)gridDim.x * blockDim.x) {
        const KjKmer iv = cur[t / 20u]; const uint32_t a = (uint32_t)(t % 20u); KjKmer o; o.lo = 0; o.hi = 0;
        if (iv.lo < iv.hi) { o.lo = kj_bld_rank<IdxT>(*ix, a + 1u, iv.lo); o.hi = kj_bld_rank<IdxT>(*ix, a + 1u, iv.hi); if (o.lo >= o.hi) { o.lo = 0; o.hi = 0; } }
        nxt[t] = o;
    }
}
__global__ void kj_bld_kmer_narrow(const KjKmer* __restrict__ src, uint64_t n, KjKmer32* __restrict__ dst) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x) { dst[t].lo = (uint32_t)src[t].lo; dst[t].hi = (uint32_t)src[t].hi; }
}

// chunked upload of a pageable host array
static int kj_bld_upload(void* d, const void* h, size_t bytes) {
    const size_t CH = (size_t)1 << 30;
    for (size_t o = 0; o < bytes; o += CH) CK(cudaMemcpy((char*)d + o, (const char*)h + o, std::min(CH, bytes - o), cudaMemcpyHostToDevice));
    return KJ_OK;
}

// ---- compact layout (kj_layout.h): one CTA per 65536-row superblock, one thread per 128-row record.  A record depends only on its own
// superblock, so the BWT can be built a chunk of whole superblocks at a time.  `bwt` holds rows [row0, ...) (rep == 1) or the whole base BWT
// (rep > 1: row r of the K-fold index is base row r / K).  sb_tot[s][c] = #c in superblock s (KJ_CSB_STRIDE per superblock).
// Record b goes to `dev` below the split record nb_dev, else to `host` (the host tier of kj_create_tiered: pinned host memory mapped into the
// device's address space).  The build writes the host tier directly through the mapped pointer rather than staging it in HBM and copying: the
// stores are posted PCIe writes of whole 16-byte words, each byte is written once, and no HBM is needed for a staging buffer -- HBM is exactly
// what an index with a host tier lacks.
// The output addressing is a policy, Out::rec(...) = where record b goes: KjBldOutTwo for the HBM / host-tier split (rec_out, rec_host, nb_dev),
// KjBldOutSpread for the segments of a group (kj_create_group, the table `spread`), which the build on the group's first device stores straight
// into the owning device's HBM over peer access -- the same direct stores as into the host tier, and no staging copy.  Both instances take every
// parameter and each reads only its own, so the two-output instance compiles to the code it had before the policy.
#define KJ_CSB_RECS (1u << (KJ_CSB_SHIFT - 7))
struct KjBldOutTwo {
    static __device__ __forceinline__ uint64_t* rec(uint64_t* dev, uint64_t* host, uint64_t nb_dev, const KjSpreadRef&, uint64_t b) {
        return b < nb_dev ? dev + b * KJ_RANK_WORDS_COMPACT : host + (b - nb_dev) * KJ_RANK_WORDS_COMPACT;
    }
};
struct KjBldOutSpread {
    static __device__ __forceinline__ uint64_t* rec(uint64_t*, uint64_t*, uint64_t, const KjSpreadRef& s, uint64_t b) {
        const uint32_t g = kj_spread_seg(s, b); return (uint64_t*)s.base[g] + (b - s.first[g]) * KJ_RANK_WORDS_COMPACT;
    }
};
template <class Out>
__global__ void __launch_bounds__(KJ_BLD_THREADS) kj_bld_compact(const uint8_t* __restrict__ bwt, const __grid_constant__ KjBuildLcode lc, uint64_t s0, uint64_t row0, uint64_t n,
                                                                  uint32_t rep, uint64_t nb, uint64_t* __restrict__ rec_out, uint64_t* __restrict__ rec_host, uint64_t nb_dev,
                                                                  uint32_t* __restrict__ sb_tot, const __grid_constant__ KjSpreadRef spread) {
    __shared__ uint8_t lcs[256];
    __shared__ __align__(16) uint16_t cnt[KJ_CSB_RECS][KJ_MAX_ALEN];    // #c in the first half of each record, then the midpoint counts
    __shared__ uint8_t full[KJ_CSB_RECS][KJ_MAX_ALEN];                  // #c in each record
    lcs[threadIdx.x] = lc.v[threadIdx.x];
    for (uint32_t i = threadIdx.x; i < KJ_CSB_RECS * KJ_MAX_ALEN; i += KJ_BLD_THREADS) { (&cnt[0][0])[i] = 0; (&full[0][0])[i] = 0; }
    __syncthreads();
    const uint64_t s = s0 + blockIdx.x;
    for (uint32_t r = threadIdx.x; r < KJ_CSB_RECS; r += KJ_BLD_THREADS) {
        const uint64_t b = (s << (KJ_CSB_SHIFT - 7)) + r;
        if (b >= nb) break;
        uint64_t pw[10];
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            uint64_t p0 = 0, p1 = 0, p2 = 0, p3 = 0, p4 = 0;
            for (uint32_t i = 0; i < 64; i++) {
                const uint64_t row = b * 128u + (uint32_t)h * 64u + i;
                uint32_t l = 31;                                             // rows past the end: a letter no rank query counts
                if (row < n) { l = lcs[bwt[rep == 1 ? row - row0 : row / rep]]; full[r][l]++; if (h == 0) cnt[r][l]++; }
                p0 |= (uint64_t)(l & 1u) << i; p1 |= (uint64_t)((l >> 1) & 1u) << i; p2 |= (uint64_t)((l >> 2) & 1u) << i;
                p3 |= (uint64_t)((l >> 3) & 1u) << i; p4 |= (uint64_t)((l >> 4) & 1u) << i;
            }
            pw[5 * h] = p0; pw[5 * h + 1] = p1; pw[5 * h + 2] = p2; pw[5 * h + 3] = p3; pw[5 * h + 4] = p4;
        }
        ulonglong2* o = (ulonglong2*)Out::rec(rec_out, rec_host, nb_dev, spread, b);
        #pragma unroll
        for (int q = 0; q < 5; q++) o[q] = make_ulonglong2(pw[2 * q], pw[2 * q + 1]);
    }
    __syncthreads();
    if (threadIdx.x < KJ_MAX_ALEN) {                                     // per letter: running count over the superblock's records
        const uint32_t c = threadIdx.x; uint32_t run = 0;
        for (uint32_t r = 0; r < KJ_CSB_RECS; r++) { const uint32_t h = cnt[r][c]; cnt[r][c] = (uint16_t)(run + h); run += full[r][c]; }
        sb_tot[s * KJ_CSB_STRIDE + c] = run;
    }
    __syncthreads();
    for (uint32_t r = threadIdx.x; r < KJ_CSB_RECS; r += KJ_BLD_THREADS) {
        const uint64_t b = (s << (KJ_CSB_SHIFT - 7)) + r;
        if (b >= nb) break;
        const ulonglong2* src = (const ulonglong2*)&cnt[r][0]; ulonglong2* o = (ulonglong2*)(Out::rec(rec_out, rec_host, nb_dev, spread, b) + KJ_CPT_COUNT_WORD);
        #pragma unroll
        for (int q = 0; q < 3; q++) o[q] = src[q];
    }
}
// superblock table: C[c] + the exclusive prefix of the superblock totals (already in `csb`)
__global__ void kj_bld_csb_add_c(uint64_t* __restrict__ csb, uint64_t nsb, const uint64_t* __restrict__ Cdev, int alen) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nsb * KJ_CSB_STRIDE; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = (uint32_t)(i % KJ_CSB_STRIDE); if (c < (uint32_t)alen) csb[i] += Cdev[c];
    }
}

// rows per chunk of the compact build (a whole number of superblocks); KJ_BUILD_CHUNK_ROWS: developer hook that forces many chunks on small indexes
static uint64_t kj_compact_chunk_rows() {
    uint64_t ch = 1ull << 30;
    if (const char* e = getenv("KJ_BUILD_CHUNK_ROWS")) { const long long x = atoll(e); if (x > 0 && (x & ((1ll << KJ_CSB_SHIFT) - 1)) == 0) ch = (uint64_t)x; }
    return ch;
}
// The compact layout's records and superblock table in one pass over the BWT: the raw bytes go up one chunk at a time (rep == 1), so the peak is
// the final arrays plus one chunk; a scan over the per-superblock totals then gives the superblock table and C[].
static int kj_device_build_compact(kj_ctx* c, const kj_index_view& v, const KjBuildLcode& lc, uint32_t rep, uint64_t& tot) {
    KjHostIndex& H = c->H; const int alen = H.alen; const uint64_t n = H.bwtlen, nb = H.nb, nsb = kj_csb_count(n);
    const uint64_t CH = kj_compact_chunk_rows(), sb_per_chunk = CH >> KJ_CSB_SHIFT;
    int rc; KjDevBuf bwt, sbt, small;
    const uint64_t nd = c->nb_dev;                      // records [nd, nb) go to the host tier (kj_choose_layout)
    if (c->group) {                                     // the group's segments are allocated (kj_group_alloc) and counted per device already
        if ((rc = c->letters.grow(nsb * KJ_CSB_STRIDE * 8))) return rc;
        tot += nsb * KJ_CSB_STRIDE * 8;
    } else {
        if ((rc = c->rank.grow(nd * KJ_RANK_WORDS_COMPACT * 8)) || (rc = c->rank_host.grow((nb - nd) * KJ_RANK_WORDS_COMPACT * 8)) || (rc = c->letters.grow(nsb * KJ_CSB_STRIDE * 8))) return rc;
        tot += nd * KJ_RANK_WORDS_COMPACT * 8 + nsb * KJ_CSB_STRIDE * 8; c->host_bytes += (nb - nd) * KJ_RANK_WORDS_COMPACT * 8;
    }
    if ((rc = sbt.grow(nsb * KJ_CSB_STRIDE * 4)) || (rc = small.grow(3 * KJ_MAX_ALEN * 8 + 64))) return rc;
    uint64_t* d_tot = small.as<uint64_t>(); uint64_t* d_C = d_tot + KJ_MAX_ALEN + 1;
    if (rep == 1) { if ((rc = bwt.grow((size_t)std::min(CH, n)))) return rc; }
    else if ((rc = bwt.grow((size_t)v.bwtlen)) || (rc = kj_bld_upload(bwt.p, v.bwt, (size_t)v.bwtlen))) return rc;
    for (uint64_t s0 = 0; s0 < nsb; s0 += sb_per_chunk) {
        const uint64_t row0 = s0 << KJ_CSB_SHIFT, nsc = std::min(sb_per_chunk, nsb - s0);
        if (rep == 1 && row0 < n) CK(cudaMemcpy(bwt.p, v.bwt + row0, (size_t)(std::min(n, row0 + CH) - row0), cudaMemcpyHostToDevice));
        if (c->group) kj_bld_compact<KjBldOutSpread><<<(unsigned)nsc, KJ_BLD_THREADS>>>(bwt.as<uint8_t>(), lc, s0, row0, n, rep, nb, nullptr, nullptr, 0, sbt.as<uint32_t>(), c->group->ref);
        else kj_bld_compact<KjBldOutTwo><<<(unsigned)nsc, KJ_BLD_THREADS>>>(bwt.as<uint8_t>(), lc, s0, row0, n, rep, nb, c->rank.as<uint64_t>(), c->rank_host.as<uint64_t>(), nd, sbt.as<uint32_t>(), KjSpreadRef{});
        CK(cudaGetLastError()); c->launches++;
        if (rep == 1) CK(cudaDeviceSynchronize());          // the next chunk's upload overwrites the staging buffer
    }
    bwt.reset();
    kj_bld_scan_tiles<<<1, 32 * KJ_MAX_ALEN>>>(sbt.as<uint32_t>(), nsb, c->letters.as<uint64_t>(), d_tot);
    CK(cudaGetLastError());
    uint64_t tots[KJ_MAX_ALEN]; CK(cudaMemcpy(tots, d_tot, sizeof tots, cudaMemcpyDeviceToHost));
    H.C[0] = 0; for (int a = 0; a < alen; a++) H.C[a + 1] = H.C[a] + tots[a];
    if (H.C[alen] != n) { kj_err() = "letter counts do not add up"; return KJ_ERR_IO; }
    CK(cudaMemcpy(d_C, H.C, sizeof(uint64_t) * (size_t)(alen + 1), cudaMemcpyHostToDevice));
    kj_bld_csb_add_c<<<c->sm_count * 4, 256>>>(c->letters.as<uint64_t>(), nsb, d_C, alen);
    CK(cudaGetLastError()); CK(cudaDeviceSynchronize()); c->launches += 2;
    return KJ_OK;
}

// HBM the placement of kj_create_tiered leaves free next to an index with a host tier, for classification: the two pipeline slots' staging and
// outputs for chunks of 2^20 read pairs (~0.7 GB), the per-warp spill, variant-ring and work-space scratch of the persistent grid (~0.3 GB for
// PE150 on 132 SMs x 4 CTAs x 8 warps), the Greedy path's prepared-item buffers (4 x 1/16 of the free memory, at least 1 GB at this size) and the
// CUDA context's own allocations, with room to spare for a read set that needs more scratch than PE150.
#define KJ_TIER_HEADROOM (4ull << 30)
// Layout of a 64-bit index built on the device: wide exactly when the peak HBM of the wide construction fits in the memory free now, else
// compact; when the compact construction does not fit either, KJ_ERR_NOMEM before anything large is allocated.  A peak is the maximum over the
// construction's phases: (1) BWT staging + scratch + the rank arrays, (2) rank arrays + suffix-array arrays + the upload chunk of the sampled
// suffix array, (3) rank arrays + suffix-array arrays + the two level buffers of the k-mer table.
// With a host memory budget (kj_create_tiered, host_budget > 0), a compact index whose peak does not fit gets a host tier in mapped pinned host
// memory instead, planned in this order, before anything large is allocated:
//   tier 1: the suffix-array taxon and accession arrays (sa_tax, seq_tax, sa_acc, seq_acc; read once at the end of each SA walk) -- layout 2;
//   tier 2: also the records [nb_dev, nb), nb_dev the largest count that leaves KJ_TIER_HEADROOM of HBM free -- layout 3 (compact tiered).
// KJ_ERR_NOMEM when the host tier would exceed the budget.  KJ_TIER_DEVICE_RECORDS=n (developer hook, any compact index built with a budget):
// nb_dev = n, tier 1 alone when n >= nb.
static int kj_choose_layout(kj_ctx* c, const kj_index_view& v, uint32_t rep, uint64_t host_budget) {
    KjHostIndex& H = c->H;
    if (H.wide == KJ_LAYOUT_NARROW) return KJ_OK;
    const uint64_t n = H.bwtlen, alen = (uint64_t)H.alen;
    size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to));
    const uint64_t n_sa = rep == 1 ? (uint64_t)v.ncheck + 1 : (uint64_t)std::max<int64_t>((int64_t)((n - 1) >> H.sa_exp) - H.sa_bias + 1, 4);
    const uint64_t acc = H.seq_acc.empty() ? 1 : 2;
    const uint64_t sa = acc * (n_sa + (uint64_t)H.nseq) * 4, upload = rep == 1 ? std::min<uint64_t>(1ull << 26, n_sa) * (uint64_t)v.nbytes : 0;
    uint64_t levels = 0;
    { const char* ek = getenv("KJ_KMER_K"); const int k = ek ? atoi(ek) : kj_default_kmer_k(n);
      if (k >= 2 && k <= 7 && alen == 21) { levels = 2 * sizeof(KjKmer); for (int d = 0; d < k; d++) levels *= 20; } }
    auto peak = [&](uint64_t arrays, uint64_t build) { return std::max(std::max(arrays + build, arrays + sa + upload), arrays + sa + levels); };
    const uint64_t nb_w = n / KJ_RANK_ROWS_WIDE + 1, ntiles = (nb_w + KJ_BLD_THREADS - 1) / KJ_BLD_THREADS;
    const uint64_t wide_peak = peak(kj_rank_array_words(KJ_LAYOUT_WIDE, H.alen, nb_w) * 8 + kj_letters_words(KJ_LAYOUT_WIDE, n) * 8, (uint64_t)v.bwtlen + ntiles * KJ_MAX_ALEN * 12);
    if (H.wide == KJ_LAYOUT_WIDE && wide_peak <= fr) return KJ_OK;
    const uint64_t nb_c = n / KJ_RANK_ROWS_COMPACT + 1, nsb = kj_csb_count(n);
    const uint64_t compact_peak = peak(kj_rank_array_words(KJ_LAYOUT_COMPACT, H.alen, nb_c) * 8 + kj_letters_words(KJ_LAYOUT_COMPACT, n) * 8,
                                       nsb * KJ_CSB_STRIDE * 4 + (rep == 1 ? std::min(kj_compact_chunk_rows(), n) : (uint64_t)v.bwtlen));
    const char* hook = host_budget ? getenv("KJ_TIER_DEVICE_RECORDS") : nullptr;
    if (compact_peak <= fr && !hook) { H.wide = KJ_LAYOUT_COMPACT; H.nb = nb_c; c->nb_dev = nb_c; return KJ_OK; }
    char b[400];
    if (!host_budget) {
        snprintf(b, sizeof b, "index of %llu rows does not fit in HBM: building it needs %llu bytes (compact layout), %llu bytes are free",
                 (unsigned long long)n, (unsigned long long)compact_peak, (unsigned long long)fr);
        kj_err() = b; return KJ_ERR_NOMEM;
    }
    // the host tier: what stays in HBM is the superblock table, records [0, nd) and the largest transient buffer of the construction
    const uint64_t rec = KJ_RANK_WORDS_COMPACT * 8, csb = kj_letters_words(KJ_LAYOUT_COMPACT, n) * 8;
    const uint64_t transient = std::max(std::max(nsb * KJ_CSB_STRIDE * 4 + (rep == 1 ? std::min(kj_compact_chunk_rows(), n) : (uint64_t)v.bwtlen), upload), levels);
    uint64_t nd = nb_c;
    if (hook) nd = std::min<uint64_t>((uint64_t)std::max(0ll, atoll(hook)), nb_c);
    else if (nb_c * rec + csb + transient + KJ_TIER_HEADROOM > fr) {
        const uint64_t fixed = csb + transient + KJ_TIER_HEADROOM;
        if (fixed > fr) {
            snprintf(b, sizeof b, "index of %llu rows does not fit: %llu bytes of HBM are free, its superblock table and construction buffers need %llu bytes next to %llu bytes of headroom",
                     (unsigned long long)n, (unsigned long long)fr, (unsigned long long)(csb + transient), (unsigned long long)KJ_TIER_HEADROOM);
            kj_err() = b; return KJ_ERR_NOMEM;
        }
        nd = std::min<uint64_t>(nb_c, (fr - fixed) / rec);
    }
    const uint64_t host_need = sa + 64 + (nb_c - nd) * rec;
    if (host_need > host_budget) {
        snprintf(b, sizeof b, "index of %llu rows does not fit: %llu bytes of HBM are free, its host tier needs %llu bytes of pinned host memory, the budget (host_bytes) is %llu bytes",
                 (unsigned long long)n, (unsigned long long)fr, (unsigned long long)host_need, (unsigned long long)host_budget);
        kj_err() = b; return KJ_ERR_NOMEM;
    }
    H.wide = nd < nb_c ? KJ_LAYOUT_COMPACT_TIERED : KJ_LAYOUT_COMPACT; H.nb = nb_c; c->nb_dev = nd;
    c->sa_tax.on_host = c->seq_tax.on_host = c->sa_acc.on_host = c->seq_acc.on_host = true;
    return KJ_OK;
}

// Placement of a compact spread index (kj_create_group) over the group's contexts cs[0..n) (cs[0] holds the meta data), before anything large is
// allocated.  It starts from the HBM free on each distinct device (a device listed twice shares its free memory between its two segments) and
// reserves, in this order:
//   1. on each context's device: its replicas (superblock table, k-mer table, taxonomy and tables, counts) and KJ_TIER_HEADROOM for classifying;
//   2. on the first device: the largest transient buffer of the construction (BWT chunk + superblock totals, suffix-array upload chunk, the second
//      k-mer level buffer), which runs there;
//   3. the suffix-array arrays (sa_tax, sa_acc, seq_tax, seq_acc), each whole on the device with the most room left;
//   4. the records, cut into contiguous segments in group order, in proportion to the room each group member has left.
// KJ_ERR_NOMEM when the group is too small; the message names the bytes needed and the bytes free on each device.  KJ_SPREAD_RECORDS=n0,n1,...
// (developer hook) forces the record count of every segment but the last, which takes the rest.
static int kj_plan_group(kj_ctx* const* cs, int n, const kj_index_view& v, uint32_t rep, KjGroup& G) {
    kj_ctx* c0 = cs[0]; KjHostIndex& H = c0->H;
    const uint64_t rows = H.bwtlen, nb = rows / KJ_RANK_ROWS_COMPACT + 1, nsb = kj_csb_count(rows), rec = KJ_RANK_WORDS_COMPACT * 8;
    if (nb >= 0xffffffffull) { kj_err() = "kj_create_group: index of " + std::to_string(rows) + " rows has more than 2^32 - 2 compact records"; return KJ_ERR_UNSUPPORTED; }
    H.wide = KJ_LAYOUT_COMPACT_SPREAD; H.nb = nb; c0->nb_dev = nb;
    // free HBM per distinct device
    std::vector<int> devs; std::vector<uint64_t> fr;
    for (int g = 0; g < n; g++) {
        if (std::find(devs.begin(), devs.end(), cs[g]->device) != devs.end()) continue;
        KjDevGuard d(cs[g]->device); size_t f = 0, t = 0; CK(cudaMemGetInfo(&f, &t));
        devs.push_back(cs[g]->device); fr.push_back(f);
    }
    auto slot = [&](int dev) { return (size_t)(std::find(devs.begin(), devs.end(), dev) - devs.begin()); };
    std::vector<int64_t> room(fr.begin(), fr.end());
    // 1. replicas + headroom per context
    uint64_t kmer = 0;
    { const char* ek = getenv("KJ_KMER_K"); const int k = ek ? atoi(ek) : kj_default_kmer_k(rows);
      if (k >= 2 && k <= 7 && H.alen == 21) { kmer = sizeof(KjKmer); for (int d = 0; d < k; d++) kmer *= 20; } }
    const uint64_t csb = nsb * KJ_CSB_STRIDE * 8, small = H.tax_parent.size() * 4 + H.tax_depth.size() * 4 + H.tax_id.size() * 8 + H.lnfact.size() * 8 +
                         sizeof(KjTables) + (H.tax_id.size() + 1) * 16 + 4096;
    const uint64_t replica = csb + kmer + small + KJ_TIER_HEADROOM;
    for (int g = 0; g < n; g++) room[slot(cs[g]->device)] -= (int64_t)replica;
    // 2. the construction's largest transient buffer, on the first device
    const uint64_t n_sa = rep == 1 ? (uint64_t)v.ncheck + 1 : (uint64_t)std::max<int64_t>((int64_t)((rows - 1) >> H.sa_exp) - H.sa_bias + 1, 4);
    const uint64_t upload = rep == 1 ? std::min<uint64_t>(1ull << 26, n_sa) * (uint64_t)v.nbytes : 0;
    const uint64_t transient = std::max(std::max(nsb * KJ_CSB_STRIDE * 4 + (rep == 1 ? std::min(kj_compact_chunk_rows(), rows) : (uint64_t)v.bwtlen), upload), kmer);
    room[slot(c0->device)] -= (int64_t)transient;
    // 3. the suffix-array arrays, whole, each on the device with the most room left
    const bool acc = !H.seq_acc.empty();
    const uint64_t sa_bytes = std::max<uint64_t>(n_sa * 4 + 4, 16), seq_bytes = std::max<uint64_t>((uint64_t)H.nseq * 4, 16);
    struct { KjTierBuf* b; uint64_t bytes; } arrays[4] = {{&c0->sa_tax, sa_bytes}, {&c0->sa_acc, acc ? sa_bytes : 0}, {&c0->seq_tax, seq_bytes}, {&c0->seq_acc, acc ? seq_bytes : 0}};
    uint64_t sa_total = 0;
    for (auto& a : arrays) {
        if (!a.bytes) continue;
        const size_t best = (size_t)(std::max_element(room.begin(), room.end()) - room.begin());
        a.b->device = devs[best]; room[best] -= (int64_t)a.bytes; sa_total += a.bytes;
    }
    // 4. the records, in proportion to the room left per group member
    std::vector<uint64_t> share((size_t)n, 0); unsigned __int128 total_share = 0; bool fits = true;
    for (size_t d = 0; d < devs.size(); d++) if (room[d] < 0) fits = false;
    for (int g = 0; g < n; g++) {
        const size_t d = slot(cs[g]->device); const int64_t members = (int64_t)std::count_if(cs, cs + n, [&](const kj_ctx* x) { return x->device == devs[d]; });
        share[(size_t)g] = room[d] > 0 ? (uint64_t)(room[d] / members) : 0; total_share += share[(size_t)g];
    }
    const char* hook = getenv("KJ_SPREAD_RECORDS");
    if (!hook && (!fits || total_share < (unsigned __int128)nb * rec)) {
        uint64_t need = nb * rec + sa_total + replica * (uint64_t)n + transient;
        std::string m = "index of " + std::to_string(rows) + " rows does not fit in the HBM of the group: it needs " + std::to_string(need) + " bytes (records " +
                        std::to_string(nb * rec) + ", suffix-array arrays " + std::to_string(sa_total) + ", " + std::to_string(replica) + " per context for its replicas and " +
                        std::to_string((uint64_t)KJ_TIER_HEADROOM) + " bytes of headroom, construction " + std::to_string(transient) + "); free:";
        for (size_t d = 0; d < devs.size(); d++) m += (d ? ", device " : " device ") + std::to_string(devs[d]) + " " + std::to_string(fr[d]) + " bytes";
        kj_err() = m; return KJ_ERR_NOMEM;
    }
    G.n = n; G.first[0] = 0;
    if (hook) {
        const char* p = hook;
        for (int g = 0; g + 1 < n; g++) {
            const uint64_t want = *p ? strtoull(p, (char**)&p, 10) : 0; if (*p == ',') p++;
            G.first[g + 1] = std::min(nb, G.first[g] + want);
        }
    } else {
        unsigned __int128 cum = 0;
        for (int g = 0; g + 1 < n; g++) { cum += share[(size_t)g]; G.first[g + 1] = (uint64_t)((unsigned __int128)nb * cum / total_share); }
    }
    G.first[n] = nb;
    for (int g = 0; g < n; g++) G.dev[g] = cs[g]->device;
    return KJ_OK;
}
// The segments kj_plan_group laid out, each on its owner's device, and the segment table of the descriptors.
static int kj_group_alloc(KjGroup& G) {
    memset(&G.ref, 0, sizeof G.ref);
    for (int g = 0; g < KJ_MAX_GROUP; g++) G.ref.first[g] = ~0ull;
    for (int g = 0; g < G.n; g++) {
        KjDevGuard d(G.dev[g]);
        int rc = G.seg[g].grow((size_t)(G.first[g + 1] - G.first[g]) * KJ_RANK_WORDS_COMPACT * 8); if (rc) return rc;
        G.ref.base[g] = G.seg[g].as<const uint64_t>(); G.ref.first[g] = G.first[g];
    }
    G.ref.n = (uint32_t)G.n;
    return KJ_OK;
}

// The one-hot layouts (narrow, wide): rank records and packed letters from the whole BWT on the device.
static int kj_device_build_onehot(kj_ctx* c, const kj_index_view& v, const KjBuildLcode& lc, uint32_t rep, uint64_t& tot) {
    KjHostIndex& H = c->H; const int alen = H.alen; const uint64_t n = H.bwtlen, nb = H.nb; const int wide = H.wide;
    const uint32_t RB = kj_rank_rows(wide), RW = kj_rank_words(wide);
    const int grid_big = c->sm_count * 16;
    // ---- BWT bytes to the device (freed again below)
    KjDevBuf bwt; int rc = bwt.grow((size_t)v.bwtlen); if (rc) return rc;
    const uint8_t* d_bwt = bwt.as<uint8_t>();
    if ((rc = kj_bld_upload(bwt.p, v.bwt, (size_t)v.bwtlen))) return rc;
    // ---- letter counts per tile, C[]
    const uint64_t ntiles = (nb + KJ_BLD_THREADS - 1) / KJ_BLD_THREADS;
    if (ntiles >= (1ull << 31)) { kj_err() = "index too large"; return KJ_ERR_UNSUPPORTED; }
    KjDevBuf tc, tp, small;
    if ((rc = tc.grow(ntiles * KJ_MAX_ALEN * 4)) || (rc = tp.grow(ntiles * KJ_MAX_ALEN * 8)) || (rc = small.grow(3 * KJ_MAX_ALEN * 8 + 64))) return rc;
    uint32_t* d_tc = tc.as<uint32_t>(); uint64_t* d_tp = tp.as<uint64_t>();
    uint64_t* d_tot = small.as<uint64_t>(); uint64_t* d_C = d_tot + KJ_MAX_ALEN + 1;
    if (wide) kj_bld_count<KJ_RANK_ROWS_WIDE><<<(unsigned)ntiles, KJ_BLD_THREADS>>>(d_bwt, lc, n, rep, alen, d_tc);
    else kj_bld_count<KJ_RANK_ROWS_NARROW><<<(unsigned)ntiles, KJ_BLD_THREADS>>>(d_bwt, lc, n, rep, alen, d_tc);
    kj_bld_scan_tiles<<<1, 32 * KJ_MAX_ALEN>>>(d_tc, ntiles, d_tp, d_tot);
    CK(cudaGetLastError());
    uint64_t tots[KJ_MAX_ALEN]; CK(cudaMemcpy(tots, d_tot, sizeof tots, cudaMemcpyDeviceToHost));
    H.C[0] = 0; for (int a = 0; a < alen; a++) H.C[a + 1] = H.C[a] + tots[a];
    if (H.C[alen] != n) { kj_err() = "letter counts do not add up"; return KJ_ERR_IO; }
    CK(cudaMemcpy(d_C, H.C, sizeof(uint64_t) * (size_t)(alen + 1), cudaMemcpyHostToDevice));
    // ---- rank records
    const size_t rank_bytes = (size_t)alen * nb * RW * 8;
    if ((rc = c->rank.grow(rank_bytes))) return rc;
    tot += rank_bytes;
    {
        const size_t smem = (size_t)KJ_BLD_THREADS * (RB + 4) + 64;
        if (wide) {
            CK(cudaFuncSetAttribute(kj_bld_records<KJ_RANK_ROWS_WIDE, KJ_RANK_WORDS_WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kj_bld_records<KJ_RANK_ROWS_WIDE, KJ_RANK_WORDS_WIDE><<<(unsigned)ntiles, KJ_BLD_THREADS, smem>>>(d_bwt, lc, n, rep, alen, nb, d_tp, d_C, c->rank.as<uint64_t>());
        } else kj_bld_records<KJ_RANK_ROWS_NARROW, KJ_RANK_WORDS_NARROW><<<(unsigned)ntiles, KJ_BLD_THREADS, smem>>>(d_bwt, lc, n, rep, alen, nb, d_tp, d_C, c->rank.as<uint64_t>());
        CK(cudaGetLastError());
    }
    // ---- packed letters
    const uint64_t nwords = n / KJ_LETTERS_PER_WORD + 2;
    if ((rc = c->letters.grow(nwords * 8))) return rc;
    tot += nwords * 8;
    kj_bld_letters<<<grid_big, 256>>>(d_bwt, lc, n, rep, nwords, c->letters.as<uint64_t>());
    CK(cudaGetLastError()); CK(cudaDeviceSynchronize());
    c->launches += 4;
    return KJ_OK;       // the BWT and tile arrays go before the suffix-array arrays are allocated
}

// Builds the large arrays of the context on the device.  c->H holds the meta data (kj_build_host_meta); `base` (scaled build only) is a
// finished context over the same index with copies = 1, whose device index resolves base suffix-array rows to taxa.
static int kj_device_build(kj_ctx* c, const kj_index_view& v, const uint8_t lcode[256], uint32_t rep, const kj_ctx* base, uint64_t& tot) {
    KjHostIndex& H = c->H; const uint64_t n = H.bwtlen; int rc;
    KjBuildLcode lc; memcpy(lc.v, lcode, 256);
    const int grid_big = c->sm_count * 16;
    if ((rc = kj_is_compact(H.wide) ? kj_device_build_compact(c, v, lc, rep, tot) : kj_device_build_onehot(c, v, lc, rep, tot))) return rc;
    // ---- sequence -> taxon, sampled suffix array -> taxon (in HBM, or in the host tier: kj_choose_layout)
    if ((rc = tier_upload(c, H.seq_tax, c->seq_tax, tot))) return rc;
    if (!H.seq_acc.empty() && (rc = tier_upload(c, H.seq_acc, c->seq_acc, tot))) return rc;
    uint32_t* d_err = c->err.as<uint32_t>();
    uint64_t n_sa;
    if (rep == 1) {
        n_sa = (uint64_t)v.ncheck;
        if ((rc = tier_grow(c, c->sa_tax, (n_sa + 1) * 4, tot)) || (rc = c->sa_tax.fill(n_sa * 4, 0xff, 4))) return rc;   // guard entry (see create_ctx): the last sampled row has no entry in a reference-built index
        if (c->seq_acc.p && ((rc = tier_grow(c, c->sa_acc, (n_sa + 1) * 4, tot)) || (rc = c->sa_acc.fill(n_sa * 4, 0xff, 4)))) return rc;
        const uint64_t CHE = (uint64_t)1 << 26;                        // entries per upload chunk
        KjDevBuf sa; if ((rc = sa.grow((size_t)std::min<uint64_t>(CHE, std::max<uint64_t>(n_sa, 1)) * (size_t)v.nbytes))) return rc;
        for (uint64_t e0 = 0; e0 < n_sa; e0 += CHE) {
            const uint64_t m = std::min(CHE, n_sa - e0);
            CK(cudaMemcpy(sa.p, v.sa + e0 * (uint64_t)v.nbytes, (size_t)m * (size_t)v.nbytes, cudaMemcpyHostToDevice));
            kj_bld_sa_tax<<<grid_big, 256>>>(sa.as<uint8_t>(), m, e0, v.nbytes, v.pbits, (uint32_t)v.nseq, c->seq_tax.as<uint32_t>(), c->sa_tax.as<uint32_t>(), d_err);
            if (c->sa_acc.p) kj_bld_sa_tax<<<grid_big, 256>>>(sa.as<uint8_t>(), m, e0, v.nbytes, v.pbits, (uint32_t)v.nseq, c->seq_acc.as<uint32_t>(), c->sa_acc.as<uint32_t>(), d_err);
            CK(cudaGetLastError()); CK(cudaDeviceSynchronize()); c->launches++;
        }
        uint32_t e = 0; CK(cudaMemcpy(&e, d_err, 4, cudaMemcpyDeviceToHost));
        if (e & 64u) { CK(cudaMemset(d_err, 0, 4)); kj_err() = "corrupt suffix array (sequence number out of range)"; return KJ_ERR_IO; }
    } else {
        const int64_t last = (int64_t)((n - 1) >> H.sa_exp) - H.sa_bias;  // entry of the last sampled row
        n_sa = last >= 0 ? (uint64_t)last + 1 : 0;
        if ((rc = tier_grow(c, c->sa_tax, std::max<size_t>(n_sa * 4, 16), tot))) return rc;
        if (base->H.wide == KJ_LAYOUT_COMPACT_SPREAD) kj_bld_sa_tax_scaled<KjSpreadIdx><<<grid_big, 256>>>(base->ix.as<KjDevIndex>(), n_sa, H.sa_bias, H.sa_exp, n, rep, c->sa_tax.as<uint32_t>());
        else if (base->H.wide == KJ_LAYOUT_COMPACT_TIERED) kj_bld_sa_tax_scaled<KjTieredIdx><<<grid_big, 256>>>(base->ix.as<KjDevIndex>(), n_sa, H.sa_bias, H.sa_exp, n, rep, c->sa_tax.as<uint32_t>());
        else if (base->H.wide == KJ_LAYOUT_COMPACT) kj_bld_sa_tax_scaled<KjCompactIdx><<<grid_big, 256>>>(base->ix.as<KjDevIndex>(), n_sa, H.sa_bias, H.sa_exp, n, rep, c->sa_tax.as<uint32_t>());
        else if (base->H.wide) kj_bld_sa_tax_scaled<uint64_t><<<grid_big, 256>>>(base->ix.as<KjDevIndex>(), n_sa, H.sa_bias, H.sa_exp, n, rep, c->sa_tax.as<uint32_t>());
        else kj_bld_sa_tax_scaled<uint32_t><<<grid_big, 256>>>(base->ix.as<KjDevIndex>(), n_sa, H.sa_bias, H.sa_exp, n, rep, c->sa_tax.as<uint32_t>());
        CK(cudaGetLastError()); CK(cudaDeviceSynchronize()); c->launches++;
    }
    c->n_sa = n_sa;
    return KJ_OK;
}

// quirk constants and the k-mer table need rank queries on the finished records: run after the device descriptor exists
// dst/k_out: where the table and its k go (the context's table for both modes, or the second, larger table of the MEM kernels)
static int kj_device_build_kmer(kj_ctx* c, int k, uint64_t& tot, KjDevBuf& dst, int& k_out) {
    KjHostIndex& H = c->H; const int wide = H.wide; const KjDevIndex* ix = c->ix.as<KjDevIndex>();
    if (H.quirk_lo != ~0ull && &dst == &c->kmer) {
        if (wide == KJ_LAYOUT_COMPACT_SPREAD) kj_bld_quirk<KjSpreadIdx><<<1, 32>>>(ix, H.bwtlen - 65536ull, c->quirk.as<uint64_t>());
        else if (wide == KJ_LAYOUT_COMPACT_TIERED) kj_bld_quirk<KjTieredIdx><<<1, 32>>>(ix, H.bwtlen - 65536ull, c->quirk.as<uint64_t>());
        else if (wide == KJ_LAYOUT_COMPACT) kj_bld_quirk<KjCompactIdx><<<1, 32>>>(ix, H.bwtlen - 65536ull, c->quirk.as<uint64_t>());
        else if (wide) kj_bld_quirk<uint64_t><<<1, 32>>>(ix, H.bwtlen - 65536ull, c->quirk.as<uint64_t>()); else kj_bld_quirk<uint32_t><<<1, 32>>>(ix, H.bwtlen - 65536ull, c->quirk.as<uint64_t>());
        CK(cudaGetLastError()); CK(cudaMemcpy(H.quirk_d, c->quirk.p, sizeof H.quirk_d, cudaMemcpyDeviceToHost)); c->launches++;
    }
    k_out = 0;
    if (k < 2 || k > 7 || H.alen != 21) return KJ_OK;
    uint64_t n_final = 1; for (int d = 0; d < k; d++) n_final *= 20;
    { size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to));      // two level buffers + the final table next to the index: a smaller k when that does not fit
      while (k > 2 && (double)n_final * (2.0 * sizeof(KjKmer) + sizeof(KjKmer32)) > 0.8 * (double)fr) { k--; n_final /= 20; } }
    KjDevBuf a, b; int rc;
    if ((rc = a.grow(n_final * sizeof(KjKmer))) || (rc = b.grow(n_final * sizeof(KjKmer)))) return rc;
    std::vector<KjKmer> first(20); for (uint32_t l = 0; l < 20; l++) { first[l].lo = H.C[l + 1]; first[l].hi = H.C[l + 2]; }
    CK(cudaMemcpy(a.p, first.data(), 20 * sizeof(KjKmer), cudaMemcpyHostToDevice));
    uint64_t n_cur = 20;
    for (int d = 1; d < k; d++) {
        const unsigned g = (unsigned)std::min<uint64_t>((n_cur * 20 + 255) / 256, (uint64_t)c->sm_count * 32);
        if (wide == KJ_LAYOUT_COMPACT_SPREAD) kj_bld_kmer_level<KjSpreadIdx><<<g, 256>>>(ix, a.as<KjKmer>(), n_cur, b.as<KjKmer>());
        else if (wide == KJ_LAYOUT_COMPACT_TIERED) kj_bld_kmer_level<KjTieredIdx><<<g, 256>>>(ix, a.as<KjKmer>(), n_cur, b.as<KjKmer>());
        else if (wide == KJ_LAYOUT_COMPACT) kj_bld_kmer_level<KjCompactIdx><<<g, 256>>>(ix, a.as<KjKmer>(), n_cur, b.as<KjKmer>());
        else if (wide) kj_bld_kmer_level<uint64_t><<<g, 256>>>(ix, a.as<KjKmer>(), n_cur, b.as<KjKmer>()); else kj_bld_kmer_level<uint32_t><<<g, 256>>>(ix, a.as<KjKmer>(), n_cur, b.as<KjKmer>());
        CK(cudaGetLastError()); c->launches++;
        std::swap(a, b); n_cur *= 20;
    }
    if (wide) { dst = std::move(a); tot += n_final * sizeof(KjKmer); }
    else {
        if ((rc = dst.grow(n_final * sizeof(KjKmer32)))) return rc;
        tot += n_final * sizeof(KjKmer32);
        kj_bld_kmer_narrow<<<c->sm_count * 8, 256>>>(a.as<KjKmer>(), n_final, dst.as<KjKmer32>()); CK(cudaGetLastError()); c->launches++;
    }
    CK(cudaDeviceSynchronize());
    k_out = k;
    return KJ_OK;
}

// The dense row -> taxon array of a finished narrow index (descriptor uploaded, k-mer tables decided), when it fits next to the index with
// KJ_ROW_TAX_MARGIN to spare.  Not for wide indexes (4 B per row next to 3.5 B of rank records) nor for the base context that kj_create_scaled
// throws away after the construction.
#define KJ_ROW_TAX_MARGIN (8ull << 30)
static int kj_device_build_row_tax(kj_ctx* c, uint64_t& tot) {
    const KjHostIndex& H = c->H;
    if (H.wide || kj_transient_ctx) return KJ_OK;
    const size_t bytes = (size_t)H.bwtlen * 4;
    size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to));
    if (bytes + KJ_ROW_TAX_MARGIN > fr) return KJ_OK;
    int rc = c->row_tax.grow(bytes); if (rc) return rc;
    kj_bld_row_tax<<<c->sm_count * 16, 256>>>(c->ix.as<KjDevIndex>(), H.bwtlen, c->row_tax.as<uint32_t>());
    CK(cudaGetLastError()); CK(cudaDeviceSynchronize()); c->launches++;
    tot += bytes;
    return KJ_OK;
}
