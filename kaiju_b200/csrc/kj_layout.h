// kj_layout.h -- HBM data layout of the index, taxonomy and tables (shared by host builder and kernels).
//
// The reference keeps the BWT as one byte per letter that also encodes a distance to the nearest 256-
// checkpoint (bwt/compactfmi.c:44-65) plus two checkpoint tables behind row pointers
// (bwt/fmicommon.h:60-73).  A rank query there costs two dependent pointer derefs plus a byte scan of
// ~18-30 bytes.  Rank values are a pure function of the decoded letters (SURVEY.md 8a exactness note a),
// so the device uses its own layout, built at load time from the decoded letters:
//
//   rank[c][b] : one record per (letter c, block b of 64 or 192 BWT positions; one-hot layouts, below); the 192-row one:
//                { hdr = C[c] + #{p < 192 b : L[p] == c} (40 bit) + the popcounts of w0 and w0|w1 (2 x 8 bit),
//                  w0,w1,w2 = one-hot bitmap of L[p]==c }
//                -> FMindex(c,k) touches exactly ONE 32-byte DRAM sector and needs ONE 64-bit popcount.
//   letters    : the decoded BWT packed 12 letters (5 bit) per 64-bit word, read only by the SA walk.
//   sa_tax     : the sampled suffix array reduced to what classification needs -- the (compact) taxon of
//                the sequence each sampled suffix belongs to (bwt/suffixArray.h:47-51 + ConsumerThread.cpp:812-832).
//   seq_tax    : compact taxon per sequence number (used when the LF walk runs into a terminator, bwt.c:119).
//   row_tax    : compact taxon per BWT row (4 B per row), built on the device from the three arrays above by walking every row once:
//                resolves a matched row with one load instead of an LF walk of ~2^sa_exp dependent steps.
//   tax_*      : taxonomy re-indexed densely: ids present in nodes.dmp get indices [0,n_present), DB taxa
//                absent from nodes.dmp get the indices after that (depth 0 marks "absent", util.cpp:206).
#pragma once
#include <stddef.h>
#include <stdint.h>

// Three record layouts, chosen per index at load time:
//   narrow (bwtlen < 2^32, 32-bit interval kernels): 16-byte records per 64 rows  { hdr = C[c] + #c before the block, w0 = one-hot bitmap }
//          -> one 16-byte load + one popcount per rank query, no division; 5.25 B per BWT row (faster than the 192-row layout where both fit)
//   wide   (bwtlen >= 2^32, 64-bit interval kernels): 32-byte records per 192 rows { hdr (40-bit count | popc(w0) | popc(w0)+popc(w1)), w0, w1, w2 }
//          -> 3.5 B per row: an index of 1.2e10 rows takes 42 GB of the 80 GB HBM instead of 63 GB
//   compact (64-bit kernels, indexes whose wide construction does not fit in HBM): the letters themselves, not one bitmap per letter.
//          128-byte records per 128 rows { 5 bit-planes of rows 0-63 | 5 bit-planes of rows 64-127 (2 x 40 B) | 24 x uint16: #c from the start
//          of the record's 65536-row superblock to the record's midpoint (row 64) }, plus `csb` = C[c] + #c before each superblock (24 x uint64
//          per superblock).  FMindex(c,k) = csb + mid count +/- the popcount of "plane word == c" between k and the midpoint: 5 plane words, one
//          count word and one superblock word, all addressed from (c,k) alone.  The same record gives the letter of row k (no `letters` array).
//          1.003 B per row: refseq_ref (2.7e10 rows) fits an 80 GB H100.  Rows past bwtlen hold letter 31, which no rank query counts.
//   compact tiered (kj_create_tiered, indexes whose compact construction does not fit in HBM either): the compact records, split at record
//          nb_dev: records [0, nb_dev) in HBM, records [nb_dev, nb) in pinned host memory mapped into the device's address space (read over PCIe).
//          Everything else of the index stays in HBM.  The record format is the compact one; only the address of record b depends on the split.
//   compact spread (kj_create_group, indexes larger than the HBM of one GPU): the compact records cut into at most KJ_MAX_GROUP contiguous
//          segments, segment g = records [first[g], first[g+1]) in the HBM of the group's g-th device, read by the kernels of every device of
//          the group over peer access (NVLink).  Each device holds its own superblock table, k-mer table and taxonomy; the suffix-array arrays
//          lie whole on one device each.  The record format is the compact one; only the address of record b depends on the segments.
// Layout codes (KjDevIndex::wide, KjHostIndex::wide): 0 narrow, 1 wide, 2 compact, 3 compact tiered, 4 compact spread.
#define KJ_LAYOUT_NARROW 0
#define KJ_LAYOUT_WIDE 1
#define KJ_LAYOUT_COMPACT 2
#define KJ_LAYOUT_COMPACT_TIERED 3
#define KJ_LAYOUT_COMPACT_SPREAD 4
#define KJ_MAX_GROUP 8             // devices (and record segments) of a compact spread index
#define KJ_RANK_ROWS_NARROW 64
#define KJ_RANK_ROWS_WIDE 192
#define KJ_RANK_ROWS_COMPACT 128
#define KJ_RANK_WORDS_NARROW 2
#define KJ_RANK_WORDS_WIDE 4
#define KJ_RANK_WORDS_COMPACT 16
#define KJ_CPT_COUNT_WORD 10       // compact record: the 16-bit midpoint counts start at word 10
#define KJ_CSB_SHIFT 16            // compact superblock: 2^16 rows = 512 records
#define KJ_CSB_STRIDE 24           // compact superblock table: words per superblock (KJ_MAX_ALEN)
static inline bool kj_is_compact(int layout) { return layout == KJ_LAYOUT_COMPACT || layout == KJ_LAYOUT_COMPACT_TIERED || layout == KJ_LAYOUT_COMPACT_SPREAD; }     // the compact record format
static inline uint32_t kj_rank_rows(int layout) { return kj_is_compact(layout) ? KJ_RANK_ROWS_COMPACT : layout ? KJ_RANK_ROWS_WIDE : KJ_RANK_ROWS_NARROW; }
static inline uint32_t kj_rank_words(int layout) { return kj_is_compact(layout) ? KJ_RANK_WORDS_COMPACT : layout ? KJ_RANK_WORDS_WIDE : KJ_RANK_WORDS_NARROW; }
// 64-bit words of the rank array: one record per (letter, block) in the one-hot layouts, one record per block in the compact one
static inline uint64_t kj_rank_array_words(int layout, int alen, uint64_t nb) { return (kj_is_compact(layout) ? 1ull : (uint64_t)alen) * nb * kj_rank_words(layout); }
static inline uint64_t kj_csb_count(uint64_t bwtlen) { return (bwtlen >> KJ_CSB_SHIFT) + 1; }     // superblocks of a compact index (k = bwtlen included)
#define KJ_LETTERS_PER_WORD 12
// 64-bit words of the `letters` array: the packed letters, or the superblock table of the compact layout
static inline uint64_t kj_letters_words(int layout, uint64_t bwtlen) { return kj_is_compact(layout) ? kj_csb_count(bwtlen) * KJ_CSB_STRIDE : bwtlen / KJ_LETTERS_PER_WORD + 2; }
#define KJ_MAX_ALEN 24
#define KJ_MAX_IDS 21              // max_match_ids = 20 -> the set holds at most 21 (ConsumerThread.cpp:805)
#define KJ_MAX_BEST_SI 20          // max_matches_SI (Config.hpp:35)
#define KJ_TAX_BAD 0xffffffffu     // "bad number" database name (ConsumerThread.cpp:817-820): skipped
#define KJ_MAX_MM 8                // max supported -e
#define KJ_SEG_WINDOW 12
#define KJ_KEPT_SMEM 20            // winners kept in shared memory before spilling = max_matches_SI (20): greedy keeps its best list there

// wide records: hdr = cnt (40 bit: C[c] + #c before the block) | popc(w0) << 40 | (popc(w0)+popc(w1)) << 48 ; w0..w2 = one-hot bitmap.
#define KJ_CNT_MASK 0xffffffffffull
#define KJ_P1_SHIFT 40
#define KJ_P2_SHIFT 48

struct KjKmer { uint64_t lo, hi; };    // SA interval of a k-mer (empty if lo >= hi), indexes >= 2^32
struct KjKmer32 { uint32_t lo, hi; };  // same, for indexes with bwtlen < 2^32

struct KjTables {
    uint8_t codon_aa[64];            // (n0<<4|n1<<2|n2) -> alphabet index, 0 = stop  (ConsumerThread.cpp:117-181 + sequence.c:68-97)
    int8_t b62[KJ_MAX_ALEN][KJ_MAX_ALEN];   // BLOSUM62 indexed by ALPHABET index        (ConsumerThread.cpp:88-107)
    uint8_t subst[KJ_MAX_ALEN][20];  // substitution try-order per residue, alphabet indices (ConsumerThread.cpp:10-30)
    int32_t seg_logfix[KJ_SEG_WINDOW + 1];  // round(2^24 log2(12/c)) : entropy of a 12-window in fixed point
    int32_t seg_locut_fix, seg_hicut_fix;   // 12*2.2*2^24, 12*2.5*2^24 (margins checked on host against FP64)
    char letters[KJ_MAX_ALEN];       // alphabet index -> letter (fragment strings of the verbose output)
    uint8_t aa_index[32];            // protein input: upper-case letter - 'A' -> alphabet index, 0 = splits the read (ConsumerThread.cpp:664)
};

// compact tiered layout: records [nb_dev, nb) start at `host` (the device alias of mapped pinned host memory), record b at host + (b - nb_dev) * 16
struct KjTierRef { const uint64_t* host; uint64_t nb_dev; };
// compact spread layout: segment g holds records [first[g], first[g+1]) from base[g] on (a device address in the HBM of the group's g-th device);
// first[] does not decrease, and the slots g >= n hold first[g] = ~0 (never selected) and base[g] = null
struct KjSpreadRef { const uint64_t* base[KJ_MAX_GROUP]; uint64_t first[KJ_MAX_GROUP]; uint32_t n, pad; };
// (the 32-bit members are paired so that the descriptor has no padding holes: the kernels stage it in shared memory next to the work spaces)
struct KjDevIndex {
    const uint64_t* rank; uint64_t nb;          // [alen][nb] records of 2 (narrow) or 4 (wide) 64-bit words; compact: [nb] records of 16 words
                                                // (compact tiered: records [0, tier.nb_dev) only; compact spread: segment 0)
    union {
        const uint64_t* rank_base[KJ_MAX_ALEN]; // narrow, wide: records of letter c (saves the multiply in the inner loop)
        KjTierRef tier;                         // compact tiered: where records [nb_dev, nb) are (the compact layouts do not use rank_base)
        KjSpreadRef spread;                     // compact spread: the segment table
    };
    union {
        const uint64_t* letters;                // narrow, wide: the packed letters
        const uint64_t* csb;                    // compact: [superblock][KJ_CSB_STRIDE] C[c] + #c before the superblock
    };
    uint64_t bwtlen; int alen; uint32_t nseq;
    uint64_t C[KJ_MAX_ALEN + 1];                // C[c] = first SA row of letter c; C[alen] = bwtlen
    const uint32_t* sa_tax; const uint32_t* seq_tax;
    const uint32_t* sa_acc; const uint32_t* seq_acc;     // accession rank per sampled suffix / sequence (NULL unless the index view carried seq_accession)
    uint64_t sa_check; int sa_exp; int64_t sa_bias; uint64_t n_sa;
    const uint32_t* row_tax;                    // taxon of every BWT row, = the SA walk's result (narrow indexes that have room for it; NULL = walk)
    const uint32_t* tax_parent; const uint32_t* tax_depth; const uint64_t* tax_id; uint32_t n_tax; int n_lnfact;
    const double* lnfact;
    const void* kmer; int kmer_k;               // direct-address table of k-mer intervals (KjKmer32 if !wide else KjKmer; 0 = off)
    int wide;                                   // layout code: 0 narrow (32-bit interval kernels), 1 wide, 2 compact, 3 compact tiered, 4 compact spread (64-bit interval kernels)
    int mono;                                   // 1: true FM index (match starts monotone in the end position); 0: the reference's checkpoint quirk applies (no chain bounds)
    uint64_t quirk_lo; const uint64_t* quirk_d;         // rows k >= quirk_lo: FMindex(c,k) -= quirk_d[c] (reference checkpoint quirk, ~0 = none; [KJ_MAX_ALEN] in global memory)
    const KjTables* tables;
};
// The tier reference shares rank_base's bytes: the descriptor keeps the size and member offsets the shared-memory carve-up and the launch
// geometry of every kernel were derived from.
static_assert(sizeof(KjTierRef) <= sizeof(const uint64_t*) * KJ_MAX_ALEN && sizeof(KjDevIndex) == 592 && offsetof(KjDevIndex, rank_base) == 16 &&
              offsetof(KjDevIndex, tier) == 16 && offsetof(KjDevIndex, letters) == 208 && offsetof(KjDevIndex, tables) == 584, "KjDevIndex layout changed");
static_assert(sizeof(KjSpreadRef) == 136 && sizeof(KjSpreadRef) <= sizeof(const uint64_t*) * KJ_MAX_ALEN && offsetof(KjDevIndex, spread) == 16,
              "the segment table must fit in rank_base's bytes");

struct KjRunParams {
    int mode;                       // 0 MEM, 1 GREEDY
    uint32_t m, e, min_score, seed_length;
    int use_evalue, seg, protein, name_mode;
    // E-value gate as an integer threshold: ev_breaks[k] = the largest query length (double) for which score k passes,
    // so the minimal passing score of a read is the number of breaks below its query length (kj_build_evalue_breaks)
    const double* ev_breaks; uint32_t n_ev_breaks;
    // per-warp scratch geometry
    uint32_t max_len;               // longest read (bases) in the batch, rounded up
    uint32_t max_frag;              // longest fragment (residues)
    uint32_t item_cap;              // fragment-queue capacity per warp
    uint32_t kept_cap_smem;         // winners kept in shared memory before spilling
    uint32_t scratch_entries;       // global spill entries per warp
    uint32_t variant_cap;           // Greedy: entries of the per-warp substituted-variant ring
    uint32_t ws_global;             // 1: the per-warp work space lives in global memory (reads too long for shared memory)
};
