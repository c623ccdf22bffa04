// kj_host.h -- host side of the boundary: .fmi / nodes.dmp loaders (the on-disk formats are the input
// contract, SURVEY.md 8a row 14) and the transcoder from the reference's in-memory index to the device
// layout of kj_layout.h.  Pure C++ (no CUDA) so the test emulator can share it.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/kaiju_b200.h"
#include "kj_layout.h"

struct kj_fmi {
    int64_t len = 0; int32_t nseq = 0, alen = 0; std::string alphabet;
    int64_t sa_len = 0, ncheck = 0; int32_t chpt_exp = 0, nbytes = 0, sbits = 0, pbits = 0; int64_t mask = 0, check = 0;
    std::vector<std::string> ids; std::vector<uint64_t> seq_taxon; std::vector<uint8_t> sa;
    std::vector<uint32_t> seq_acc; std::vector<std::string> acc_names;       // accession rank per sequence (0xffffffff = none), distinct accessions sorted
    int64_t bwtlen = 0; int32_t N1 = 0, N2 = 0; std::vector<uint8_t> bwt; std::vector<int32_t> startLcode;
};
struct kj_nodes { std::vector<uint64_t> node, parent; };

// device-layout arrays, built on the host
struct KjHostIndex {
    std::vector<uint64_t> rank; uint64_t nb = 0;   // [alen][nb] records of kj_rank_words(wide) words over kj_rank_rows(wide) rows
    std::vector<uint64_t> letters;
    uint64_t bwtlen = 0; int alen = 0; uint64_t C[KJ_MAX_ALEN + 1] = {0};
    std::vector<uint32_t> sa_tax, seq_tax;
    std::vector<uint32_t> sa_acc, seq_acc;      // accession rank per sampled suffix / per sequence (only when the view carries seq_accession)
    uint64_t sa_check = 0; int sa_exp = 0; int64_t sa_bias = 0; uint32_t nseq = 0;
    std::vector<uint32_t> tax_parent, tax_depth; std::vector<uint64_t> tax_id; uint32_t n_present = 0;   // tax_id = [ids of nodes.dmp, ascending | DB taxa absent from it, ascending]
    std::vector<double> lnfact;
    std::vector<KjKmer> kmer; std::vector<KjKmer32> kmer32; int kmer_k = 0; int wide = 0;   // k-mer suffix intervals (letters 1..20)
    KjTables tables;
    double db_length = 0;          // bwt.len - bwt.nseq (Config.cpp:20)
    uint64_t quirk_lo = ~0ull, quirk_d[KJ_MAX_ALEN] = {0};   // the reference's checkpoint quirk for bwtlen = m * 2^16, m >= 2 (kj_build_host_index)
};

std::string& kj_err();             // thread-local last error text
uint64_t kj_mix_bytes(uint64_t h, const void* p, size_t n);   // order-sensitive 64-bit checksum (index files, test hooks)
int kj_build_host_index(const kj_index_view& v, const kj_taxonomy_view& t, KjHostIndex& out);
// the small / BWT-independent part only (the large arrays are then built on the device, kj_build.h); lcode = byte code -> letter
int kj_build_host_meta(const kj_index_view& v, const kj_taxonomy_view& t, uint32_t copies, KjHostIndex& out, uint8_t lcode[256]);
// FMindex(c, k) on the transcoder's arrays (any layout, the checkpoint quirk applied): the CPU reference of the device rank query
uint64_t kj_host_rank(const KjHostIndex& H, uint32_t c, uint64_t k);
// SA intervals of all 20^k k-mers over the 20 residue letters (exactness-preserving shortcut for the first k LF steps)
void kj_build_kmer_table(KjHostIndex& H, int k);
// k of the k-mer interval table: 6 letters (20^6 entries, 0.5-1 GB) once the index is large enough that 6-mers are mostly present
// (faster for MEM on the 2e8-row index in an A/B run), 5 letters (26-51 MB) below that
static inline int kj_default_kmer_k(uint64_t bwtlen) { return bwtlen >= 50000000ull ? 6 : 5; }
// device-native index file (SURVEY.md 8f-4): the transcoded arrays as they are uploaded, so that loading is one sequential read
int kj_host_index_write(const KjHostIndex& H, const char* path);
int kj_host_index_read(const char* path, KjHostIndex& H);
int kj_check_params(const kj_params& p);
// E-value gate (ConsumerThread.cpp:500-513) as the minimal passing integer score per (len1,len2)
int kj_build_evalue_breaks(const kj_params& p, double db_length, std::vector<double>& breaks);
// per-warp scratch geometry for a batch whose longest mate has max_len bases
void kj_fill_run_params(const kj_params& p, uint32_t max_len, KjRunParams& rp);
#define KJ_LNFACT_REF 10001                                  // entries of the reference's ln(n!) table (blast_seg.c:53-1306)
#define KJ_LNFACT_LEN (KJ_MAX_LONG_READ_LEN / 3 + 16)        // ln(n!) for every SEG region length of a KJ_MAX_LONG_READ_LEN read
void kj_lnfact_table(std::vector<double>& t);
