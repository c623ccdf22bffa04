// kj_device.cu -- CUDA side of libkaijub200.so: index upload, the persistent classification kernel and the
// C ABI entry points kj_create / kj_classify / kj_classify_device / kj_destroy (include/kaiju_b200.h).
//
// Execution model: one warp classifies one read item at a time (kj_core.h); a persistent grid of
// (#SM x resident CTAs) pulls read indices from a global counter, so fast ("U" after the length gate)
// and slow (long matches, SEG trims) reads balance without a host-side scheduler -- the GPU replacement of
// the reference's ProducerConsumerQueue + N ConsumerThreads (kaiju.cpp:250-257, 288-396).
// There is no CPU fallback: without a GPU kj_create() fails with KJ_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "kj_core.h"
#include "kj_core_greedy.h"
#include "kj_host.h"

#define KJ_WARPS_PER_CTA 8
#define KJ_MIN_BLOCKS 4          // resident CTAs per SM the register allocation is tuned for (the search is latency-bound; on an H100 (400 W) 4 beat 3 CTAs, 50.6 vs 46.5 M pairs/s MEM)
#define KJ_MIN_BLOCKS_GREEDY_SPLIT 4   // front-end / search kernels of the two-kernel Greedy path: on an H100 (400 W) 4 CTAs (64 registers) beat 5 (48), 13.8 vs 12.9 M pairs/s
#define KJ_MIN_BLOCKS_GREEDY 4   // 5 CTAs (48 registers) was slower in an A/B run: more warps, but more spill traffic and more instruction-fetch stalls
#define KJ_CLAIM 4               // read items claimed per atomic by a warp
#define KJ_CHUNK_READS (1u << 20)
#define KJ_CHUNK_BYTES (1ull << 28)  // and at most this many bases of one mate per chunk (long reads)
#define KJ_LONG_GAP 4096u        // short reads in a row that end a chunk of the long-read kernels (kj_classify: fewer run with it)

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { kj_err() = std::string(#call) + ": " + cudaGetErrorString(e_); return KJ_ERR_CUDA; } } while (0)

struct KjCtaShared { KjDevIndex ix; KjTables tb; };

// GWS = false: the per-warp work space is carved out of shared memory (the compiler keeps every access in the shared
// address space); GWS = true (reads too long for that): the same carve-up in a global buffer, generic loads and stores.
// FIX = true: the work-space carve-up of the standard short-read case (mates up to 152 bases, -m 11) as compile-time constants: every offset
// becomes an immediate of the shared-memory instructions instead of a value that is kept in (or re-derived into) registers.
static __host__ __device__ __forceinline__ KjRunParams kj_fixed_profile(int mode) {
    KjRunParams p{}; p.mode = mode; p.m = 11; p.max_len = 152; p.max_frag = 152 / 3 + 1; p.item_cap = 128; p.kept_cap_smem = KJ_KEPT_SMEM;
    return p;
}
// VB = true: the verbose outputs (id sets, accession sets, fragment strings) are compiled in; the kernels of the normal path carry none of it.
// ROLE: 0 = the whole item in this kernel; 1 = front end only (translation, fragments, ranked queue -> a record per item in `prep`); 2 = search only (from the records).
// Greedy runs as the pair 1 + 2 over sub-batches of the launch (kj_core.h: the search loop then shares the instruction cache with nothing it does not need).
// LONG = true: the long-read kernels (kj_classify_long_kernel; the work space in global memory, the general profile, ROLE 0).
#define KJ_CLASSIFY_PARAMS const KjDevIndex* __restrict__ g_ix, const __grid_constant__ KjRunParams rp, const __grid_constant__ KjSmemLayout lay, \
                   const uint8_t* __restrict__ seq1, const uint64_t* __restrict__ off1, \
                   const uint8_t* __restrict__ seq2, const uint64_t* __restrict__ off2, \
                   uint64_t base1, uint64_t base2, uint64_t n_reads, \
                   uint64_t* __restrict__ taxon_out, uint32_t* __restrict__ best_out, uint64_t* __restrict__ ids_out, uint8_t* __restrict__ nids_out, uint32_t* __restrict__ compact_out, \
                   unsigned long long* __restrict__ counter, KjKept* __restrict__ spill, uint8_t* __restrict__ gscratch, \
                   uint32_t gscratch_bytes, uint8_t* __restrict__ gws, unsigned long long* __restrict__ counts, uint32_t* __restrict__ err, \
                   uint32_t* __restrict__ acc_out, uint8_t* __restrict__ nacc_out, char* __restrict__ frag_out, uint32_t frag_stride, uint32_t* __restrict__ frag_len_out, \
                   uint8_t* __restrict__ prep, uint32_t prep_stride, uint64_t r_begin
#define KJ_CLASSIFY_ARGS g_ix, rp, lay, seq1, off1, seq2, off2, base1, base2, n_reads, taxon_out, best_out, ids_out, nids_out, compact_out, counter, spill, gscratch, \
                   gscratch_bytes, gws, counts, err, acc_out, nacc_out, frag_out, frag_stride, frag_len_out, prep, prep_stride, r_begin
template <int MODE, class IdxT, bool GWS, bool FIX, bool VB, int ROLE, bool LONG>
static __device__ __forceinline__ void kj_classify_body(const KjDevIndex* __restrict__ g_ix, const KjRunParams& rp, const KjSmemLayout& lay,
                   const uint8_t* __restrict__ seq1, const uint64_t* __restrict__ off1,
                   const uint8_t* __restrict__ seq2, const uint64_t* __restrict__ off2,
                   uint64_t base1, uint64_t base2, uint64_t n_reads,
                   uint64_t* __restrict__ taxon_out, uint32_t* __restrict__ best_out, uint64_t* __restrict__ ids_out, uint8_t* __restrict__ nids_out, uint32_t* __restrict__ compact_out,
                   unsigned long long* __restrict__ counter, KjKept* __restrict__ spill, uint8_t* __restrict__ gscratch,
                   uint32_t gscratch_bytes, uint8_t* __restrict__ gws, unsigned long long* __restrict__ counts, uint32_t* __restrict__ err,
                   uint32_t* __restrict__ acc_out, uint8_t* __restrict__ nacc_out, char* __restrict__ frag_out, uint32_t frag_stride, uint32_t* __restrict__ frag_len_out,
                   uint8_t* __restrict__ prep, uint32_t prep_stride, uint64_t r_begin) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    KjCtaShared* sh = (KjCtaShared*)smem_raw;
    {   // stage the index descriptor (C[] etc.) and the small tables once per CTA
        const uint32_t* src = (const uint32_t*)g_ix; uint32_t* dst = (uint32_t*)&sh->ix;
        KJ_ROLLED
        for (uint32_t i = threadIdx.x; i < sizeof(KjDevIndex) / 4; i += blockDim.x) dst[i] = src[i];
        const uint32_t* ts = (const uint32_t*)g_ix->tables; uint32_t* td = (uint32_t*)&sh->tb;
        KJ_ROLLED
        for (uint32_t i = threadIdx.x; i < sizeof(KjTables) / 4; i += blockDim.x) td[i] = ts[i];
    }
    __syncthreads();
    const int warp_in_cta = threadIdx.x >> 5;
    KjWarpCtx cx;
    cx.w.lane = threadIdx.x & 31;
    cx.ix = &sh->ix; cx.rp = &rp; cx.tb = &sh->tb;
    if (FIX) cx.L = kj_smem_layout(kj_fixed_profile(MODE));      // folded at compile time
    else cx.L = lay;                                 // computed on the host, read from the parameter bank
    const uint64_t gwarp = (uint64_t)blockIdx.x * KJ_WARPS_PER_CTA + (uint64_t)warp_in_cta;
    // per-warp work space: shared memory, or (reads too long for it) a slice of a global buffer that stays L1/L2-resident
    if (GWS) cx.smem = gws + gwarp * cx.L.total;
    else cx.smem = smem_raw + kj_align((uint32_t)sizeof(KjCtaShared), 16) + (uint32_t)warp_in_cta * cx.L.total;
    cx.spill = spill + gwarp * rp.scratch_entries;
    cx.gscratch = gscratch + gwarp * gscratch_bytes;
    cx.err = err; cx.text = nullptr; cx.text_cap = frag_stride; cx.text_len = 0; cx.want_acc = VB && acc_out != nullptr;
    const bool paired = seq2 != nullptr;
    // work distribution: a warp claims KJ_CLAIM consecutive items per atomic and fetches their offsets with one coalesced load
    KJ_ROLLED
    for (;;) {
        unsigned long long r0 = 0;
        if (cx.w.lane == 0) r0 = r_begin + atomicAdd(counter, (unsigned long long)KJ_CLAIM);      // this launch covers items [r_begin, n_reads)
        r0 = cx.w.shfl64(r0, 0);
        if (r0 >= n_reads) break;
        const unsigned long long ri = r0 + (unsigned long long)cx.w.lane;
        uint64_t o1 = 0, o2 = 0;
        if (cx.w.lane <= KJ_CLAIM && ri <= n_reads) { o1 = off1[ri] - base1; if (paired) o2 = off2[ri] - base2; }
        KJ_ROLLED
        for (int k = 0; k < KJ_CLAIM; k++) {
            const unsigned long long r = r0 + (unsigned long long)k;
            if (r >= n_reads) break;
            const uint64_t a0 = cx.w.shfl64(o1, k), a1 = cx.w.shfl64(o1, k + 1), b0 = cx.w.shfl64(o2, k), b1 = cx.w.shfl64(o2, k + 1);
            const uint8_t* p1 = seq1 + a0;
            const uint8_t* p2 = paired ? seq2 + b0 : nullptr;
            uint32_t best = 0;
            if (VB && frag_out) { cx.text = frag_out + r * frag_stride; cx.text_len = 0; }
            uint32_t t = kj_classify_item<MODE, IdxT, ROLE, LONG>(cx, p1, (int)(a1 - a0), p2, (int)(b1 - b0), paired, best, ROLE ? prep + (size_t)(r - r_begin) * prep_stride : nullptr);
            if (ROLE == 1) { cx.w.sync(); continue; }
            const uint64_t id = t == KJ_TAX_BAD ? 0ull : sh->ix.tax_id[t];
            if (cx.w.lane == 0) {
                if (taxon_out) taxon_out[r] = id;
                if (compact_out) compact_out[r] = id ? t : KJ_TAX_BAD;
                if (best_out) best_out[r] = id ? best : 0u;
                // per-taxon read counts (kaiju2table's first pass), fused: a separate counting kernel behind a persistent grid would stall the chunk pipeline
                if (counts) atomicAdd(counts + (id ? t : sh->ix.n_tax), 1ull);
            }
            if (VB && ids_out) {   // column 5 of the reference's -v output: the match-id set in ascending order (std::set), classified reads only
                const uint32_t nids = id ? cx.nids : 0u; const uint32_t* ids = (const uint32_t*)(cx.smem + cx.L.ids_off);
                if ((uint32_t)cx.w.lane < nids) {
                    const uint64_t mine = sh->ix.tax_id[ids[cx.w.lane]]; uint32_t rank = 0;
                    KJ_ROLLED
                    for (uint32_t u = 0; u < nids; u++) rank += sh->ix.tax_id[ids[u]] < mine ? 1u : 0u;
                    ids_out[r * KJ_MAX_IDS + rank] = mine;
                }
                if (cx.w.lane == 0) nids_out[r] = (uint8_t)nids;
            }
            if (VB && acc_out) {   // column 6: accession ranks of the visited sequences, ascending (the reference's std::set<std::string> order)
                const uint32_t* accs = (const uint32_t*)(cx.smem + cx.L.accs_off); const uint32_t nacc = id ? accs[20] : 0u;
                if ((uint32_t)cx.w.lane < nacc) {
                    const uint32_t mine = accs[cx.w.lane]; uint32_t rank = 0;
                    KJ_ROLLED
                    for (uint32_t u = 0; u < nacc; u++) rank += accs[u] < mine ? 1u : 0u;
                    acc_out[r * KJ_MAX_MATCH_ACC + rank] = mine;
                }
                if (cx.w.lane == 0) nacc_out[r] = (uint8_t)nacc;
            }
            if (VB && frag_len_out && cx.w.lane == 0) frag_len_out[r] = id ? cx.text_len : 0u;
            cx.w.sync();
        }
    }
}
template <int MODE, class IdxT, bool GWS, bool FIX, bool VB, int ROLE>
__global__ void __launch_bounds__(KJ_WARPS_PER_CTA * 32, MODE == 0 ? KJ_MIN_BLOCKS : ROLE != 0 ? KJ_MIN_BLOCKS_GREEDY_SPLIT : KJ_MIN_BLOCKS_GREEDY)
kj_classify_kernel(KJ_CLASSIFY_PARAMS) { kj_classify_body<MODE, IdxT, GWS, FIX, VB, ROLE, false>(KJ_CLASSIFY_ARGS); }
// mates longer than KJ_MAX_READ_LEN (kj_set_max_read_len): wide fields (kj_core.h KjW<true>); same signature, so the host launches it like the others
template <int MODE, class IdxT, bool VB>
__global__ void __launch_bounds__(KJ_WARPS_PER_CTA * 32, MODE == 0 ? KJ_MIN_BLOCKS : KJ_MIN_BLOCKS_GREEDY)
kj_classify_long_kernel(KJ_CLASSIFY_PARAMS) { kj_classify_body<MODE, IdxT, true, false, VB, 0, true>(KJ_CLASSIFY_ARGS); }

// Every instantiation has the same signature: the host picks one per launch (kj_select_kernel), sets it up and launches it through the pointer.
using KjKernel = decltype(&kj_classify_kernel<0, uint32_t, false, false, false, 0>);
// The fixed profile and the two-kernel pair exist for Greedy only (kj_use_fixed, launch()); neither applies to the verbose kernels or to a work space in global memory.
template <int MODE, class T>
static KjKernel kj_select_kernel_t(bool gws, bool fixed, bool verbose, int role) {
    if (verbose) return gws ? kj_classify_kernel<MODE, T, true, false, true, 0> : kj_classify_kernel<MODE, T, false, false, true, 0>;
    if (gws) return kj_classify_kernel<MODE, T, true, false, false, 0>;
    if constexpr (MODE == 1) {
        if (fixed) return role == 1 ? kj_classify_kernel<1, T, false, true, false, 1> : role == 2 ? kj_classify_kernel<1, T, false, true, false, 2> : kj_classify_kernel<1, T, false, true, false, 0>;
        if (role) return role == 1 ? kj_classify_kernel<1, T, false, false, false, 1> : kj_classify_kernel<1, T, false, false, false, 2>;
    }
    return kj_classify_kernel<MODE, T, false, false, false, 0>;
}
template <int MODE, class T>
static KjKernel kj_select_long_kernel_t(bool verbose) { return verbose ? kj_classify_long_kernel<MODE, T, true> : kj_classify_long_kernel<MODE, T, false>; }
// layout: 0 narrow (32-bit intervals), 1 wide, 2 compact, 3 compact tiered, 4 compact spread (64-bit intervals; kj_layout.h).  long_reads: the batch holds mates longer than
// KJ_MAX_READ_LEN (only the work space in global memory, the general profile and ROLE 0 exist for them).
static KjKernel kj_select_kernel(int mode, int layout, bool gws, bool fixed, bool verbose, int role, bool long_reads = false) {
    if (long_reads) {
        if (layout == KJ_LAYOUT_COMPACT_SPREAD) return mode == 0 ? kj_select_long_kernel_t<0, KjSpreadIdx>(verbose) : kj_select_long_kernel_t<1, KjSpreadIdx>(verbose);
        if (layout == KJ_LAYOUT_COMPACT_TIERED) return mode == 0 ? kj_select_long_kernel_t<0, KjTieredIdx>(verbose) : kj_select_long_kernel_t<1, KjTieredIdx>(verbose);
        if (layout == KJ_LAYOUT_COMPACT) return mode == 0 ? kj_select_long_kernel_t<0, KjCompactIdx>(verbose) : kj_select_long_kernel_t<1, KjCompactIdx>(verbose);
        if (mode == 0) return layout ? kj_select_long_kernel_t<0, uint64_t>(verbose) : kj_select_long_kernel_t<0, uint32_t>(verbose);
        return layout ? kj_select_long_kernel_t<1, uint64_t>(verbose) : kj_select_long_kernel_t<1, uint32_t>(verbose);
    }
    if (layout == KJ_LAYOUT_COMPACT_SPREAD) return mode == 0 ? kj_select_kernel_t<0, KjSpreadIdx>(gws, fixed, verbose, role) : kj_select_kernel_t<1, KjSpreadIdx>(gws, fixed, verbose, role);
    if (layout == KJ_LAYOUT_COMPACT_TIERED) return mode == 0 ? kj_select_kernel_t<0, KjTieredIdx>(gws, fixed, verbose, role) : kj_select_kernel_t<1, KjTieredIdx>(gws, fixed, verbose, role);
    if (layout == KJ_LAYOUT_COMPACT) return mode == 0 ? kj_select_kernel_t<0, KjCompactIdx>(gws, fixed, verbose, role) : kj_select_kernel_t<1, KjCompactIdx>(gws, fixed, verbose, role);
    if (mode == 0) return layout ? kj_select_kernel_t<0, uint64_t>(gws, fixed, verbose, role) : kj_select_kernel_t<0, uint32_t>(gws, fixed, verbose, role);
    return layout ? kj_select_kernel_t<1, uint64_t>(gws, fixed, verbose, role) : kj_select_kernel_t<1, uint32_t>(gws, fixed, verbose, role);
}

__global__ void kj_maxlen_kernel(const uint64_t* __restrict__ off, uint64_t n, unsigned int* __restrict__ out) {
    unsigned int m = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) { uint64_t l = off[i + 1] - off[i]; m = max(m, (unsigned int)min(l, (uint64_t)0xffffffffu)); }
    for (int s = 16; s > 0; s >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, s));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// Per-taxon read counts (the input of kaiju2table, src/kaiju2table.cpp:186-245): dense index of each result by binary search in the
// two ascending runs of tax_id (nodes.dmp ids | DB taxa absent from it); slot n_tax = unclassified.
__global__ void kj_count_kernel(const uint64_t* __restrict__ taxon, uint64_t n, const uint64_t* __restrict__ tax_id, uint32_t n_present, uint32_t n_tax,
                                unsigned long long* __restrict__ counts) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t id = taxon[r]; uint32_t slot = n_tax;
        if (id) {
            uint32_t lo = 0, hi = n_present;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (tax_id[mid] < id) lo = mid + 1; else hi = mid; }
            if (lo < n_present && tax_id[lo] == id) slot = lo;
            else { lo = n_present; hi = n_tax; while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (tax_id[mid] < id) lo = mid + 1; else hi = mid; } if (lo < n_tax && tax_id[lo] == id) slot = lo; }
        }
        atomicAdd(counts + slot, 1ull);
    }
}
__global__ void kj_count_commit(unsigned long long* __restrict__ total, unsigned long long* __restrict__ pending, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { total[i] += pending[i]; pending[i] = 0; }
}

// ------------------------------------------------------------------------------------------------
// The owner of every device allocation of the library: move-only, freed by its destructor (or early by reset()).
struct KjDevBuf {
    void* p = nullptr; size_t cap = 0;
    KjDevBuf() = default;
    KjDevBuf(const KjDevBuf&) = delete; KjDevBuf& operator=(const KjDevBuf&) = delete;
    KjDevBuf(KjDevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    KjDevBuf& operator=(KjDevBuf&& o) noexcept { if (this != &o) { reset(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; } return *this; }
    ~KjDevBuf() { reset(); }
    void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    // room for `need` bytes: only when the capacity is smaller, the buffer is freed and `alloc` (>= need) bytes are allocated
    int grow(size_t need, size_t alloc) {
        if (need <= cap) return KJ_OK;
        reset(); void* q = nullptr; CK(cudaMalloc(&q, alloc)); p = q; cap = alloc; return KJ_OK;
    }
    int grow(size_t need) { return grow(need, need); }
    template <class T> T* as() const { return (T*)p; }
};

// The host-side counterpart of KjDevBuf: pinned host memory mapped into the device's address space (the host tier of kj_create_tiered).
// `p` is the host address, `d` the device alias the kernels read it through.  Move-only, freed by its destructor.
struct KjHostBuf {
    void* p = nullptr; void* d = nullptr; size_t cap = 0;
    KjHostBuf() = default;
    KjHostBuf(const KjHostBuf&) = delete; KjHostBuf& operator=(const KjHostBuf&) = delete;
    KjHostBuf(KjHostBuf&& o) noexcept : p(o.p), d(o.d), cap(o.cap) { o.p = o.d = nullptr; o.cap = 0; }
    KjHostBuf& operator=(KjHostBuf&& o) noexcept { if (this != &o) { reset(); p = o.p; d = o.d; cap = o.cap; o.p = o.d = nullptr; o.cap = 0; } return *this; }
    ~KjHostBuf() { reset(); }
    void reset() { if (p) cudaFreeHost(p); p = d = nullptr; cap = 0; }
    int grow(size_t need) {
        if (need <= cap) return KJ_OK;
        reset(); void* q = nullptr; CK(cudaHostAlloc(&q, need, cudaHostAllocMapped)); p = q; cap = need;
        void* dq = nullptr; CK(cudaHostGetDevicePointer(&dq, q, 0)); d = dq; return KJ_OK;
    }
    template <class T> T* as() const { return (T*)d; }
};
// Makes `dev` the current device for its lifetime and restores the previous one (dev < 0: changes nothing).  The arrays of a group
// (kj_create_group) are allocated, written and freed with the device that holds them current.
struct KjDevGuard {
    int prev = -1;
    explicit KjDevGuard(int dev) { if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~KjDevGuard() { if (prev >= 0) cudaSetDevice(prev); }
    KjDevGuard(const KjDevGuard&) = delete; KjDevGuard& operator=(const KjDevGuard&) = delete;
};
// An index array the placement of kj_create_tiered may move to the host tier (kj_choose_layout sets on_host before it is allocated): in HBM or
// in mapped pinned host memory, read by the kernels through `p` either way.  device >= 0: in the HBM of that device (a suffix-array array of a
// group, placed by kj_plan_group), read by the group's other devices over peer access.
struct KjTierBuf {
    KjDevBuf dev; KjHostBuf host; bool on_host = false; void* p = nullptr; int device = -1;
    int grow(size_t need) { KjDevGuard g(device); const int rc = on_host ? host.grow(need) : dev.grow(need); p = on_host ? host.d : dev.p; return rc; }
    template <class T> T* as() const { return (T*)p; }
    size_t cap() const { return on_host ? host.cap : dev.cap; }
    // bytes [off, off + n) = val; the host tier is written by the CPU (nothing on the device writes it at this point)
    int fill(size_t off, int val, size_t n) { KjDevGuard g(device); if (on_host) memset((char*)host.p + off, val, n); else CK(cudaMemset((char*)dev.p + off, val, n)); return KJ_OK; }
    int put(const void* src, size_t n) { KjDevGuard g(device); if (on_host) memcpy(host.p, src, n); else CK(cudaMemcpy(dev.p, src, n, cudaMemcpyHostToDevice)); return KJ_OK; }
    void reset() { KjDevGuard g(device); dev.reset(); host.reset(); p = nullptr; }
};

// The index a group of contexts shares (kj_create_group, layout 4): the record segments, each in the HBM of its group member's device, and the
// suffix-array arrays, each whole on the device kj_plan_group chose.  Every context of the group holds a shared_ptr to it; the last kj_destroy
// frees every array with its owning device current.
struct KjGroup {
    int n = 0; int dev[KJ_MAX_GROUP] = {0};         // group member g: its device, and segment g = records [first[g], first[g + 1]) in seg[g]
    uint64_t first[KJ_MAX_GROUP + 1] = {0};
    KjDevBuf seg[KJ_MAX_GROUP];
    KjSpreadRef ref{};                              // the segment table of the descriptors (kj_group_alloc)
    KjTierBuf sa_tax, seq_tax, sa_acc, seq_acc;     // moved here from the first context once the construction has written them
    KjGroup() = default; KjGroup(const KjGroup&) = delete; KjGroup& operator=(const KjGroup&) = delete;
    ~KjGroup() {
        for (int g = 0; g < n; g++) { KjDevGuard d(dev[g]); seg[g].reset(); }
        for (KjTierBuf* b : {&sa_tax, &seq_tax, &sa_acc, &seq_acc}) b->reset();
    }
};

// One of the two pipeline slots (the chunks of kj_classify, the lanes of kj_classify_files): staging, outputs, scratch, streams.
// Two slots may be in flight, and their launches may have different run parameters (kj_classify_files derives them from each batch's longest
// read): each slot has its own scratch, sized and grown from that slot's launches alone.  Carving both slots out of one buffer at offsets
// computed from the current launch's parameters would let a launch with a smaller per-warp size land inside the region the other slot's
// kernel is still using.  A slot's buffers are only replaced when its own previous work is complete; the cudaFree of the old buffer also
// waits for the other slot's kernels.
// Within one slot, the front-end kernel of the two-kernel Greedy path (ROLE 1) runs beside the search kernel (ROLE 2) of the previous
// sub-batch; it touches neither the spill entries nor the variant ring (translation, queue ranking and the record store only use the
// shared-memory work space), and the split path never uses the global work space, so the two share the slot's scratch safely.
struct KjSlot {
    KjDevBuf seq[2], off[2];                                        // staging of kj_classify (host buffers), one per mate
    KjDevBuf tax, best, ids, nids, acc, nacc, frag, fraglen;        // outputs of a chunk
    KjDevBuf spill, gscratch, ws;                                   // per-warp global scratch: spill entries, Greedy variant ring, work space of long reads
    bool long_scratch = false;                                      // the scratch was sized by a launch of the long-read kernels (released by the next other launch)
    cudaStream_t stream = nullptr, fstream = nullptr;               // the slot's stream, and the front-end stream of the two-kernel Greedy path
    cudaEvent_t ev_in = nullptr, ev_f[2] = {nullptr, nullptr}, ev_s[2] = {nullptr, nullptr};     // hand-over events between the two
};

struct KjFilesState; static void kj_files_state_free(KjFilesState* S);      // kj_ingest.h
struct kj_ctx {
    std::unique_ptr<KjFilesState, void (*)(KjFilesState*)> files{nullptr, kj_files_state_free};   // buffers of kj_classify_files, kept between calls
    int device = 0; kj_params params{}; int sm_count = 0;
    KjHostIndex H;                 // big arrays are released after upload; small ones stay
    KjDevIndex dix{};              // host copy of the descriptor (device pointers inside)
    KjDevBuf ix, tables;
    KjDevBuf ix_mem, kmer_mem; int kmer_k_mem = 0;      // the MEM kernels' own descriptor: same index, 7-mer table (kj_create)
    KjDevBuf rank, letters, tax_parent, tax_depth, tax_id, lnfact, kmer;    // compact layout: `letters` holds the superblock table
    KjTierBuf sa_tax, seq_tax, sa_acc, seq_acc;     // in HBM, or in the host tier of a kj_create_tiered context
    KjHostBuf rank_host; uint64_t nb_dev = 0;       // compact tiered layout: records [nb_dev, nb) in the host tier, records [0, nb_dev) in `rank`
    std::shared_ptr<KjGroup> group;                 // compact spread layout: the records and suffix-array arrays the group shares (`rank` and the
                                                    // suffix-array members above stay empty; the superblock and k-mer tables are this context's own)
    KjDevBuf row_tax;              // taxon per BWT row (kj_device_build_row_tax; empty: the kernels walk)
    KjTierBuf out_str[2], out_off[2]; uint64_t out_n[2] = {0, 0}, out_bytes[2] = {0, 0}; bool out_have[2] = {false, false};   // kj_set_output_strings, by kind
    uint64_t index_bytes = 0, host_bytes = 0; uint64_t n_sa = 0; double build_ms = 0.0;      // HBM and pinned host memory of the index
    // run state
    KjDevBuf counter, err, maxlen, quirk;
    KjDevBuf evbreaks; uint32_t n_evbreaks = 0;
    KjDevBuf counts, counts_pending; uint32_t n_counts = 0, n_present = 0;   // per-taxon read counts (+1 slot: unclassified)
    uint32_t variant_boost = 1;    // Greedy variant-ring capacity multiplier, raised after an overflow (flag 4) so that a retry succeeds
    uint32_t max_read_len = KJ_MAX_READ_LEN;    // longest mate admitted (kj_set_max_read_len); protein reads: a third of it
    KjDevBuf prep;                 // prepared-item records of the two-kernel Greedy path (two slots x two buffers)
    KjSlot slot[2];
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    uint64_t launches = 0; double last_kernel_ms = 0.0;
    int grid = 0; size_t smem_bytes = 0; KjKernel grid_kernel = nullptr;      // the last launch's geometry, and the kernel whose occupancy gave the grid
};

// Where a launch writes its results (null: not wanted).  launch() takes device arrays; classify_host takes the host arrays the chunks are
// copied back to (`compact` stays a device array) and fills in the slot's device arrays per chunk.
struct KjOut {
    uint64_t* tax = nullptr; uint32_t* best = nullptr; uint32_t* compact = nullptr;
    uint64_t* ids = nullptr; uint8_t* nids = nullptr;                       // match-id sets (kj_classify_verbose)
    uint32_t* acc = nullptr; uint8_t* nacc = nullptr;                        // accession sets (kj_classify_verbose2)
    char* frag = nullptr; uint32_t frag_stride = 0; uint32_t* fraglen = nullptr;   // fragment strings (kj_classify_verbose2)
    unsigned long long* counts = nullptr;                                    // per-taxon counts (launch() only)
};

template <class T> static int upload(const std::vector<T>& v, KjDevBuf& d, uint64_t& total) {
    size_t bytes = std::max<size_t>(v.size() * sizeof(T), 16);
    int rc = d.grow(bytes); if (rc) return rc;
    if (!v.empty()) CK(cudaMemcpy(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    total += bytes; return KJ_OK;
}
// an array that may live in the host tier: its bytes count towards the context's host bytes there, towards `total` (HBM) otherwise (a group's
// array, placed on a device of its own, is counted by create_group_device)
static int tier_grow(kj_ctx* c, KjTierBuf& b, size_t bytes, uint64_t& total) {
    int rc = b.grow(bytes); if (rc) return rc;
    if (b.device < 0) (b.on_host ? c->host_bytes : total) += bytes;
    return KJ_OK;
}
template <class T> static int tier_upload(kj_ctx* c, const std::vector<T>& v, KjTierBuf& b, uint64_t& total) {
    int rc = tier_grow(c, b, std::max<size_t>(v.size() * sizeof(T), 16), total); if (rc) return rc;
    return v.empty() ? KJ_OK : b.put(v.data(), v.size() * sizeof(T));
}

// Shared-memory work space while three CTAs still fit on an SM; beyond that (mates longer than ~280 bases) the same
// carve-up is addressed in a global buffer instead, which keeps the grid at full occupancy for any read length.
// (A/B, MEM kernel-only: shared memory wins for PE150 and PE250 at 3 CTAs/SM, the global buffer wins for PE350 where only 2 CTAs/SM would fit.)
#define KJ_SMEM_WS_LIMIT (75u * 1024u)
// the fixed-profile kernels apply when the batch's carve-up is exactly the compiled-in one
static bool kj_use_fixed(const KjRunParams& rp) {
    if (rp.ws_global || rp.mode != 1) return false;      // Greedy only: faster for Greedy in an A/B run, slightly slower for MEM
    const KjSmemLayout a = kj_smem_layout(rp), b = kj_smem_layout(kj_fixed_profile(rp.mode));
    return memcmp(&a, &b, sizeof a) == 0 && rp.max_len == 152 && rp.kept_cap_smem == KJ_KEPT_SMEM;
}
// Prepares the kernels of one launch (`front` may be null) for `smem` bytes of dynamic shared memory and sets the persistent grid from the
// occupancy of `kern`: with the Greedy front-end / search pair that is the search kernel, and the front end needs no more than that.
static int configure_launch(kj_ctx* c, KjKernel front, KjKernel kern, size_t smem) {
    {   // The max-dynamic-shared-memory attribute belongs to the kernel instantiation on the device, not to a context: several contexts
        // (or batches with different read lengths) share it, so it is only ever raised (process-wide table), never lowered.
        static std::mutex attr_mu; static std::map<std::pair<int, KjKernel>, size_t> attr_set;
        std::lock_guard<std::mutex> lk(attr_mu);
        for (KjKernel k : {front, kern}) {
            if (!k) continue;
            size_t& cur = attr_set[{c->device, k}];
            if (smem > cur) { CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); cur = smem; }
        }
    }
    if (kern == c->grid_kernel && smem == c->smem_bytes && c->grid > 0) return KJ_OK;
    int per_sm = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, KJ_WARPS_PER_CTA * 32, smem));
    if (per_sm < 1) { kj_err() = "kernel does not fit on an SM"; return KJ_ERR_UNSUPPORTED; }
    c->grid = c->sm_count * per_sm;          // persistent grid: a whole number of CTAs per SM
    c->grid_kernel = kern; c->smem_bytes = smem;
    return KJ_OK;
}

// E-value gate: break points of the minimal passing score (kj_build_evalue_breaks), rebuilt when the parameters change
static int upload_evalue_breaks(kj_ctx* c) {
    c->evbreaks.reset(); c->n_evbreaks = 0;
    std::vector<double> br; int rc = kj_build_evalue_breaks(c->params, c->H.db_length, br); if (rc) return rc;
    if (br.empty()) return KJ_OK;
    if ((rc = c->evbreaks.grow(br.size() * sizeof(double)))) return rc;
    CK(cudaMemcpy(c->evbreaks.p, br.data(), br.size() * sizeof(double), cudaMemcpyHostToDevice));
    c->n_evbreaks = (uint32_t)br.size();
    return KJ_OK;
}

static thread_local bool kj_transient_ctx = false;      // the base context of kj_create_scaled lives for the construction only: no second k-mer table
static int new_ctx(kj_ctx** out, int device, const kj_params* params) {
    int rc = kj_check_params(*params); if (rc) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { kj_err() = "no CUDA device available (this library has no CPU fallback)"; return KJ_ERR_NO_DEVICE; }
    if (device < 0 || device >= ndev) { kj_err() = "device ordinal out of range"; return KJ_ERR_ARG; }
    CK(cudaSetDevice(device));
    kj_ctx* c = new kj_ctx(); c->device = device; c->params = *params;
    std::unique_ptr<kj_ctx, void (*)(kj_ctx*)> guard(c, kj_destroy);
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, device)); c->sm_count = prop.multiProcessorCount;
    if ((rc = c->err.grow(sizeof(uint32_t)))) return rc;
    CK(cudaMemset(c->err.p, 0, sizeof(uint32_t)));
    if ((rc = c->quirk.grow(sizeof c->H.quirk_d))) return rc;
    CK(cudaMemset(c->quirk.p, 0, sizeof c->H.quirk_d));
    *out = guard.release(); return KJ_OK;
}
// device descriptor from the context's device arrays + meta data
static int upload_descriptor(kj_ctx* c) {
    KjHostIndex& H = c->H; KjDevIndex& D = c->dix; memset(&D, 0, sizeof D);
    D.rank = c->rank.as<const uint64_t>(); D.nb = H.nb; D.letters = c->letters.as<const uint64_t>(); D.bwtlen = H.bwtlen; D.alen = H.alen;
    for (int a = 0; a <= H.alen; a++) D.C[a] = H.C[a];
    if (!kj_is_compact(H.wide)) for (int a = 0; a < H.alen; a++) D.rank_base[a] = D.rank + (uint64_t)a * H.nb * kj_rank_words(H.wide);
    if (H.wide == KJ_LAYOUT_COMPACT_TIERED) { D.tier.host = c->rank_host.as<const uint64_t>(); D.tier.nb_dev = c->nb_dev; }
    const KjGroup* G = c->group.get();
    if (H.wide == KJ_LAYOUT_COMPACT_SPREAD) { D.spread = G->ref; D.rank = G->ref.base[0]; }
    const KjTierBuf& sa_acc = G ? G->sa_acc : c->sa_acc; const KjTierBuf& seq_acc = G ? G->seq_acc : c->seq_acc;
    const KjTierBuf& sa_tax = G ? G->sa_tax : c->sa_tax; const KjTierBuf& seq_tax = G ? G->seq_tax : c->seq_tax;
    D.sa_acc = sa_acc.as<const uint32_t>(); D.seq_acc = seq_acc.as<const uint32_t>();
    D.sa_tax = sa_tax.as<const uint32_t>(); D.seq_tax = seq_tax.as<const uint32_t>(); D.sa_check = H.sa_check; D.sa_exp = H.sa_exp; D.sa_bias = H.sa_bias;
    D.n_sa = c->n_sa; D.row_tax = c->row_tax.as<const uint32_t>(); D.nseq = H.nseq;
    D.tax_parent = c->tax_parent.as<const uint32_t>(); D.tax_depth = c->tax_depth.as<const uint32_t>(); D.tax_id = c->tax_id.as<const uint64_t>(); D.n_tax = (uint32_t)H.tax_id.size();
    D.lnfact = c->lnfact.as<const double>(); D.n_lnfact = (int)H.lnfact.size(); D.kmer = H.kmer_k ? c->kmer.p : nullptr; D.kmer_k = H.kmer_k; D.wide = H.wide; D.tables = c->tables.as<KjTables>();
    D.quirk_lo = H.quirk_lo; D.mono = H.quirk_lo == ~0ull ? 1 : 0; D.quirk_d = c->quirk.as<uint64_t>();
    int rc = c->ix.grow(sizeof(KjDevIndex)); if (rc) return rc;
    CK(cudaMemcpy(c->ix.p, &D, sizeof(KjDevIndex), cudaMemcpyHostToDevice));
    if (c->kmer_mem.p && c->kmer_k_mem) {
        KjDevIndex M = D; M.kmer = c->kmer_mem.p; M.kmer_k = c->kmer_k_mem;
        if ((rc = c->ix_mem.grow(sizeof(KjDevIndex)))) return rc;
        CK(cudaMemcpy(c->ix_mem.p, &M, sizeof(KjDevIndex), cudaMemcpyHostToDevice));
    }
    return KJ_OK;
}
static int upload_small(kj_ctx* c, uint64_t& tot) {
    KjHostIndex& H = c->H; int rc;
    if ((rc = upload(H.tax_parent, c->tax_parent, tot)) || (rc = upload(H.tax_depth, c->tax_depth, tot)) || (rc = upload(H.tax_id, c->tax_id, tot)) || (rc = upload(H.lnfact, c->lnfact, tot)) ||
        (rc = c->tables.grow(sizeof(KjTables)))) return rc;
    CK(cudaMemcpy(c->tables.p, &H.tables, sizeof(KjTables), cudaMemcpyHostToDevice));
    return KJ_OK;
}
static int kj_device_build_row_tax(kj_ctx* c, uint64_t& tot);      // kj_build.h
static int finish_ctx(kj_ctx* c, uint64_t tot) {
    KjHostIndex& H = c->H; int rc;
    CK(cudaMemcpy(c->quirk.p, H.quirk_d, sizeof H.quirk_d, cudaMemcpyHostToDevice));
    // the row -> taxon array is built by walking the finished index; both descriptors then carry it
    if ((rc = upload_descriptor(c)) || (rc = kj_device_build_row_tax(c, tot)) || (rc = upload_descriptor(c))) return rc;
    c->index_bytes = tot;
    if ((rc = c->counter.grow(4 * sizeof(unsigned long long))) || (rc = c->maxlen.grow(2 * sizeof(unsigned int)))) return rc;       // counters: [slot] classify / search, [2 + slot] front end
    for (KjSlot& S : c->slot) {
        CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&S.fstream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&S.ev_in, cudaEventDisableTiming));
        for (int b = 0; b < 2; b++) { CK(cudaEventCreateWithFlags(&S.ev_f[b], cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&S.ev_s[b], cudaEventDisableTiming)); }
    }
    CK(cudaEventCreate(&c->ev_a)); CK(cudaEventCreate(&c->ev_b));
    if ((rc = upload_evalue_breaks(c))) return rc;
    c->n_counts = (uint32_t)H.tax_id.size() + 1u; c->n_present = H.n_present;
    if ((rc = c->counts.grow((size_t)c->n_counts * 8)) || (rc = c->counts_pending.grow((size_t)c->n_counts * 8))) return rc;
    CK(cudaMemset(c->counts.p, 0, (size_t)c->n_counts * 8)); CK(cudaMemset(c->counts_pending.p, 0, (size_t)c->n_counts * 8));
    return KJ_OK;
}

// kj_create_from_native (and kj_create with KJ_HOST_BUILD=1): `fill` produces the host arrays of the device layout, the rest uploads them
template <class Fill> static int create_ctx(kj_ctx** out, int device, const kj_params* params, Fill fill) {
    kj_ctx* c = nullptr; int rc = new_ctx(&c, device, params); if (rc) return rc;
    std::unique_ptr<kj_ctx, void (*)(kj_ctx*)> guard(c, kj_destroy);      // every early return below releases what was allocated so far
    rc = fill(c->H); if (rc) return rc;
    KjHostIndex& H = c->H; uint64_t tot = 0;
    // one guard entry: the reference's header counts one sampled row less than kaiju-mkbwt writes (suffixArray.c:160 vs 206-216), so the last
    // sampled row of an index has no entry; the reference reads past its array there, the device reads "no taxon"
    c->n_sa = H.sa_tax.size(); H.sa_tax.push_back(KJ_TAX_BAD);
    if (!H.seq_acc.empty()) { H.sa_acc.push_back(0xffffffffu); if ((rc = tier_upload(c, H.sa_acc, c->sa_acc, tot)) || (rc = tier_upload(c, H.seq_acc, c->seq_acc, tot))) return rc; }
    if ((rc = upload(H.rank, c->rank, tot)) || (rc = upload(H.letters, c->letters, tot)) || (rc = tier_upload(c, H.sa_tax, c->sa_tax, tot)) ||
        (rc = tier_upload(c, H.seq_tax, c->seq_tax, tot)) || (rc = upload_small(c, tot)) || (rc = (H.wide ? upload(H.kmer, c->kmer, tot) : upload(H.kmer32, c->kmer, tot)))) return rc;
    // host copies of the big arrays are no longer needed
    std::vector<uint64_t>().swap(H.rank); std::vector<uint64_t>().swap(H.letters); std::vector<uint32_t>().swap(H.sa_tax); std::vector<KjKmer>().swap(H.kmer); std::vector<KjKmer32>().swap(H.kmer32);
    if ((rc = finish_ctx(c, tot))) return rc;
    *out = guard.release(); return KJ_OK;
}

#include "kj_build.h"
// kj_create / kj_create_scaled / kj_create_tiered: the large arrays are built on the device from the raw BWT bytes and suffix-array samples
// (kj_build.h); host_budget > 0: a compact index that does not fit in HBM may take up to that many bytes of pinned host memory (kj_choose_layout)
static int create_ctx_device(kj_ctx** out, int device, const kj_params* params, const kj_index_view& v, const kj_taxonomy_view& t, uint32_t copies, const kj_ctx* base,
                             uint64_t host_budget) {
    kj_ctx* c = nullptr; int rc = new_ctx(&c, device, params); if (rc) return rc;
    std::unique_ptr<kj_ctx, void (*)(kj_ctx*)> guard(c, kj_destroy);
    const auto t0 = std::chrono::steady_clock::now();
    uint8_t lcode[256]; rc = kj_build_host_meta(v, t, copies, c->H, lcode); if (rc) return rc;
    if ((rc = kj_choose_layout(c, v, copies, host_budget))) return rc;
    uint64_t tot = 0;
    if ((rc = upload_small(c, tot)) || (rc = kj_device_build(c, v, lcode, copies, base, tot))) return rc;
    c->H.kmer_k = 0;
    if ((rc = upload_descriptor(c))) return rc;
    { const char* ek = getenv("KJ_KMER_K"); if ((rc = kj_device_build_kmer(c, ek ? atoi(ek) : kj_default_kmer_k(c->H.bwtlen), tot, c->kmer, c->H.kmer_k))) return rc; }
    // MEM runs faster with the intervals of all 20^7 7-mers (10.2 GB below 2^32 rows): one look-up replaces the first LF step of every chain, the one
    // with all 32 lanes alive.  Greedy loses with it (its seeds rarely get that far), so it keeps the 6-mer table: two descriptors, one index.
    // Only where HBM is plentiful: narrow indexes, and the two level buffers of the construction (41 GB) must fit next to the index.
    if (!c->H.wide && c->H.kmer_k == 6 && !kj_transient_ctx && !getenv("KJ_KMER_K") && !getenv("KJ_NO_KMER7")) {
        size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to));
        if ((double)fr > 1.28e9 * (2.0 * sizeof(KjKmer) + sizeof(KjKmer32)) + 16e9 && (rc = kj_device_build_kmer(c, 7, tot, c->kmer_mem, c->kmer_k_mem))) return rc;
    }
    std::vector<uint32_t>().swap(c->H.seq_tax);
    if ((rc = finish_ctx(c, tot))) return rc;
    CK(cudaDeviceSynchronize());
    c->build_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = guard.release(); return KJ_OK;
}

extern "C" int kj_create(kj_ctx** out, int device, const kj_params* params, const kj_index_view* index, const kj_taxonomy_view* taxonomy) {
    if (!out || !params || !index || !taxonomy) { kj_err() = "kj_create: null argument"; return KJ_ERR_ARG; }
    if (getenv("KJ_HOST_BUILD")) return create_ctx(out, device, params, [&](KjHostIndex& H) { return kj_build_host_index(*index, *taxonomy, H); });   // developer hook: host transcoder + upload
    return create_ctx_device(out, device, params, *index, *taxonomy, 1, nullptr, 0);
}
static int create_scaled(kj_ctx** out, int device, const kj_params* params, const kj_index_view* index, const kj_taxonomy_view* taxonomy, uint32_t copies, uint64_t host_budget) {
    if (copies <= 1) return create_ctx_device(out, device, params, *index, *taxonomy, 1, nullptr, host_budget);
    kj_ctx* base = nullptr; kj_transient_ctx = true; int rc = create_ctx_device(&base, device, params, *index, *taxonomy, 1, nullptr, host_budget); kj_transient_ctx = false; if (rc) return rc;
    rc = create_ctx_device(out, device, params, *index, *taxonomy, copies, base, host_budget);
    kj_destroy(base);
    return rc;
}
extern "C" int kj_create_scaled(kj_ctx** out, int device, const kj_params* params, const kj_index_view* index, const kj_taxonomy_view* taxonomy, uint32_t copies) {
    if (!out || !params || !index || !taxonomy) { kj_err() = "kj_create_scaled: null argument"; return KJ_ERR_ARG; }
    if (copies <= 1) return kj_create(out, device, params, index, taxonomy);
    return create_scaled(out, device, params, index, taxonomy, copies, 0);
}
extern "C" int kj_create_tiered(kj_ctx** out, int device, const kj_params* params, const kj_index_view* index, const kj_taxonomy_view* taxonomy, uint32_t copies, uint64_t host_bytes) {
    if (!out || !params || !index || !taxonomy) { kj_err() = "kj_create_tiered: null argument"; return KJ_ERR_ARG; }
    if (host_bytes == 0) return kj_create_scaled(out, device, params, index, taxonomy, copies);
    return create_scaled(out, device, params, index, taxonomy, copies < 1 ? 1 : copies, host_bytes);
}

// Peer access between every ordered pair of distinct devices of a group: the kernels of each device read the record segments of the others.
// Per-process CUDA context state; an access enabled before (by an earlier group) is kept, and none is ever disabled.
static int kj_enable_peers(const int* devices, int n) {
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            const int a = devices[i], b = devices[j];
            if (a == b) continue;
            int can = 0; CK(cudaDeviceCanAccessPeer(&can, a, b));
            if (!can) { kj_err() = "kj_create_group: device " + std::to_string(a) + " has no peer access to device " + std::to_string(b) + " (its kernels could not read the records held there)"; return KJ_ERR_UNSUPPORTED; }
            KjDevGuard d(a);
            const cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else if (e != cudaSuccess) { kj_err() = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e); return KJ_ERR_CUDA; }
        }
    return KJ_OK;
}
// kj_create_group: one compact spread index over the HBM of devices[0..n), one context per listed device.  The construction runs on the first
// device (kj_plan_group, kj_group_alloc, kj_device_build: the records go straight into their owners' HBM); the first context's superblock and
// k-mer tables are then copied peer to peer to the other contexts, which upload their own taxonomy, tables and run state.
static int create_group_device(kj_ctx** out, int n, const int* devices, const kj_params* params, const kj_index_view& v, const kj_taxonomy_view& t, uint32_t copies) {
    std::vector<std::unique_ptr<kj_ctx, void (*)(kj_ctx*)>> cs;      // every early return below releases all contexts, and with the last the group
    std::vector<kj_ctx*> raw;
    for (int g = 0; g < n; g++) {
        kj_ctx* c = nullptr; int rc = new_ctx(&c, devices[g], params); if (rc) return rc;
        cs.emplace_back(c, kj_destroy); raw.push_back(c);
    }
    int rc = kj_enable_peers(devices, n); if (rc) return rc;
    auto G = std::make_shared<KjGroup>();
    for (kj_ctx* c : raw) c->group = G;
    kj_ctx* c0 = raw[0];
    CK(cudaSetDevice(c0->device));
    const auto t0 = std::chrono::steady_clock::now();
    // the scaled build resolves its suffix-array rows through a base context of the index on the first device (freed after the construction)
    std::unique_ptr<kj_ctx, void (*)(kj_ctx*)> base(nullptr, kj_destroy);
    if (copies > 1) {
        kj_ctx* b = nullptr; kj_transient_ctx = true; rc = create_ctx_device(&b, c0->device, params, v, t, 1, nullptr, 0); kj_transient_ctx = false; if (rc) return rc;
        base.reset(b); CK(cudaSetDevice(c0->device));
    }
    uint8_t lcode[256]; if ((rc = kj_build_host_meta(v, t, copies, c0->H, lcode))) return rc;
    if ((rc = kj_plan_group(raw.data(), n, v, copies, *G)) || (rc = kj_group_alloc(*G))) return rc;
    uint64_t tot = 0;
    if ((rc = upload_small(c0, tot)) || (rc = kj_device_build(c0, v, lcode, copies, base.get(), tot))) return rc;
    base.reset();
    G->sa_tax = std::move(c0->sa_tax); G->seq_tax = std::move(c0->seq_tax); G->sa_acc = std::move(c0->sa_acc); G->seq_acc = std::move(c0->seq_acc);
    c0->H.kmer_k = 0;
    if ((rc = upload_descriptor(c0))) return rc;
    { const char* ek = getenv("KJ_KMER_K"); if ((rc = kj_device_build_kmer(c0, ek ? atoi(ek) : kj_default_kmer_k(c0->H.bwtlen), tot, c0->kmer, c0->H.kmer_k))) return rc; }
    std::vector<uint32_t>().swap(c0->H.seq_tax);
    if ((rc = finish_ctx(c0, tot))) return rc;
    // the other members: the first context's meta data, its superblock and k-mer tables (peer to peer), their own small arrays and run state
    for (int g = 1; g < n; g++) {
        kj_ctx* c = raw[g]; CK(cudaSetDevice(c->device));
        c->H = c0->H; c->nb_dev = c0->nb_dev; c->n_sa = c0->n_sa; uint64_t ct = 0;
        if ((rc = upload_small(c, ct)) || (rc = c->letters.grow(c0->letters.cap))) return rc;
        CK(cudaMemcpyPeer(c->letters.p, c->device, c0->letters.p, c0->device, c0->letters.cap)); ct += c0->letters.cap;
        if (c0->kmer.p) {
            if ((rc = c->kmer.grow(c0->kmer.cap))) return rc;
            CK(cudaMemcpyPeer(c->kmer.p, c->device, c0->kmer.p, c0->device, c0->kmer.cap)); ct += c0->kmer.cap;
        }
        if ((rc = finish_ctx(c, ct))) return rc;
    }
    // kj_index_bytes: each context's replicas, its segment, and the suffix-array arrays on its device (counted at the first context there)
    for (int g = 0; g < n; g++) {
        kj_ctx* c = raw[g]; c->index_bytes += G->seg[g].cap;
        if (std::find(devices, devices + g, c->device) != devices + g) continue;
        for (const KjTierBuf* b : {&G->sa_tax, &G->seq_tax, &G->sa_acc, &G->seq_acc}) if (b->p && b->device == c->device) c->index_bytes += b->cap();
    }
    for (kj_ctx* c : raw) { CK(cudaSetDevice(c->device)); CK(cudaDeviceSynchronize()); }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (int g = 0; g < n; g++) { raw[g]->build_ms = ms; out[g] = cs[g].release(); }
    return KJ_OK;
}
extern "C" int kj_create_group(kj_ctx** out, int n, const int* devices, const kj_params* params, const kj_index_view* index, const kj_taxonomy_view* taxonomy, uint32_t copies) {
    if (!out || !devices || !params || !index || !taxonomy) { kj_err() = "kj_create_group: null argument"; return KJ_ERR_ARG; }
    if (n < 1 || n > KJ_MAX_GROUP) { kj_err() = "kj_create_group: a group has 1 to " + std::to_string(KJ_MAX_GROUP) + " devices, not " + std::to_string(n); return KJ_ERR_ARG; }
    const int ndev = kj_device_count();
    for (int g = 0; g < n; g++)
        if (ndev > 0 && (devices[g] < 0 || devices[g] >= ndev)) { kj_err() = "kj_create_group: device ordinal " + std::to_string(devices[g]) + " out of range"; return KJ_ERR_ARG; }
    for (int g = 0; g < n; g++) out[g] = nullptr;
    return create_group_device(out, n, devices, params, *index, *taxonomy, copies < 1 ? 1 : copies);
}
extern "C" double kj_index_build_ms(const kj_ctx* c) { return c ? c->build_ms : 0.0; }
// test hook: checksums of the index arrays as they sit in memory (rank, letters or the compact superblock table, sa_tax, seq_tax, kmer | bwtlen,
// layout, n_sa), to compare the device construction with the host transcoder array for array.  The records of a compact tiered index are its
// HBM part followed by its host part.
extern "C" int kj_debug_index_checksums(kj_ctx* c, uint64_t out[8]) {
    if (!c || !out) return KJ_ERR_ARG; CK(cudaSetDevice(c->device)); CK(cudaDeviceSynchronize());
    const KjHostIndex& H = c->H; memset(out, 0, 64);
    const size_t sz[5] = {(size_t)kj_rank_array_words(H.wide, H.alen, H.nb) * 8, (size_t)kj_letters_words(H.wide, H.bwtlen) * 8, (size_t)c->n_sa * 4, (size_t)H.nseq * 4,
                          H.kmer_k ? (size_t)pow(20.0, H.kmer_k) * (H.wide ? sizeof(KjKmer) : sizeof(KjKmer32)) : 0};
    const KjGroup* G = c->group.get();
    const void* ptr[5] = {c->rank.p, c->letters.p, G ? G->sa_tax.p : c->sa_tax.p, G ? G->seq_tax.p : c->seq_tax.p, c->kmer.p};
    const size_t dev0 = H.wide == KJ_LAYOUT_COMPACT_TIERED ? (size_t)c->nb_dev * KJ_RANK_WORDS_COMPACT * 8 : G ? 0 : sz[0];      // bytes of the records in `rank`
    for (int i = 0; i < 5; i++) {
        std::vector<uint8_t> h(sz[i]); const size_t nd = i == 0 ? dev0 : sz[i];
        if (nd) CK(cudaMemcpy(h.data(), ptr[i], nd, cudaMemcpyDefault));
        if (i == 0 && G) {      // compact spread: the segments in group order
            for (int g = 0; g < G->n; g++) {
                const size_t o = (size_t)G->first[g] * KJ_RANK_WORDS_COMPACT * 8, b = (size_t)(G->first[g + 1] - G->first[g]) * KJ_RANK_WORDS_COMPACT * 8;
                if (b) CK(cudaMemcpy(h.data() + o, G->seg[g].p, b, cudaMemcpyDefault));
            }
        } else if (i == 0 && sz[0] > dev0) memcpy(h.data() + dev0, c->rank_host.p, sz[0] - dev0);
        out[i] = kj_mix_bytes(0x6b616a75ull + i, h.data(), h.size());
    }
    out[5] = H.bwtlen; out[6] = (uint64_t)H.wide; out[7] = c->n_sa;
    return KJ_OK;
}

// device-native index file (SURVEY.md 8f-4): written once from the reference's .fmi + nodes.dmp, loaded without the transcode
extern "C" int kj_native_index_write(const kj_index_view* index, const kj_taxonomy_view* taxonomy, const char* path) {
    if (!index || !taxonomy || !path) { kj_err() = "kj_native_index_write: null argument"; return KJ_ERR_ARG; }
    KjHostIndex H; int rc = kj_build_host_index(*index, *taxonomy, H); if (rc) return rc;
    return kj_host_index_write(H, path);
}
extern "C" int kj_create_from_native(kj_ctx** out, int device, const kj_params* params, const char* path) {
    if (!out || !params || !path) { kj_err() = "kj_create_from_native: null argument"; return KJ_ERR_ARG; }
    return create_ctx(out, device, params, [&](KjHostIndex& H) { return kj_host_index_read(path, H); });
}

extern "C" int kj_set_max_read_len(kj_ctx* c, uint32_t bases) {
    if (!c) { kj_err() = "kj_set_max_read_len: null argument"; return KJ_ERR_ARG; }
    if (bases < KJ_MAX_READ_LEN || bases > KJ_MAX_LONG_READ_LEN) { kj_err() = "kj_set_max_read_len: the limit must lie in [KJ_MAX_READ_LEN, KJ_MAX_LONG_READ_LEN] = [16383, 1048575]"; return KJ_ERR_ARG; }
    c->max_read_len = bases; return KJ_OK;
}

extern "C" int kj_set_params(kj_ctx* c, const kj_params* p) {
    if (!c || !p) { kj_err() = "kj_set_params: null argument"; return KJ_ERR_ARG; }
    int rc = kj_check_params(*p); if (rc) return rc;
    CK(cudaSetDevice(c->device));
    c->params = *p;
    // the record buffers of the two-kernel Greedy path (up to 32 GB) go back when the context leaves Greedy mode
    if (c->params.mode != 1 && c->prep.p) { CK(cudaDeviceSynchronize()); c->prep.reset(); }
    return upload_evalue_breaks(c);
}

extern "C" void kj_destroy(kj_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    c->files.reset();      // first: it joins the parser thread
    for (KjSlot& S : c->slot) { if (S.stream) cudaStreamDestroy(S.stream); if (S.fstream) cudaStreamDestroy(S.fstream); if (S.ev_in) cudaEventDestroy(S.ev_in);
                               for (int b = 0; b < 2; b++) { if (S.ev_f[b]) cudaEventDestroy(S.ev_f[b]); if (S.ev_s[b]) cudaEventDestroy(S.ev_s[b]); } }
    if (c->ev_a) cudaEventDestroy(c->ev_a); if (c->ev_b) cudaEventDestroy(c->ev_b);
    delete c;              // the device buffers go with their owners
}

// The grid of a long-read launch: per-warp scratch grows linearly with the longest read (about 100 MB per warp at 1 Mb), so the persistent grid is
// cut to the CTAs whose scratch fits half of the free HBM (the other pipeline slot may need the same); this slot's current buffers count as free,
// they are replaced.  A read is never spread over warps: if not even one CTA fits, the launch fails.
static int long_read_grid(kj_ctx* c, const KjSlot& S, const KjRunParams& rp, size_t per_warp, int& grid) {
    size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to));
    const size_t reserve = 256ull << 20, avail = fr + S.spill.cap + S.gscratch.cap + S.ws.cap;
    size_t budget = avail > reserve ? (avail - reserve) / 2 : 0;
    if (const char* v = getenv("KJ_LONG_BUDGET_MB")) budget = (size_t)atoll(v) << 20;      // test hook: a smaller budget
    const size_t per_cta = per_warp * KJ_WARPS_PER_CTA, ctas = budget / per_cta;
    if (ctas < 1) {
        char b[240]; snprintf(b, sizeof b, "reads of up to %u bases need %zu bytes of work space per warp (%zu per CTA of %d warps); the budget of free device memory is %zu bytes",
                              rp.max_len, per_warp, per_cta, KJ_WARPS_PER_CTA, budget);
        kj_err() = b; return KJ_ERR_NOMEM;
    }
    if ((size_t)grid > ctas) grid = (int)ctas;
    c->grid = grid; c->grid_kernel = nullptr;      // the geometry of this launch; the next launch derives its own
    return KJ_OK;
}

// one launch over reads [0,n) whose sequences/offsets are resident on the device
static int launch(kj_ctx* c, int slot, const uint8_t* d_seq1, const uint64_t* d_off1, const uint8_t* d_seq2, const uint64_t* d_off2, uint64_t base1, uint64_t base2,
                  uint64_t n, uint32_t max1, uint32_t max2, const KjOut& o, cudaStream_t st, bool time_it) {
    const bool raised = c->max_read_len != KJ_MAX_READ_LEN; char msg[200];
    if (c->params.input_is_protein) {
        if (d_seq2) { kj_err() = "protein input only supports one input (kaiju.cpp:201)"; return KJ_ERR_ARG; }
        if (max1 > c->max_read_len / 3) {
            if (!raised) kj_err() = "protein read longer than KJ_MAX_PROTEIN_LEN (5461 residues) is not supported";
            else { snprintf(msg, sizeof msg, "protein read longer than %u residues (a third of kj_set_max_read_len's %u bases) is not supported", c->max_read_len / 3, c->max_read_len); kj_err() = msg; }
            return KJ_ERR_UNSUPPORTED;
        }
    } else if (max1 > c->max_read_len || max2 > c->max_read_len) {
        if (!raised) kj_err() = "read longer than KJ_MAX_READ_LEN (16383 bases) is not supported";
        else { snprintf(msg, sizeof msg, "read longer than %u bases (kj_set_max_read_len) is not supported", c->max_read_len); kj_err() = msg; }
        return KJ_ERR_UNSUPPORTED;
    }
    // the kernel follows from the read lengths alone: mates beyond KJ_MAX_READ_LEN need the long-read kernels' wide fields
    const bool long_reads = c->params.input_is_protein ? max1 > KJ_MAX_PROTEIN_LEN : std::max(max1, max2) > KJ_MAX_READ_LEN;
    KjRunParams rp; kj_fill_run_params(c->params, std::max(max1, max2), rp);
    rp.ev_breaks = c->evbreaks.as<double>(); rp.n_ev_breaks = c->n_evbreaks;
    rp.variant_cap *= c->variant_boost;
    const bool verbose = o.ids || o.acc || o.frag;
    const KjSmemLayout lay = long_reads ? kj_smem_layout<true>(rp) : kj_smem_layout(rp);
    const uint32_t gs_bytes = long_reads ? kj_greedy_scratch_bytes<true>(rp) : kj_greedy_scratch_bytes(rp);
    const size_t head = kj_align((uint32_t)sizeof(KjCtaShared), 16), ws_smem = head + (size_t)KJ_WARPS_PER_CTA * lay.total;
    rp.ws_global = long_reads || ws_smem > KJ_SMEM_WS_LIMIT ? 1u : 0u;
    const size_t smem = rp.ws_global ? head : ws_smem;
    const bool fixed = !verbose && kj_use_fixed(rp);
    // Greedy with the work space in shared memory: front-end kernel + search kernel over sub-batches (the records of a sub-batch live in d_prep)
    const bool split = rp.mode == 1 && !rp.ws_global && !verbose && !getenv("KJ_NO_SPLIT");
    const KjKernel kern = kj_select_kernel(rp.mode, c->H.wide, rp.ws_global, fixed, verbose, split ? 2 : 0, long_reads);
    const KjKernel front = split ? kj_select_kernel(rp.mode, c->H.wide, false, fixed, false, 1) : nullptr;
    int rc = configure_launch(c, front, kern, smem); if (rc) return rc;
    int grid = c->grid;
    KjSlot& S = c->slot[slot];
    // the scratch of a long-read launch (up to half of the free HBM) goes back when this slot next launches without long reads
    if (S.long_scratch && !long_reads) { S.spill.reset(); S.gscratch.reset(); S.ws.reset(); }
    S.long_scratch = long_reads;
    if (long_reads && (rc = long_read_grid(c, S, rp, (size_t)lay.total + (size_t)rp.scratch_entries * sizeof(KjKept) + gs_bytes, grid))) return rc;
    const size_t warps = (size_t)grid * KJ_WARPS_PER_CTA;
    if ((rc = S.spill.grow(warps * rp.scratch_entries * sizeof(KjKept))) || (rc = S.gscratch.grow(warps * (size_t)gs_bytes)) ||
        (rc = S.ws.grow(rp.ws_global ? warps * (size_t)lay.total : 0))) return rc;
    if (time_it) CK(cudaEventRecord(c->ev_a, st));
    const KjDevIndex* dix = (rp.mode == 0 && c->ix_mem.p && rp.m >= (uint32_t)c->kmer_k_mem) ? c->ix_mem.as<KjDevIndex>() : c->ix.as<KjDevIndex>();
    const uint32_t pstride = split ? kj_prep_stride(rp) : 0u; uint64_t sub = n;
    if (split) {
        // records of one sub-batch per buffer; two buffers per slot (the front end of sub-batch b+1 runs in the tail of the search of sub-batch b).
        // Up to 8 GB per buffer where HBM is plentiful: fewer, longer search launches (3 M rather than 750 k pairs per launch was faster in an A/B run)
        uint64_t per_buf = c->prep.cap / 4;
        if (per_buf < (8ull << 30) && per_buf < n * (uint64_t)pstride) {       // (re)allocate: what this launch needs, at least 1 GB, at most 8 GB or 1/16 of the free memory
            size_t fr = 0, to = 0; CK(cudaMemGetInfo(&fr, &to)); fr += c->prep.cap;
            const uint64_t lim = std::max<uint64_t>(64ull << 20, std::min<uint64_t>(8ull << 30, fr / 16));
            const uint64_t want = std::min<uint64_t>(lim, std::max<uint64_t>(1ull << 30, n * (uint64_t)pstride + (n * (uint64_t)pstride) / 4));
            if (want > per_buf) { if ((rc = c->prep.grow((size_t)want * 4))) return rc; per_buf = want; }
        }
        sub = std::max<uint64_t>(1024, per_buf / pstride);
        if (const char* v = getenv("KJ_SPLIT_SUB")) { const long long x = atoll(v); if (x >= 1024 && (uint64_t)x < sub) sub = (uint64_t)x; }
        sub = std::min(sub, n);
    }
    // one kernel launch over items [b0, b1), claimed through the counter `ctr` (zeroed on the launch's stream first)
    auto run = [&](KjKernel k, cudaStream_t s, unsigned long long* ctr, uint8_t* pbuf, uint64_t b0, uint64_t b1) -> int {
        CK(cudaMemsetAsync(ctr, 0, sizeof(unsigned long long), s));
        k<<<grid, KJ_WARPS_PER_CTA * 32, smem, s>>>(dix, rp, lay, d_seq1, d_off1, d_seq2, d_off2, base1, base2, b1, o.tax, o.best, o.ids, o.nids, o.compact,
                                                     ctr, S.spill.as<KjKept>(), S.gscratch.as<uint8_t>(), gs_bytes, rp.ws_global ? S.ws.as<uint8_t>() : nullptr,
                                                     o.counts, c->err.as<uint32_t>(), o.acc, o.nacc, o.frag, o.frag_stride, o.fraglen, pbuf, pstride, b0);
        c->launches++;
        return KJ_OK;
    };
    unsigned long long* counter = c->counter.as<unsigned long long>();
    if (split) {
        // front end on the slot's own stream, search on the caller's: F(b) -> S(b) through ev_f, S(b) -> F(b+2) (same buffer) through ev_s.
        // (A search grid that leaves one CTA slot per SM to the front end of the next sub-batch was slower in an A/B run.)
        cudaStream_t fs = S.fstream; uint8_t* base = c->prep.as<uint8_t>() + (size_t)slot * (c->prep.cap / 2); uint64_t k = 0;
        CK(cudaEventRecord(S.ev_in, st)); CK(cudaStreamWaitEvent(fs, S.ev_in, 0));      // the inputs may have been produced on the caller's stream
        for (uint64_t b0 = 0; b0 < n; b0 += sub, k++) {
            const uint64_t b1 = std::min(n, b0 + sub); const int pb = (int)(k & 1);
            uint8_t* pbuf = base + (size_t)pb * (c->prep.cap / 4);
            CK(cudaStreamWaitEvent(fs, S.ev_s[pb], 0));                 // the search that last read this buffer (of this or an earlier launch; no-op if none)
            if ((rc = run(front, fs, counter + 2 + slot, pbuf, b0, b1))) return rc;
            CK(cudaEventRecord(S.ev_f[pb], fs));
            CK(cudaStreamWaitEvent(st, S.ev_f[pb], 0));
            if ((rc = run(kern, st, counter + slot, pbuf, b0, b1))) return rc;
            CK(cudaEventRecord(S.ev_s[pb], st));
        }
    } else if ((rc = run(kern, st, counter + slot, nullptr, 0, n))) return rc;
    CK(cudaGetLastError());
    if (time_it) CK(cudaEventRecord(c->ev_b, st));
    return KJ_OK;
}

static int count_taxa(kj_ctx* c, const uint64_t* d_tax, uint64_t n, unsigned long long* d_dst, cudaStream_t st) {
    if (!n) return KJ_OK;
    kj_count_kernel<<<c->sm_count * 4, 256, 0, st>>>(d_tax, n, c->dix.tax_id, c->n_present, c->n_counts - 1u, d_dst);
    CK(cudaGetLastError()); c->launches++;
    return KJ_OK;
}

static int check_err_flag(kj_ctx* c) {
    uint32_t e = 0; CK(cudaMemcpy(&e, c->err.p, sizeof e, cudaMemcpyDeviceToHost));
    if (e) {
        CK(cudaMemset(c->err.p, 0, sizeof e));
        // flag 4 = the Greedy variant ring of some read was full: the next launch gets a ring 4x as large (the reference's heap is unbounded)
        if ((e & 4u) && c->variant_boost < 256u) c->variant_boost *= 4u;
        char b[160]; snprintf(b, sizeof b, "per-read work queue overflow on the device (flags 0x%x)%s", e, (e & 4u) ? "; the variant ring was enlarged, call again" : (e & 128u) ? "; the fragment strings of a read exceed frag_stride" : ""); kj_err() = b;
        return KJ_ERR_OVERFLOW;
    }
    return KJ_OK;
}

extern "C" int kj_classify_device2(kj_ctx* c, const char* d_seq1, const uint64_t* d_off1, const char* d_seq2, const uint64_t* d_off2, uint64_t n,
                                   uint32_t max_len1, uint32_t max_len2, uint64_t* d_tax, uint32_t* d_best, uint32_t* d_compact, void* cuda_stream) {
    if (!c || !d_seq1 || !d_off1 || (!d_tax && !d_compact) || (d_seq2 && !d_off2)) { kj_err() = "kj_classify_device: null argument"; return KJ_ERR_ARG; }
    if (n == 0) return KJ_OK;
    CK(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    if (max_len1 == 0 || (d_seq2 && max_len2 == 0)) {
        unsigned int* d_maxlen = c->maxlen.as<unsigned int>();
        CK(cudaMemsetAsync(d_maxlen, 0, 2 * sizeof(unsigned int), st));
        kj_maxlen_kernel<<<256, 256, 0, st>>>(d_off1, n, d_maxlen); c->launches++;
        if (d_seq2) { kj_maxlen_kernel<<<256, 256, 0, st>>>(d_off2, n, d_maxlen + 1); c->launches++; }
        unsigned int h[2] = {0, 0}; CK(cudaMemcpyAsync(h, d_maxlen, sizeof h, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st));
        max_len1 = h[0]; max_len2 = h[1];
    }
    return launch(c, 0, (const uint8_t*)d_seq1, d_off1, (const uint8_t*)d_seq2, d_off2, 0, 0, n, max_len1, max_len2, KjOut{d_tax, d_best, d_compact}, st, true);
}

extern "C" int kj_classify_device(kj_ctx* c, const char* d_seq1, const uint64_t* d_off1, const char* d_seq2, const uint64_t* d_off2, uint64_t n,
                                  uint32_t max_len1, uint32_t max_len2, uint64_t* d_tax, uint32_t* d_best, void* cuda_stream) {
    if (!d_tax) { kj_err() = "kj_classify_device: null argument"; return KJ_ERR_ARG; }
    return kj_classify_device2(c, d_seq1, d_off1, d_seq2, d_off2, n, max_len1, max_len2, d_tax, d_best, nullptr, cuda_stream);
}

// `o` holds the caller's host arrays (and a device array for `compact`)
static int classify_host(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n, const KjOut& o) {
    if (!c || !seq1 || !off1 || !o.tax || (seq2 && !off2) || ((o.ids == nullptr) != (o.nids == nullptr))) { kj_err() = "kj_classify: null argument"; return KJ_ERR_ARG; }
    if (n == 0) return KJ_OK;
    CK(cudaSetDevice(c->device));
    const bool paired = seq2 != nullptr;
    // batch-wide length bounds (fix the shared-memory carve-up for all chunks): of all reads, and of the reads the short kernels take; and the
    // reads that need the long-read kernels (a mate above KJ_MAX_READ_LEN bases, protein: KJ_MAX_PROTEIN_LEN residues), in input order
    uint32_t max1 = 0, max2 = 0, smax1 = 0, smax2 = 0; std::vector<uint64_t> longs;
    {
        const uint32_t lim = c->params.input_is_protein ? KJ_MAX_PROTEIN_LEN : KJ_MAX_READ_LEN;
        unsigned nthr = std::max(1u, std::min(64u, std::thread::hardware_concurrency())); if (n < 65536) nthr = 1;
        std::vector<uint32_t> m1(nthr, 0), m2(nthr, 0), s1(nthr, 0), s2(nthr, 0); std::vector<std::vector<uint64_t>> lg(nthr); std::vector<std::thread> th;
        for (unsigned t = 0; t < nthr; t++) th.emplace_back([&, t] { uint64_t a = n * t / nthr, b = n * (t + 1) / nthr; uint32_t x = 0, y = 0, sx = 0, sy = 0;
            for (uint64_t i = a; i < b; i++) { uint64_t l = off1[i + 1] - off1[i]; if (l > 0xffffffffull) l = 0xffffffffull; x = std::max(x, (uint32_t)l);
                                               uint64_t k = 0; if (paired) { k = off2[i + 1] - off2[i]; if (k > 0xffffffffull) k = 0xffffffffull; y = std::max(y, (uint32_t)k); }
                                               if (l > lim || k > lim) lg[t].push_back(i); else { sx = std::max(sx, (uint32_t)l); sy = std::max(sy, (uint32_t)k); } }
            m1[t] = x; m2[t] = y; s1[t] = sx; s2[t] = sy; });
        for (auto& x : th) x.join();
        for (unsigned t = 0; t < nthr; t++) { max1 = std::max(max1, m1[t]); max2 = std::max(max2, m2[t]); smax1 = std::max(smax1, s1[t]); smax2 = std::max(smax2, s2[t]); longs.insert(longs.end(), lg[t].begin(), lg[t].end()); }
    }
    CK(cudaMemset(c->counts_pending.p, 0, (size_t)c->n_counts * 8));                // counts of this call: committed only if the whole call succeeds
    uint64_t chunk_reads = KJ_CHUNK_READS;
    if (const char* v = getenv("KJ_CHUNK_READS")) { long x = atol(v); if (x >= 1024 && x <= (1 << 24)) chunk_reads = (uint64_t)x; }       // tuning hook
    if (o.acc || o.frag) {
        if (o.acc && !c->dix.sa_acc) { kj_err() = "kj_classify_verbose2: the context was created without kj_index_view.seq_accession"; return KJ_ERR_UNSUPPORTED; }
        if ((o.acc && !o.nacc) || (o.frag && (!o.fraglen || o.frag_stride < 16))) { kj_err() = "kj_classify_verbose2: null argument"; return KJ_ERR_ARG; }
    }
    // per-read arrays of both slots, for the largest chunk
    const size_t reads = std::min<uint64_t>(n, chunk_reads); int rc;
    for (KjSlot& S : c->slot) {
        if ((rc = S.off[0].grow((reads + 1) * sizeof(uint64_t))) || (rc = S.off[1].grow((reads + 1) * sizeof(uint64_t))) ||
            (rc = S.tax.grow(reads * sizeof(uint64_t))) || (rc = S.best.grow(reads * sizeof(uint32_t)))) return rc;
        if (o.ids && ((rc = S.ids.grow(reads * KJ_MAX_IDS * sizeof(uint64_t))) || (rc = S.nids.grow(reads)))) return rc;
        if (o.acc && ((rc = S.acc.grow(reads * KJ_MAX_MATCH_ACC * 4)) || (rc = S.nacc.grow(reads)))) return rc;
        if (o.frag && ((rc = S.frag.grow(reads * (size_t)o.frag_stride)) || (rc = S.fraglen.grow(reads * 4)))) return rc;
    }
    // software pipeline over chunks: H2D + kernel + D2H of chunk k on stream k&1 overlap with chunk k+1
    const bool trace = getenv("KJ_TRACE") != nullptr;            // developer hook: per-chunk timeline on stderr
    struct Tr { cudaEvent_t e[4]; double host_ms; uint64_t cnt; }; std::vector<Tr> tr; cudaEvent_t tr0 = nullptr; const auto th0 = std::chrono::steady_clock::now();
    if (trace) { cudaEventCreate(&tr0); cudaEventRecord(tr0, c->slot[0].stream); }
    for (uint64_t start = 0, k = 0, cnt = 0; start < n; start += cnt, k++) {
        KjSlot& S = c->slot[k & 1]; cudaStream_t st = S.stream;
        cnt = std::min<uint64_t>(chunk_reads, n - start);
        // long reads: bound the bases per chunk as well (at least one read)
        {
            const uint64_t* e1p = std::upper_bound(off1 + start + 1, off1 + start + cnt + 1, off1[start] + KJ_CHUNK_BYTES);
            uint64_t lim = std::max<uint64_t>(1, (uint64_t)(e1p - (off1 + start + 1)));
            if (paired) { const uint64_t* e2p = std::upper_bound(off2 + start + 1, off2 + start + cnt + 1, off2[start] + KJ_CHUNK_BYTES); lim = std::min(lim, std::max<uint64_t>(1, (uint64_t)(e2p - (off2 + start + 1)))); }
            cnt = std::min(cnt, lim);
        }
        // Reads that need the long-read kernels run in chunks of their own, so that the short reads of the call keep the short kernels and their
        // full grid: a chunk is either a stretch without long reads, or it starts at a long read (or at fewer than KJ_LONG_GAP short reads before
        // one) and ends where KJ_LONG_GAP short reads in a row follow; the few short reads inside it run on the long kernels with the same results.
        bool long_chunk = false;
        if (!longs.empty()) {
            auto it = std::lower_bound(longs.begin(), longs.end(), start);
            const uint64_t nl = it == longs.end() ? n : *it;
            if (nl == n || nl - start >= KJ_LONG_GAP) cnt = std::min(cnt, nl - start);
            else {
                long_chunk = true; uint64_t e = nl + 1;
                for (auto jt = it + 1; e - start < cnt; ++jt) { const uint64_t nx = jt == longs.end() ? n : *jt; if (nx == n || nx - e >= KJ_LONG_GAP) break; e = nx + 1; }
                cnt = std::min(cnt, e - start);
            }
        }
        CK(cudaStreamSynchronize(st));                      // slot s free again (its previous D2H has landed)
        if (trace) { Tr t; for (auto& e : t.e) cudaEventCreate(&e); t.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - th0).count(); t.cnt = 0; tr.push_back(t); cudaEventRecord(tr.back().e[0], st); }
        const uint64_t b1 = off1[start], e1 = off1[start + cnt], b2 = paired ? off2[start] : 0, e2 = paired ? off2[start + cnt] : 0;
        const size_t bytes1 = (size_t)(e1 - b1), bytes2 = (size_t)(e2 - b2);      // staging bases with 1/8 slack
        if ((rc = S.seq[0].grow(bytes1, bytes1 + bytes1 / 8 + 4096)) || (rc = S.seq[1].grow(bytes2, bytes2 + bytes2 / 8 + 4096))) return rc;
        CK(cudaMemcpyAsync(S.seq[0].p, seq1 + b1, bytes1, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(S.off[0].p, off1 + start, (cnt + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
        if (paired) {
            CK(cudaMemcpyAsync(S.seq[1].p, seq2 + b2, bytes2, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(S.off[1].p, off2 + start, (cnt + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
        }
        if (trace) { tr.back().cnt = cnt; cudaEventRecord(tr.back().e[1], st); }
        KjOut d;
        d.tax = S.tax.as<uint64_t>(); d.best = o.best ? S.best.as<uint32_t>() : nullptr; d.compact = o.compact ? o.compact + start : nullptr;
        if (o.ids) { d.ids = S.ids.as<uint64_t>(); d.nids = S.nids.as<uint8_t>(); }
        if (o.acc) { d.acc = S.acc.as<uint32_t>(); d.nacc = S.nacc.as<uint8_t>(); }
        if (o.frag) { d.frag = S.frag.as<char>(); d.fraglen = S.fraglen.as<uint32_t>(); }
        d.frag_stride = o.frag_stride; d.counts = c->counts_pending.as<unsigned long long>();
        if ((rc = launch(c, (int)(k & 1), S.seq[0].as<uint8_t>(), S.off[0].as<uint64_t>(), paired ? S.seq[1].as<uint8_t>() : nullptr, paired ? S.off[1].as<uint64_t>() : nullptr,
                         b1, b2, cnt, long_chunk ? max1 : smax1, long_chunk ? max2 : smax2, d, st, true))) return rc;
        if (trace) cudaEventRecord(tr.back().e[2], st);
        CK(cudaMemcpyAsync(o.tax + start, d.tax, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        if (o.best) CK(cudaMemcpyAsync(o.best + start, d.best, cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        if (o.ids) {
            CK(cudaMemcpyAsync(o.ids + start * KJ_MAX_IDS, d.ids, cnt * KJ_MAX_IDS * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(o.nids + start, d.nids, cnt, cudaMemcpyDeviceToHost, st));
        }
        if (o.acc) {
            CK(cudaMemcpyAsync(o.acc + start * KJ_MAX_MATCH_ACC, d.acc, cnt * KJ_MAX_MATCH_ACC * 4, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(o.nacc + start, d.nacc, cnt, cudaMemcpyDeviceToHost, st));
        }
        if (o.frag) {
            CK(cudaMemcpyAsync(o.frag + start * (size_t)o.frag_stride, d.frag, cnt * (size_t)o.frag_stride, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(o.fraglen + start, d.fraglen, cnt * 4, cudaMemcpyDeviceToHost, st));
        }
    }
    if (trace && !tr.empty()) cudaEventRecord(tr.back().e[3], c->slot[(tr.size() - 1) & 1].stream);
    CK(cudaStreamSynchronize(c->slot[0].stream)); CK(cudaStreamSynchronize(c->slot[1].stream));
    if (trace) {
        fprintf(stderr, "KJ_TRACE chunk reads host_issue_ms h2d_start h2d_end kernel_end (ms since call start, device)\n");
        for (size_t k = 0; k < tr.size(); k++) { float a = 0, b = 0, d = 0; cudaEventElapsedTime(&a, tr0, tr[k].e[0]); cudaEventElapsedTime(&b, tr0, tr[k].e[1]); cudaEventElapsedTime(&d, tr0, tr[k].e[2]);
            fprintf(stderr, "KJ_TRACE %zu %llu %.2f %.2f %.2f %.2f\n", k, (unsigned long long)tr[k].cnt, tr[k].host_ms, a, b, d); }
        fprintf(stderr, "KJ_TRACE end host %.2f ms\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - th0).count());
    }
    rc = check_err_flag(c);
    // the per-taxon counts of this call become visible only if the whole call succeeded (a repeated call must not count twice)
    if (rc) { CK(cudaMemset(c->counts_pending.p, 0, (size_t)c->n_counts * 8)); return rc; }
    kj_count_commit<<<c->sm_count, 256, 0, c->slot[0].stream>>>(c->counts.as<unsigned long long>(), c->counts_pending.as<unsigned long long>(), c->n_counts); c->launches++;
    CK(cudaStreamSynchronize(c->slot[0].stream));
    return KJ_OK;
}

// A full Greedy variant ring (flag 4) enlarges the ring for the next launch: repeat the call until it fits (bounded).
static int classify_host_retry(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n, const KjOut& o) {
    for (;;) {
        const uint32_t boost = c ? c->variant_boost : 0;
        int rc = classify_host(c, seq1, off1, seq2, off2, n, o);
        if (rc != KJ_ERR_OVERFLOW || !c || c->variant_boost == boost) return rc;
    }
}

extern "C" int kj_classify(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                           uint64_t* taxon_out, uint32_t* best_out) {
    return classify_host_retry(c, seq1, off1, seq2, off2, n, KjOut{taxon_out, best_out});
}
extern "C" int kj_classify2(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                            uint64_t* taxon_out, uint32_t* best_out, uint32_t* d_compact_out) {
    return classify_host_retry(c, seq1, off1, seq2, off2, n, KjOut{taxon_out, best_out, d_compact_out});
}
// In-process multi-GPU (the drop-in counterpart of the reference's `-z N` consumer threads, kaiju.cpp:250-257): contiguous shards of the batch,
// one host thread per context, results written straight into the caller's arrays.  No exchange between the GPUs: reads are independent.
extern "C" int kj_classify_multi(kj_ctx** ctxs, int n_ctx, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                                 uint64_t* taxon_out, uint32_t* best_out) {
    if (!ctxs || n_ctx < 1 || !seq1 || !off1 || !taxon_out || (seq2 && !off2)) { kj_err() = "kj_classify_multi: null argument"; return KJ_ERR_ARG; }
    for (int i = 0; i < n_ctx; i++) if (!ctxs[i]) { kj_err() = "kj_classify_multi: null context"; return KJ_ERR_ARG; }
    if (n_ctx == 1) return kj_classify(ctxs[0], seq1, off1, seq2, off2, n, taxon_out, best_out);
    std::vector<int> rc((size_t)n_ctx, KJ_OK); std::vector<std::string> msg((size_t)n_ctx); std::vector<std::thread> th;
    for (int i = 0; i < n_ctx; i++) th.emplace_back([&, i] {
        const uint64_t lo = n * (uint64_t)i / (uint64_t)n_ctx, hi = n * (uint64_t)(i + 1) / (uint64_t)n_ctx;
        if (hi > lo) rc[(size_t)i] = kj_classify(ctxs[i], seq1, off1 + lo, seq2, seq2 ? off2 + lo : nullptr, hi - lo, taxon_out + lo, best_out ? best_out + lo : nullptr);
        if (rc[(size_t)i]) msg[(size_t)i] = kj_err();
    });
    for (auto& x : th) x.join();
    for (int i = 0; i < n_ctx; i++) if (rc[(size_t)i]) { kj_err() = "device " + std::to_string(ctxs[i]->device) + ": " + msg[(size_t)i]; return rc[(size_t)i]; }
    return KJ_OK;
}
extern "C" int kj_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }
extern "C" int kj_classify_verbose(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n,
                                   uint64_t* taxon_out, uint32_t* best_out, uint64_t* ids_out, uint8_t* nids_out) {
    if (!ids_out || !nids_out) { kj_err() = "kj_classify_verbose: null argument"; return KJ_ERR_ARG; }
    return classify_host_retry(c, seq1, off1, seq2, off2, n, KjOut{taxon_out, best_out, nullptr, ids_out, nids_out});
}

extern "C" int kj_classify_verbose2(kj_ctx* c, const char* seq1, const uint64_t* off1, const char* seq2, const uint64_t* off2, uint64_t n, uint64_t* taxon_out, uint32_t* best_out,
                                    uint64_t* ids_out, uint8_t* nids_out, uint32_t* acc_out, uint8_t* nacc_out, char* frag_out, uint32_t frag_stride, uint32_t* frag_len_out) {
    if (!ids_out || !nids_out || !best_out) { kj_err() = "kj_classify_verbose2: null argument"; return KJ_ERR_ARG; }
    return classify_host_retry(c, seq1, off1, seq2, off2, n, KjOut{taxon_out, best_out, nullptr, ids_out, nids_out, acc_out, nacc_out, frag_out, frag_stride, frag_len_out});
}
extern "C" uint64_t kj_kernel_launches(const kj_ctx* c) { return c ? c->launches : 0; }
extern "C" uint64_t kj_index_bytes(const kj_ctx* c) { return c ? c->index_bytes : 0; }
extern "C" uint64_t kj_index_host_bytes(const kj_ctx* c) { return c ? c->host_bytes : 0; }
extern "C" int kj_index_layout(const kj_ctx* c) { return c ? c->H.wide : -1; }
// The string tables kj_classify_files prints (accessions of `kaiju -v`, the front-ends' sequence names): where sa_acc goes, i.e. in HBM or, when
// the context has a host tier, in mapped pinned host memory (a name table of an nr-scale index is GBs; the format pass reads a few strings per read).
extern "C" int kj_set_output_strings(kj_ctx* c, int kind, const char* blob, const uint64_t* off, uint64_t n) {
    if (!c || !off || (kind != KJ_STR_ACCESSION && kind != KJ_STR_TAXON)) { kj_err() = "kj_set_output_strings: null argument or unknown kind"; return KJ_ERR_ARG; }
    if (kind == KJ_STR_TAXON && n + 1 != c->n_counts) { kj_err() = "kj_set_output_strings: the taxon table needs kj_counts_size() - 1 = " + std::to_string(c->n_counts - 1) + " strings"; return KJ_ERR_ARG; }
    for (uint64_t k = 0; k < n; k++) if (off[k + 1] < off[k]) { kj_err() = "kj_set_output_strings: offsets must not decrease"; return KJ_ERR_ARG; }
    if (off[0] != 0 || (off[n] && !blob)) { kj_err() = "kj_set_output_strings: off[0] must be 0 and blob hold off[n] bytes"; return KJ_ERR_ARG; }
    CK(cudaSetDevice(c->device)); CK(cudaDeviceSynchronize());       // no kernel reads the table being replaced
    KjTierBuf& S = c->out_str[kind]; KjTierBuf& O = c->out_off[kind]; const bool host = c->sa_tax.on_host;
    (S.on_host ? c->host_bytes : c->index_bytes) -= c->out_bytes[kind];
    S.dev.reset(); S.host.reset(); O.dev.reset(); O.host.reset(); c->out_bytes[kind] = 0; c->out_n[kind] = 0; c->out_have[kind] = false;
    S.on_host = O.on_host = host;
    const size_t sb = std::max<size_t>((size_t)off[n], 16), ob = (size_t)(n + 1) * 8;
    for (KjTierBuf* b : {&S, &O}) {
        const size_t need = b == &S ? sb : ob;
        if (b->grow(need) != KJ_OK) {
            cudaGetLastError(); S.dev.reset(); S.host.reset();
            char m[240]; snprintf(m, sizeof m, "kj_set_output_strings: could not allocate %zu bytes of %s for the %s table (%llu strings, %llu bytes of text)", need,
                                  host ? "pinned host memory" : "device memory", kind == KJ_STR_ACCESSION ? "accession" : "taxon label", (unsigned long long)n, (unsigned long long)off[n]);
            kj_err() = m; return KJ_ERR_NOMEM;
        }
    }
    int rc; if ((off[n] && (rc = S.put(blob, (size_t)off[n]))) || (rc = O.put(off, ob))) return rc;
    c->out_bytes[kind] = sb + ob; (host ? c->host_bytes : c->index_bytes) += sb + ob;
    c->out_n[kind] = n; c->out_have[kind] = true;
    return KJ_OK;
}
extern "C" double kj_last_kernel_ms(const kj_ctx* c) {
    if (!c) return 0.0;
    float ms = 0.f; if (cudaEventSynchronize(c->ev_b) != cudaSuccess) return 0.0;
    if (cudaEventElapsedTime(&ms, c->ev_a, c->ev_b) != cudaSuccess) return 0.0;
    return (double)ms;
}
extern "C" int kj_counts_reset(kj_ctx* c) {
    if (!c) return KJ_ERR_ARG; CK(cudaSetDevice(c->device));
    CK(cudaMemset(c->counts.p, 0, (size_t)c->n_counts * 8)); return KJ_OK;
}
extern "C" uint64_t kj_counts_size(const kj_ctx* c) { return c ? c->n_counts : 0; }
extern "C" void* kj_counts_device_ptr(kj_ctx* c) { return c ? c->counts.p : nullptr; }
extern "C" int kj_counts_add_device(kj_ctx* c, const uint64_t* d_taxon, uint64_t n, void* cuda_stream) {
    if (!c || (!d_taxon && n)) { kj_err() = "kj_counts_add_device: null argument"; return KJ_ERR_ARG; }
    CK(cudaSetDevice(c->device)); return count_taxa(c, d_taxon, n, c->counts.as<unsigned long long>(), (cudaStream_t)cuda_stream);
}
extern "C" int kj_counts_get(kj_ctx* c, uint64_t* taxon_ids_out, uint64_t* counts_out) {
    if (!c || !counts_out) { kj_err() = "kj_counts_get: null argument"; return KJ_ERR_ARG; }
    CK(cudaSetDevice(c->device)); CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(counts_out, c->counts.p, (size_t)c->n_counts * 8, cudaMemcpyDeviceToHost));
    if (taxon_ids_out) { for (uint32_t i = 0; i + 1 < c->n_counts; i++) taxon_ids_out[i] = c->H.tax_id[i]; taxon_ids_out[c->n_counts - 1] = 0; }
    return KJ_OK;
}
extern "C" int kj_counts_table(kj_ctx* c, const char* nodes_dmp, const char* names_dmp, const char* label, const kj_table_opts* opts, const char* out_path, int append) {
    if (!c) { kj_err() = "kj_counts_table: null argument"; return KJ_ERR_ARG; }
    std::vector<uint64_t> ids(c->n_counts), cnt(c->n_counts);
    int rc = kj_counts_get(c, ids.data(), cnt.data()); if (rc) return rc;
    return kj_table_write(ids.data(), cnt.data(), c->n_counts, nodes_dmp, names_dmp, label, opts, out_path, append);
}
extern "C" int kj_check_errors(kj_ctx* c) { if (!c) return KJ_ERR_ARG; cudaSetDevice(c->device); return check_err_flag(c); }
extern "C" int kj_launch_geometry(const kj_ctx* c, int* grid, int* block, int* smem) { if (!c) return KJ_ERR_ARG; if (grid) *grid = c->grid; if (block) *block = KJ_WARPS_PER_CTA * 32; if (smem) *smem = (int)c->smem_bytes; return KJ_OK; }

#include "kj_ingest.h"
