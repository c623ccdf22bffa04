// kj_warp.h -- the warp-collective vocabulary the classification kernels are written in.
//
// Device build (nvcc, sm_90a): thin wrappers over the SIMT intrinsics (full-mask collectives).
// KJ_EMU build (g++, tests/emu only): the same member functions implemented on a 32-fiber
// cooperative scheduler, so the *identical* kernel source (kj_core.h) can be exercised on a machine
// without a GPU.  The emulator is test infrastructure; the product library never compiles with KJ_EMU.
#pragma once
#include <stdint.h>

#if defined(KJ_EMU)
// ------------------------------------------------------------------ emulation (tests only)
#include <string.h>
#define KJ_DEV inline
#define KJ_HD inline
#define KJ_ROLLED
#define KJ_NOINLINE static
namespace kjemu {
struct Sched;                         // defined in tests/emu/kj_emu.cpp
uint64_t rendezvous(Sched* s, int lane, uint64_t v, int src_kind, int src_arg);
uint32_t rendezvous_ballot(Sched* s, int lane, bool p);
}
static inline int kj_popc(uint32_t x) { return __builtin_popcount(x); }
static inline int kj_popcll(uint64_t x) { return __builtin_popcountll(x); }
static inline int kj_ffs(uint32_t x) { return __builtin_ffs((int)x); }
static inline int kj_clz(uint32_t x) { return x ? __builtin_clz(x) : 32; }
static inline uint32_t kj_funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
static inline uint32_t kj_vcmpeq4(uint32_t a, uint32_t b) { uint32_t r = 0; for (int i = 0; i < 4; i++) if (((a >> (8 * i)) & 0xffu) == ((b >> (8 * i)) & 0xffu)) r |= 0xffu << (8 * i); return r; }
static inline double kj_dadd(double a, double b) { volatile double r = a + b; return r; }
static inline double kj_dsub(double a, double b) { volatile double r = a - b; return r; }
static inline double kj_dmul(double a, double b) { volatile double r = a * b; return r; }
struct Warp {
    int lane;
    kjemu::Sched* s;
    KJ_DEV uint32_t ballot(bool p) const { return kjemu::rendezvous_ballot(s, lane, p); }
    KJ_DEV bool any(bool p) const { return ballot(p) != 0; }
    KJ_DEV bool all(bool p) const { return ballot(p) == 0xffffffffu; }
    KJ_DEV void sync() const { (void)kjemu::rendezvous_ballot(s, lane, false); }
    KJ_DEV uint64_t shfl64(uint64_t v, int src) const { return kjemu::rendezvous(s, lane, v, 0, src & 31); }
    KJ_DEV uint64_t shfl_xor64(uint64_t v, int m) const { return kjemu::rendezvous(s, lane, v, 1, m); }
    KJ_DEV uint32_t shfl(uint32_t v, int src) const { return (uint32_t)shfl64(v, src); }
    KJ_DEV int shfl(int v, int src) const { return (int)(uint32_t)shfl64((uint32_t)v, src); }
    KJ_DEV uint32_t shfl_xor(uint32_t v, int m) const { return (uint32_t)shfl_xor64(v, m); }
    KJ_DEV int shfl_xor(int v, int m) const { return (int)(uint32_t)shfl_xor64((uint32_t)v, m); }
    KJ_DEV double shfl_d(double v, int src) const { uint64_t u; memcpy(&u, &v, 8); u = shfl64(u, src); memcpy(&v, &u, 8); return v; }
    KJ_DEV uint32_t redux_max(uint32_t v) const { for (int m = 16; m > 0; m >>= 1) { uint32_t o = shfl_xor(v, m); v = o > v ? o : v; } return v; }
    KJ_DEV uint32_t redux_min(uint32_t v) const { for (int m = 16; m > 0; m >>= 1) { uint32_t o = shfl_xor(v, m); v = o < v ? o : v; } return v; }
};
#else
// ------------------------------------------------------------------ device (product)
#define KJ_DEV __device__ __forceinline__
#define KJ_HD __host__ __device__ __forceinline__
#define KJ_FULL 0xffffffffu
// Code size is a first-order cost here (the Greedy kernel stalls on instruction fetch when its hot loop outgrows the instruction cache):
// loops are kept rolled unless unrolling was measured to pay, and cold paths are real functions.
#define KJ_ROLLED _Pragma("unroll 1")
#define KJ_NOINLINE static __device__ __noinline__
static KJ_DEV int kj_popc(uint32_t x) { return __popc(x); }
static KJ_DEV int kj_popcll(uint64_t x) { return __popcll(x); }
static KJ_DEV int kj_ffs(uint32_t x) { return __ffs((int)x); }
static KJ_DEV int kj_clz(uint32_t x) { return __clz((int)x); }
static KJ_DEV uint32_t kj_funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) { return __funnelshift_r(lo, hi, sh); }
static KJ_DEV uint32_t kj_vcmpeq4(uint32_t a, uint32_t b) { return __vcmpeq4(a, b); }
// SEG's FP64 must round exactly like the reference's scalar x86 code: no FMA contraction.
static KJ_DEV double kj_dadd(double a, double b) { return __dadd_rn(a, b); }
static KJ_DEV double kj_dsub(double a, double b) { return __dsub_rn(a, b); }
static KJ_DEV double kj_dmul(double a, double b) { return __dmul_rn(a, b); }
struct Warp {
    int lane;
    KJ_DEV uint32_t ballot(bool p) const { return __ballot_sync(KJ_FULL, p); }
    KJ_DEV bool any(bool p) const { return __any_sync(KJ_FULL, p); }
    KJ_DEV bool all(bool p) const { return __all_sync(KJ_FULL, p); }
    KJ_DEV void sync() const { __syncwarp(KJ_FULL); }
    KJ_DEV uint64_t shfl64(uint64_t v, int src) const { return __shfl_sync(KJ_FULL, (unsigned long long)v, src); }
    KJ_DEV uint64_t shfl_xor64(uint64_t v, int m) const { return __shfl_xor_sync(KJ_FULL, (unsigned long long)v, m); }
    KJ_DEV uint32_t shfl(uint32_t v, int src) const { return __shfl_sync(KJ_FULL, v, src); }
    KJ_DEV int shfl(int v, int src) const { return __shfl_sync(KJ_FULL, v, src); }
    KJ_DEV uint32_t shfl_xor(uint32_t v, int m) const { return __shfl_xor_sync(KJ_FULL, v, m); }
    KJ_DEV int shfl_xor(int v, int m) const { return __shfl_xor_sync(KJ_FULL, v, m); }
    KJ_DEV double shfl_d(double v, int src) const { return __shfl_sync(KJ_FULL, v, src); }
    // redux.sync: one instruction per 32-bit warp reduction (sm_80+)
    KJ_DEV uint32_t redux_max(uint32_t v) const { return __reduce_max_sync(KJ_FULL, v); }
    KJ_DEV uint32_t redux_min(uint32_t v) const { return __reduce_min_sync(KJ_FULL, v); }
};
#endif

// collectives built on the primitives (identical in both builds)
static KJ_DEV uint32_t warp_max_u32(const Warp& w, uint32_t v) { return w.redux_max(v); }
static KJ_DEV int warp_max_i32(const Warp& w, int v) { return (int)(w.redux_max((uint32_t)v ^ 0x80000000u) ^ 0x80000000u); }
static KJ_DEV uint32_t warp_min_u32(const Warp& w, uint32_t v) { return w.redux_min(v); }
// 64-bit max as two 32-bit reductions: high words first, then the low words of the lanes that tie on the high word
static KJ_DEV uint64_t warp_max_u64(const Warp& w, uint64_t v) {
    const uint32_t hi = (uint32_t)(v >> 32), mh = w.redux_max(hi);
    const uint32_t ml = w.redux_max(hi == mh ? (uint32_t)v : 0u);
    return ((uint64_t)mh << 32) | ml;
}
static KJ_DEV uint32_t lanemask_lt(int lane) { return (1u << lane) - 1u; }
