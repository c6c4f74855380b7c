// scan_common.cuh -- device code used by more than one scan kernel (scan_small.cu, scan_fast.cu, and the ring and
// cluster kernels of scan_tma.cu): the per-scan outcome record, the Mode B output slots, the 64 KB presence byte
// map with its rank table, and the Mode A bin-ownership logic.
#pragma once
#include "rpl_device.cuh"
#include "scan_args.h"

namespace rpl {
namespace {

constexpr uint32_t kWords = kKeySpace / 32;     // 2048 bitmap words
constexpr uint32_t kMaxFastNodes = kKeySpace;   // more nodes cannot be tie-free

// ---- the per-scan outcome (one thread writes it) ----------------------------------------------------------------
__device__ __forceinline__ void write_outcome(const ScanBatchArgs& a, uint32_t s, uint32_t status, uint32_t beams,
                                              float inc) {
  if (a.status) a.status[s] = status;
  if (a.path) a.path[s] = 0u;
  if (a.beam_counts) a.beam_counts[s] = beams;
  if (a.angle_inc) a.angle_inc[s] = inc;
}
// no measured node: ascendScanData returns OPERATION_FAIL and leaves the buffer untouched; publish_scan publishes
// nothing
__device__ __forceinline__ void write_outcome_empty(const ScanBatchArgs& a, uint32_t s) {
  write_outcome(a, s, a.apply_ascend ? kResultOperationFail : kResultOk, 0u, 0.0f);
}
// where scan s's ascended buffer goes: its row, or its placed position (ScanBatchArgs::out_first)
__device__ __forceinline__ uint2* nodes_out_of(const ScanBatchArgs& a, uint32_t s) {
  return a.nodes_out + (a.out_first ? (size_t)a.out_first[s] : (size_t)s * a.stride);
}
// a placed launch's scan that is another kernel's (or nobody's): nothing is read or written for it
__device__ __forceinline__ bool out_skipped(const ScanBatchArgs& a, uint32_t s) {
  return a.out_first && (a.out_first[s] & kOutSkip) != 0;
}
// scan s goes to the general kernel, which runs after this one and follows the stable tie rule
__device__ __forceinline__ void hand_to_general(const ScanBatchArgs& a, uint32_t s) {
  a.fallback_list[atomicAdd(a.fallback_count, 1u)] = s;
}

// predicated streaming stores (no branch around them)
__device__ __forceinline__ void st_f32_if(float* p, float v, uint64_t pol, uint32_t pred) {
  asm volatile(
      "{ .reg .pred q; setp.ne.u32 q, %3, 0;\n\t"
      "@q st.global.L1::no_allocate.L2::cache_hint.f32 [%0], %1, %2; }" ::"l"(p),
      "f"(v), "l"(pol), "r"(pred));
}

// ---- Mode B output (reference rplidar_node.cpp:661-677) ---------------------------------------------------------
// The point of rank r among the M measured points goes to slot ob + os * r in wrapping u32 arithmetic (reference
// :673); intensities[] sits at a fixed byte distance from ranges[].
// The stores carry L2 policy `pol` (evict_first unless the kernel passes another).
struct ModeBOut {
  float* ranges;
  ptrdiff_t i_minus_r;
  uint32_t ob, os;
  uint64_t pol;
  __device__ __forceinline__ ModeBOut(float* r, float* i, uint32_t M, bool inverted,
                                      uint64_t policy = l2_policy_evict_first())
      : ranges(r),
        i_minus_r(reinterpret_cast<char*>(i) - reinterpret_cast<char*>(r)),
        ob(inverted ? M - 1u : 0u),
        os(inverted ? 0xFFFFFFFFu : 1u),
        pol(policy) {}
  __device__ __forceinline__ void store(uint32_t rank, float dist_m, float intensity, uint32_t pred) const {
    float* pr = ranges + (ob + os * rank);
    st_f32_if(pr, dist_m, pol, pred);
    st_f32_if(reinterpret_cast<float*>(reinterpret_cast<char*>(pr) + i_minus_r), intensity, pol, pred);
  }
};

// ---- the presence byte map of scan_fast.cu and scan_tma.cu --------------------------------------------------------
// One byte per key, marked with plain byte stores, then folded to bit-words by kMapThreads threads: thread t owns
// keys [128 t, 128 t + 128), a 128-byte row of eight 16-byte columns.
constexpr int kMapThreads = 512;
constexpr int kMapWarps = kMapThreads / 32;
constexpr uint32_t kWordsPerThread = kWords / kMapThreads;  // 4 bit-words per row

// barrier of the kMapThreads threads (named barrier 1: the TMA kernels' producer warp stays out)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kMapThreads) : "memory"); }

// address swizzle: within a row the 16-byte column is XORed with row & 7, so that the 128-bit reads of 8
// neighbouring threads in the fold hit 8 different bank groups.  Takes the raw first word of a node (key in the
// low 16 bits).
__device__ __forceinline__ uint32_t swz_x(uint32_t x) { return (x ^ ((x >> 3) & 0x70u)) & 0xFFFFu; }
// bit 0 of each of the four bytes of x -> bits 0..3
__device__ __forceinline__ uint32_t gather4(uint32_t x) { return (x * 0x10204080u) >> 28; }

__device__ __forceinline__ void bytemap_clear(uint8_t* bytemap, uint32_t tid) {
  uint4* bm = reinterpret_cast<uint4*>(bytemap);
  const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (uint32_t j = 0; j < kKeySpace / 16 / kMapThreads; ++j) bm[j * kMapThreads + tid] = z;
}

// fold: thread tid gathers bit 0 of the presence bytes of its row into its kWordsPerThread bit-words
__device__ __forceinline__ void fold_row(const uint8_t* bytemap, uint32_t tid, uint32_t (&wv)[kWordsPerThread]) {
#pragma unroll
  for (uint32_t j = 0; j < kWordsPerThread; ++j) wv[j] = 0;
  const uint4* bm = reinterpret_cast<const uint4*>(bytemap);
#pragma unroll
  for (uint32_t c = 0; c < 8; ++c) {
    const uint4 q = bm[tid * 8 + (c ^ (tid & 7u))];  // physical column of logical chunk c
    const uint32_t x[4] = {q.x, q.y, q.z, q.w};
    uint32_t bv = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) bv |= gather4(x[j] & 0x01010101u) << (4 * j);
    wv[c >> 1] |= bv << (16 * (c & 1));
  }
}

// Rank table from the folded bit-words, by all kMapThreads threads (two consumer_sync barriers inside):
// sm.rankV[w] = {bits of word w, set bits in the words below w}.  On entry sm.red[0 .. kMapWarps) holds the warps'
// measured counts; sm.red[2 kMapWarps .. 3 kMapWarps) is scratch.  Sets sm.totV to the set bits of the whole table and
// sm.valid_count to the measured count plus `extra_count`.  Read them after a further barrier.
template <class Smem>
__device__ __forceinline__ void rank_table(Smem& sm, const uint32_t (&wv)[kWordsPerThread], uint32_t tid,
                                           uint32_t extra_count) {
  const uint32_t lane = tid & 31, warp = tid >> 5;
  uint32_t sv = 0;
#pragma unroll
  for (uint32_t j = 0; j < kWordsPerThread; ++j) sv += __popc(wv[j]);
  const uint32_t iv = warp_inclusive_scan(sv);
  if (lane == 31) sm.red[2 * kMapWarps + warp] = iv;
  consumer_sync();
  if (warp == 0) {
    uint32_t tv = lane < kMapWarps ? sm.red[2 * kMapWarps + lane] : 0u;
    uint32_t cc = lane < kMapWarps ? sm.red[lane] : 0u;
    const uint32_t cv = warp_inclusive_scan(tv);
    cc = warp_sum(cc);
    if (lane < kMapWarps) sm.red[2 * kMapWarps + lane] = cv - tv;
    if (lane == 31) {
      sm.totV = cv;
      sm.valid_count = cc + extra_count;
    }
  }
  consumer_sync();
  uint32_t pv = sm.red[2 * kMapWarps + warp] + iv - sv;
#pragma unroll
  for (uint32_t j = 0; j < kWordsPerThread; ++j) {
    sm.rankV[tid * kWordsPerThread + j] = make_uint2(wv[j], pv);
    pv += __popc(wv[j]);
  }
}

__device__ __forceinline__ uint32_t rank_of(const uint2* rk, uint32_t key) {
  const uint2 e = rk[key >> 5];
  return e.y + __popc(e.x & ((1u << (key & 31)) - 1u));
}

// ---- Mode A (reference rplidar_node.cpp:630-660) ------------------------------------------
// beam_count = M bins; every measured point goes to bin (int)(angle / angle_increment) and the
// bin keeps the smallest dist_m (strict '<': on equal dist_m the first point in ascending key
// order, i.e. the smallest key).
//
// Bins grow with the key -- for inverted scans along "key 0 first, then descending keys" -- so in
// that order (the "u-order") the points of a bin are neighbours.  The place pass of scan_fast.cu
// and scan_tma.cu therefore records every measured point at its u-rank, ordered by
//     entry = dist_m bits << 32 | key << 8 | quality          (u64 min = min (dist_m, key))
// and the emit pass (mode_a_emit, mode_a_emit_smem) walks the entries in order: every warp owns a
// contiguous slice, finds the runs of equal bins, takes their minimum, and writes each bin exactly
// once (empty bins included) with converged, mostly coalesced stores.  No atomics, no block-wide
// barriers inside the walk.
__device__ __forceinline__ uint32_t mode_a_urank(uint32_t key, uint32_t rank, uint32_t M, bool inverted,
                                                 bool has0) {
  if (!inverted) return rank;
  if (key == 0u) return 0u;
  return (M - 1u - rank) + (has0 ? 1u : 0u);
}
__device__ __forceinline__ unsigned long long mode_a_entry(float dist_m, uint32_t key, uint32_t quality) {
  return ((unsigned long long)__float_as_uint(dist_m) << 32) | ((unsigned long long)key << 8) |
         (unsigned long long)quality;
}

struct ModeAOut {
  float* ranges;
  float* intens;
  const float2* angle;  // [65536] (angle, inverted angle) table
  uint32_t M;
  float inc;
  bool inverted, new_proto;
  uint64_t policy;
};

__device__ __forceinline__ void mode_a_store_bin(const ModeAOut& o, int bin, unsigned long long best, uint32_t pred) {
  const float dm = __uint_as_float((uint32_t)(best >> 32));
  const float it = quality_to_intensity((uint32_t)best & 0xFFu, o.new_proto);
  st_f32_if(o.ranges + bin, dm, o.policy, pred);
  st_f32_if(o.intens + bin, it, o.policy, pred);
}
__device__ __forceinline__ void mode_a_fill_empty(const ModeAOut& o, int from, int to) {  // bins [from, to)
  const float kInf = __int_as_float(0x7f800000);
  for (int e = from; e < to; ++e) {
    o.ranges[e] = kInf;
    o.intens[e] = 0.0f;
  }
}

}  // namespace
}  // namespace rpl
