// decode_formats.cu -- the measurement answer formats on the GPU (SURVEY.md 8(f) rank 1).
//
// Replaces, for framed capsules (reference src/sdk/src/dataunpacker/unpacker/):
//   0x82 express      UnpackerHandler_CapsuleNode            handler_capsules.cpp:109-266  (84 B -> 32 nodes)
//   0x84 ultra        UnpackerHandler_UltraCapsuleNode       handler_capsules.cpp:324-580  (132 B -> 96 nodes)
//   0x85 dense        UnpackerHandler_DenseCapsuleNode       handler_capsules.cpp:639-791  (84 B -> 40 nodes)
//   0x86 ultra-dense  UnpackerHandler_UltraDenseCapsuleNode  handler_capsules.cpp:852-1047 (170 B -> 64 nodes)
//   0x83 HQ           UnpackerHandler_HQNode                 handler_hqnode.cpp:93-172     (781 B -> 96 nodes)
// and, for raw byte streams,
//   0x81 standard     UnpackerHandler_NormalNode             handler_normalnode.cpp:88-141 (5 B -> 1 node)
//
// The reference decodes capsules byte by byte in a state machine: a capsule's nodes are produced when the NEXT
// capsule arrives (angles are interpolated between the two start angles), and only if both checksums hold and the
// next capsule is not a scan start (dense, ultra-dense: and the angular step is below the 100 Hz bound).  Here the
// capsule formats but HQ share one kernel, decode_capsule_kernel<F> (one CTA per stream, tiles of 256 capsules
// staged through shared memory, one thread per capsule for frame / checksum / "does this capsule release its
// predecessor", an exclusive block scan for the node offsets, then emission in the format's own grain -- a thread
// per pair of samples (one 16-byte store) for express and dense, a warp per capsule with a lane per cabin for ultra
// (3 samples) and ultra-dense (2 samples) -- into one contiguous run of the output).  What differs besides is the
// state that crosses capsules:
//   * express / ultra: none (the scan-start flag of a node is a function of its angle only);
//   * dense / ultra-dense: the last node's scan-start flag (the reference's lastNodeSyncBit,
//     sync_i = raw_i & ~sync_{i-1}), carried across capsules as a 2-bit transfer function per capsule,
//     scanned under composition;
//   * ultra-dense besides: `_last_dist_q2`, a smoothing recurrence over
//     neighbouring short-range samples.  A capsule's effect on that value is a function of at most
//     nine candidate inputs (the first sample either ignores the incoming value or averages with
//     one of 17 neighbours -> 9 results), so every capsule thread tabulates its nine outcomes, one
//     thread chains the tables across the tile, and the capsule threads then replay, from the now-known
//     input, the samples before the position where their nine candidates merged (the others were final
//     already).
// The standard-node decoder is a 5-state byte machine with resynchronisation; each thread folds its
// 30 bytes into a state->state map (5 x 3 bits), the maps are scanned under composition, and the
// threads replay their bytes from the known entry state: exact on arbitrary (misframed) streams.
#include "decode_args.h"
#include "rpl_device.cuh"

namespace rpl {

// The stream-list instantiations (a mixed byte session's launches over the streams of one answer type, StreamList) are
// compiled from this file in a translation unit of their own, decode_list.cu, with RPL_DECODE_LIST defined: there every
// stream session kernel takes a StreamList l too, CTA slot i serves stream l.streams[i] of the chunk, and the capsule
// decoders read each stream's capsules l.capsule_stride bytes apart.  Spelled as macros, so that the kernels of this
// translation unit stay token for token what they were and compile to the same code.
#ifdef RPL_DECODE_LIST
#define RPL_LIST_PARAM , StreamList l
#define RPL_LIST_ARG , l
#define RPL_FOR_STREAMS(s) \
  for (uint32_t i_ = blockIdx.x; i_ < a.n_streams; i_ += gridDim.x) if (const uint32_t s = l.streams[i_]; true)
#define RPL_STREAM_CAPSULES(s, cb) (size_t)s * l.capsule_stride
#else
#define RPL_LIST_PARAM
#define RPL_LIST_ARG
#define RPL_FOR_STREAMS(s) for (uint32_t s = blockIdx.x; s < a.n_streams; s += gridDim.x)
#define RPL_STREAM_CAPSULES(s, cb) (size_t)s * a.stride_capsules * cb
#endif
cudaError_t launch_decode_capsules_list(uint32_t ans_type, const CapsuleDecodeArgs& a, const StreamList& l, int grid,
                                        cudaStream_t stream);
cudaError_t launch_decode_normal_list(const NormalDecodeArgs& a, const StreamList& l, int grid, cudaStream_t stream);
cudaError_t decode_list_configure();

namespace {

// threads = capsules per tile: Fmt<F>::DT (smaller tiles where the per-capsule state is large: more CTAs per SM, so a
// few hundred streams are all in flight at once instead of queueing for a second wave)
constexpr uint32_t kStOk = 1, kStSync = 2, kStEmit = 4, kStDiscard = 8, kStChecksum = 16, kStEncReset = 32,
                   kStBadFrame = 64;
constexpr int kFull = 360 << 16;

enum { kExpress = 0, kUltra = 1, kUltraDense = 2, kDense = 3 };

// CB bytes and NODES nodes per capsule, the start angle at byte START, BUFFERS tile buffers of DT capsules (= threads).
// JUMP_CABINS: the cabin count in the reference's angular-jump discard threshold (0: no threshold).  SYNC_CHAIN: the
// last node's scan-start flag crosses capsules; SMOOTH_CHAIN: so does the smoothed last distance.
template <int F>
struct Fmt;
template <>
struct Fmt<kExpress> {
  static constexpr int CB = 84, NODES = 32, START = 2, BUFFERS = 2, DT = 256, JUMP_CABINS = 0;
  static constexpr bool SYNC_CHAIN = false, SMOOTH_CHAIN = false;
};
template <>
struct Fmt<kUltra> {
  // one tile buffer (more CTAs per SM instead of a prefetch: the emission is instruction-bound)
  static constexpr int CB = 132, NODES = 96, START = 2, BUFFERS = 1, DT = 256, JUMP_CABINS = 0;
  static constexpr bool SYNC_CHAIN = false, SMOOTH_CHAIN = false;
};
template <>
struct Fmt<kDense> {
  static constexpr int CB = 84, NODES = 40, START = 2, BUFFERS = 2, DT = 256, JUMP_CABINS = 40;
  static constexpr bool SYNC_CHAIN = true, SMOOTH_CHAIN = false;
};
template <>
struct Fmt<kUltraDense> {
  // one tile buffer: with the smoothing tables a second one would leave a single CTA (8 warps) per SM
  static constexpr int CB = 170, NODES = 64, START = 8, BUFFERS = 1, DT = 128, JUMP_CABINS = 32;
  static constexpr bool SYNC_CHAIN = true, SMOOTH_CHAIN = true;
};

__device__ __forceinline__ uint32_t ld16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
__device__ __forceinline__ uint32_t ld32(const uint8_t* p) { return ld16(p) | (ld16(p + 2) << 16); }

__device__ __forceinline__ uint2 pack_node(int angle_q6, uint32_t dist_q2, uint32_t sync, uint32_t quality) {
  if (angle_q6 < 0) angle_q6 += (360 << 6);
  if (angle_q6 >= (360 << 6)) angle_q6 -= (360 << 6);
  // angle_q6 >= 0 here for every wire input (start angles are 15-bit q6 values < 512 deg and the interpolated angle
  // minus its correction stays above -360 deg), so the unsigned quotient is the reference's signed one
  const uint32_t key = ((uint32_t)(angle_q6 << 8) / 90u) & 0xFFFFu;
  const uint32_t flag = sync | ((sync ^ 1u) << 1);
  uint2 nd;
  nd.x = key | (dist_q2 << 16);
  nd.y = (dist_q2 >> 16) | ((quality & 0xFFu) << 16) | (flag << 24);
  return nd;
}

__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}

// ---- express (handler_capsules.cpp:206-266) ---------------------------------------------------------
// both samples of one 5-byte cabin: angle interpolation in q16, per-sample offset (6 bits: 4 from the shared byte, 2 from
// the distance word), scan start = the interpolated angle wraps within this sample's step
__device__ __forceinline__ void cabin_express(const uint8_t* prev, int prev_q8, int diff_q8, uint32_t cabin, uint2& na,
                                              uint2& nb) {
  const int inc = diff_q8 << 3;
  const int a0 = (prev_q8 << 8) + (int)(2u * cabin) * inc, a1 = a0 + inc;
  const uint8_t* cab = prev + 4 + 5 * cabin;
  const uint32_t d0 = ld16(cab), d1 = ld16(cab + 2), ob = cab[4];
  const int off0 = (int)((ob & 0xFu) | ((d0 & 3u) << 4)), off1 = (int)((ob >> 4) | ((d1 & 3u) << 4));
  int rem = a1 % kFull;  // (a0 + inc) % full
  const uint32_t sync0 = (rem < inc) ? 1u : 0u;
  if (inc >= 0 && inc < kFull) {
    rem += inc;
    if (rem >= kFull) rem -= kFull;
  } else {
    rem = (a1 + inc) % kFull;
  }
  const uint32_t sync1 = (rem < inc) ? 1u : 0u;
  const uint32_t q0 = d0 & 0xFFFCu, q1 = d1 & 0xFFFCu;
  na = pack_node((a0 - (off0 << 13)) >> 10, q0, sync0, q0 ? (0x2Fu << 2) : 0u);
  nb = pack_node((a1 - (off1 << 13)) >> 10, q1, sync1, q1 ? (0x2Fu << 2) : 0u);
}

// ---- dense (handler_capsules.cpp:736-791) --------------------------------------------------------------
// samples 2 * pair and 2 * pair + 1: one 32-bit word of 16-bit distances, the angle interpolated in q16 (inc: step
// per sample), the two resolved scan-start flags in sync2
__device__ __forceinline__ void pair_dense(const uint8_t* prev, int prev_q8, int inc, uint32_t pair, uint32_t sync2,
                                           uint2& na, uint2& nb) {
  const int a0 = (prev_q8 << 8) + (int)(2u * pair) * inc;
  const uint32_t w = *reinterpret_cast<const uint32_t*>(prev + 4 + 4 * pair);
  const uint32_t q0 = (w & 0xFFFFu) << 2, q1 = (w >> 16) << 2;
  na = pack_node(a0 >> 10, q0, sync2 & 1u, q0 ? (0x2Fu << 2) : 0u);
  nb = pack_node((a0 + inc) >> 10, q1, sync2 >> 1, q1 ? (0x2Fu << 2) : 0u);
}

// ---- the scan-start chain (dense :768-769, ultra-dense) ---------------------------------------------------
// raw scan-start test of the N interpolated samples of a capsule as a bit mask.  One real modulo, then a running
// remainder: inc_q16 < 360 deg (the jump threshold keeps the step per sample far below a revolution), so a single
// conditional subtraction per step suffices.
template <int N>
__device__ __forceinline__ unsigned long long raw_sync_mask(int prev_q8, int inc_q16) {
  unsigned long long m = 0;
  int rem = ((prev_q8 << 8) + inc_q16) % kFull;  // (cur + inc) % full for pos = 0
  const int lim = inc_q16 << 1;
  // no wrap inside the capsule and already past the two steps after the last one: nothing to mark (most capsules)
  if (rem >= lim && rem + (N - 1) * inc_q16 < kFull) return 0ull;
#pragma unroll 8
  for (int pos = 0; pos < N; ++pos) {
    if (rem < lim) m |= 1ull << pos;
    rem += inc_q16;
    if (rem >= kFull) rem -= kFull;
  }
  return m;
}
// sync_i = raw_i & ~sync_{i-1}, sync_{-1} = s_in; only set raw bits matter
__device__ __forceinline__ unsigned long long resolve_sync(unsigned long long raw, uint32_t s_in) {
  unsigned long long s = 0, r = raw;
  while (r) {
    const int i = __ffsll((long long)r) - 1;
    r &= r - 1;
    const uint32_t prev = (i == 0) ? s_in : (uint32_t)((s >> (i - 1)) & 1ull);
    if (!prev) s |= 1ull << i;
  }
  return s;
}

// ---- ultra (handler_capsules.cpp:422-580) --------------------------------------------------------------
__device__ int g_ultra_offset[493];  // read through L1 (divergent index: not constant memory)

// One warp per released capsule, one lane per cabin (3 nodes): the two cabin words (aligned 32-bit loads: capsules
// are 132 bytes and tiles 16-byte aligned), both variable-bit-scale expansions and the base/level selection are done
// once per cabin instead of once per node; the scan-start test needs one modulo per cabin (the other two remainders
// follow by addition whenever the angle step is in [0, 360 deg)); the 493-entry angle-correction table is read from
// shared memory.  The three nodes of a lane go through a per-warp staging area so that the warp stores its 96 nodes
// as three fully coalesced 256-byte rows.
// Per cabin (handler_capsules.cpp:470-540): major = varbitscale(x3 & 0xFFF), the next cabin's major2 likewise; the
// two predictions are the signed 10-bit fields of x3 (-512 and 511 mean "no measurement"); sample 0 is major,
// sample 1 = predict1 << level1 + base1 (base1/level1 fall back to the next cabin's when major is 0), sample 2 =
// predict2 << level2 + major2; all << 2.  The angle correction depends on the distance only through
// k2 = 98361 / dist_q2 in [0, 491] (dist_q2 >= 200): a 493-entry table built on the host with the reference's own
// double arithmetic (entry 492 = the short-range default).
__device__ __forceinline__ uint32_t varbitscale_sel(uint32_t s, uint32_t& level) {
  // segment of s (< 4096): the bounds 512, 1280, 1792, 3328 are multiples of 256 -> 16 nibbles indexed by s >> 8
  const uint32_t l = (uint32_t)(0x4443333332211100ull >> (4u * (s >> 8))) & 0xFu;
  // source bases of the five segments (12 bits each); target bases 0, 1<<9, 1<<11, 1<<12, 1<<14
  const uint32_t src = (uint32_t)(0xD00700500200000ull >> (12u * l)) & 0xFFFu;
  const uint32_t dst = (l ? 512u : 0u) << ((0x53200u >> (4u * l)) & 0xFu);
  level = l;
  return dst + ((s - src) << l);
}
__device__ __forceinline__ void ultra_cabin(const uint8_t* prev, const uint8_t* cur, int prev_q8, int diff_q8,
                                            uint32_t cabin, const int* off_table, uint2* stage) {
  const int inc = (diff_q8 << 3) / 3;
  const uint32_t x3 = *reinterpret_cast<const uint32_t*>(prev + 4 + 4 * cabin);
  const uint32_t nx = (cabin == 31u) ? *reinterpret_cast<const uint32_t*>(cur + 4)
                                     : *reinterpret_cast<const uint32_t*>(prev + 8 + 4 * cabin);
  uint32_t lvl1, lvl2;
  const uint32_t major = varbitscale_sel(x3 & 0xFFFu, lvl1);
  const uint32_t major2 = varbitscale_sel(nx & 0xFFFu, lvl2);
  uint32_t base1 = major;
  if (!major && major2) {
    base1 = major2;
    lvl1 = lvl2;
  }
  const int p1 = (int)(x3 << 10) >> 22, p2 = (int)x3 >> 22;
  int dist[3];
  dist[0] = (int)(major << 2);
  dist[1] = (p1 == -512 || p1 == 511) ? 0 : (int)((((uint32_t)p1 << lvl1) + base1) << 2);
  dist[2] = (p2 == -512 || p2 == 511) ? 0 : (int)((((uint32_t)p2 << lvl2) + major2) << 2);
  const int a0 = (prev_q8 << 8) + (int)(3u * cabin) * inc;
  const bool step_ok = inc >= 0 && inc < kFull;  // warp-uniform
  int rem = (a0 + inc) % kFull;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int a = a0 + c * inc;
    if (c > 0) {
      if (step_ok) {
        rem += inc;
        if (rem >= kFull) rem -= kFull;
      } else {
        rem = (a + inc) % kFull;
      }
    }
    const uint32_t sync = (rem < inc) ? 1u : 0u;
    uint32_t k2 = 492u;
    if (dist[c] >= 200) {
      // 98361 / dist_q2 (<= 491) without the integer division: both operands are exact floats (dist_q2 < 2^22) and
      // the correctly rounded quotient cannot reach an integer the exact one stays below (it would have to be within
      // 98361/d * 2^-24 of it, but misses it by at least 1/d): truncation gives the integer quotient.
      // tests/test_device_math_proofs.py checks every dist_q2.
      k2 = __float2uint_rz(__fdiv_rn(98361.0f, __uint2float_rn((uint32_t)dist[c])));
    }
    const int angle_q6 = (a - off_table[k2]) >> 10;
    stage[3u * cabin + c] = pack_node(angle_q6, (uint32_t)dist[c], sync, dist[c] ? (0x2Fu << 2) : 0u);
  }
}

// ---- ultra-dense (handler_capsules.cpp:951-1047) -------------------------------------------------------
// raw sample: distance before smoothing, scale code, quality
__device__ __forceinline__ int ud_decode(uint32_t qds, uint32_t& scale, uint32_t& quality);
__device__ __forceinline__ int ud_sample(const uint8_t* cap, uint32_t pos, uint32_t& scale, uint32_t& quality) {
  const uint8_t* cab = cap + 10 + 5 * (pos >> 1);
  const uint32_t hi = cab[4];
  const uint32_t qds = ld16(cab + 2 * (pos & 1u)) | (((pos & 1u) ? (hi >> 4) : (hi & 0xFu)) << 16);
  return ud_decode(qds, scale, quality);
}
__device__ __forceinline__ int ud_decode(uint32_t qds, uint32_t& scale, uint32_t& quality) {
  scale = qds & 3u;
  // the four ranges without a branch (scales differ from lane to lane): field mask 0xFFC / 0x1FFC / 0x3FFC / 0x7FFC,
  // factor 2..5, base (0, 2046, 8187, 24567) << 2, quality (qds >> (12 + scale)) << scale
  const uint32_t base = (uint32_t)(((24567ull << 45) | (8187ull << 30) | (2046ull << 15)) >> (15u * scale)) & 0x7FFFu;
  quality = ((qds >> (12u + scale)) << scale) & 0xFFu;
  return (int)((qds & ((0x1000u << scale) - 4u)) * (scale + 2u) + (base << 2));
}
__device__ __forceinline__ int ud_smooth(int raw, uint32_t scale, int last) {
  if (scale == 0 && last && abs(raw - last) <= 8) return (raw + last) >> 1;
  return raw;
}

template <int F>
struct CapsuleSmem {
  static constexpr int CB = Fmt<F>::CB, DT = Fmt<F>::DT;
  static constexpr int SYNC = Fmt<F>::SYNC_CHAIN ? DT : 1, SMOOTH = Fmt<F>::SMOOTH_CHAIN ? DT : 1;
  static constexpr int kTileBytes = (DT * CB + 15) & ~15;
  uint8_t cap[Fmt<F>::BUFFERS][kTileBytes];  // tiles (double-buffered: cp.async prefetch of the next one)
  uint8_t carry[(CB + 15) & ~15];      // last capsule of the previous tile
  uint32_t start_q8[DT + 1];           // slot 0 = carry
  uint32_t okflag[DT + 1];
  uint32_t emit_list[DT];
  uint32_t warp_a[DT / 32], warp_b[DT / 32];
  uint32_t carry_nodes, tile_nodes;
  unsigned long long smask[SYNC];      // scan-start chain: final flags of the nodes each capsule releases
  // smoothing chain
  uint32_t ud_out[SMOOTH][10];         // nine outcomes of the smoothing chain + first raw sample
  uint32_t ud_first_scale[SMOOTH];     // bit 31: the capsule's outcome does not depend on its input
  uint32_t ud_last_in[SMOOTH];
  uint16_t ud_dist[SMOOTH][66];  // smoothed short-range distances (rows padded to 33 words: a thread per capsule walks a column)
  uint32_t carry_sync, red_sync, n_starts, carry_last, red_last;
  // ultra only: angle-correction table and the per-warp staging rows of the emission
  int ultra_off[F == kUltra ? 496 : 1];
  uint2 wstage[F == kUltra ? DT / 32 : 1][F == kUltra ? 96 : 1];
  // dense only: angular step per sample of the nodes each capsule releases
  int inc_q16[F == kDense ? DT : 1];
};

// STREAM: a stream session's instantiation (CapsuleDecodeArgs::node_stride != 0).  The held record stands in for the
// previous tile's last capsule and its state (sm.carry, okflag[0], start_q8[0], carry_sync, carry_last), so a push
// boundary is decoded as a tile boundary is.
template <int F, bool STREAM>
__global__ void __launch_bounds__(Fmt<F>::DT) decode_capsule_kernel(CapsuleDecodeArgs a RPL_LIST_PARAM) {
  using T = Fmt<F>;
  constexpr int CB = T::CB, NODES = T::NODES, DT = T::DT;
  constexpr bool DENSE = F == kDense;
  constexpr uint32_t kCarryWords = (CB + 3) / 4;  // whole words of the held capsule (ultra-dense: 170 -> 172 bytes)
  static_assert(kCarryWords <= kHeldCapsuleWords && 4 * kCarryWords <= sizeof(CapsuleSmem<F>::carry), "held capsule");
  extern __shared__ __align__(16) unsigned char capsule_smem_raw[];
  CapsuleSmem<F>& sm = *reinterpret_cast<CapsuleSmem<F>*>(capsule_smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int thr_q8 = 0;
  if (T::JUMP_CABINS) thr_q8 = (360 * 100 * T::JUMP_CABINS / (int)(1000000u / a.sample_duration_us)) << 8;
  if constexpr (F == kUltra) {
    for (uint32_t i = tid; i < 493u; i += DT) sm.ultra_off[i] = g_ultra_offset[i];
    __syncthreads();
  }

  RPL_FOR_STREAMS(s) {
    if constexpr (STREAM && T::JUMP_CABINS != 0)
      if (a.lidars) thr_q8 = (360 * 100 * T::JUMP_CABINS / (int)(1000000u / a.lidars[s].timing.sample_duration_us)) << 8;
    const uint32_t n = STREAM ? min(a.counts[s], a.stride_capsules) : a.counts[s];
    const uint8_t* src = a.capsules + RPL_STREAM_CAPSULES(s, CB);
    uint2* out = STREAM ? a.nodes_out + (size_t)s * a.node_stride + a.node_first
                        : a.nodes_out + (size_t)s * a.stride_capsules * NODES;
    uint32_t* st_out = a.capsule_status ? a.capsule_status + (size_t)s * a.stride_capsules : nullptr;
    uint32_t* off_out = a.capsule_node_offset ? a.capsule_node_offset + (size_t)s * a.stride_capsules : nullptr;
    uint32_t* starts = a.scan_starts ? a.scan_starts + (size_t)s * a.starts_stride : nullptr;
    const uint32_t* state_in = a.state_in ? a.state_in + (size_t)s * a.state_words : nullptr;
    if (tid == 0) {
      sm.carry_nodes = 0;
      sm.okflag[0] = 0;
      sm.start_q8[0] = 0;
      if constexpr (T::SYNC_CHAIN) sm.carry_sync = state_in ? (state_in[0] & 1u) : 0u;
      if constexpr (DENSE) sm.n_starts = 0;
      if constexpr (T::SMOOTH_CHAIN) sm.carry_last = (state_in && a.state_words == 2) ? state_in[1] : 0u;
      if constexpr (STREAM) {
        const uint32_t* held = a.held + (size_t)s * kHeldWords;
        sm.okflag[0] = held[kHeldOk];
        sm.start_q8[0] = held[kHeldStart];
        if constexpr (T::SYNC_CHAIN) sm.carry_sync = held[kHeldSync];
        if constexpr (T::SMOOTH_CHAIN) sm.carry_last = held[kHeldLast];
      }
    }
    // the held capsule takes the place of a previous tile's last capsule: the first capsule releases it if both hold
    // (ultra: its last cabin reads cabin 0 of that first capsule)
    if constexpr (STREAM)
      for (uint32_t w = tid; w < kCarryWords; w += DT)
        reinterpret_cast<uint32_t*>(sm.carry)[w] = a.held[(size_t)s * kHeldWords + w];
    __syncthreads();

    // stage a tile into buffer `b`: asynchronous 16-byte copies, 4-byte ones where the stream is only 4-byte aligned
    auto stage = [&](uint32_t c0, uint32_t b) {
      const uint32_t live = min((uint32_t)DT, n - c0);
      const uint32_t bytes = live * CB;
      const uint8_t* g = src + (size_t)c0 * CB;
      uint32_t done = 0;
      if ((reinterpret_cast<uintptr_t>(g) & 15u) == 0) {
        const uint32_t quads = bytes >> 4;
        for (uint32_t q = tid; q < quads; q += DT) cp_async16(&sm.cap[b][16 * q], g + 16 * q);
        done = quads << 4;
      } else if ((reinterpret_cast<uintptr_t>(g) & 3u) == 0) {
        const uint32_t words = bytes >> 2;
        for (uint32_t w = tid; w < words; w += DT) cp_async4(&sm.cap[b][4 * w], g + 4 * w);
        done = words << 2;
      }
      for (uint32_t w = done + tid; w < bytes; w += DT) sm.cap[b][w] = __ldg(g + w);
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (T::BUFFERS == 2 && n > 0) stage(0, 0);
    uint32_t buf = 0;
    for (uint32_t c0 = 0; c0 < n; c0 += DT, buf ^= (uint32_t)(T::BUFFERS - 1)) {
      const uint32_t live = min((uint32_t)DT, n - c0);
      if (T::BUFFERS == 1) stage(c0, 0);  // the previous tile was released by the barrier that ends its iteration
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      if (T::BUFFERS == 2 && c0 + DT < n) stage(c0 + DT, buf ^ 1u);
      const uint8_t* tile = sm.cap[buf];
      // ---- per capsule: frame, checksum, start angle ------------------------------------------------
      uint32_t st = 0, ok = 0, sync = 0;
      if (tid < live) {
        const uint8_t* c = tile + tid * CB;  // 2-byte aligned at least (CB even, tiles 16-byte aligned)
        const uint32_t b0 = c[0], b1 = c[1];
        const uint32_t start = ld16(c + T::START);
        if ((b0 >> 4) != 0xA || (b1 >> 4) != 0x5) {
          st = kStBadFrame;
        } else {
          uint32_t x = 0;
          if constexpr (CB % 4 == 0) {  // 32-bit words (half the loads of the 16-bit loop)
            const uint32_t* w = reinterpret_cast<const uint32_t*>(c);
            x = w[0] >> 16;
#pragma unroll
            for (int k = 1; k < CB / 4; ++k) x ^= w[k];
            x ^= x >> 16;
          } else {
            const uint16_t* h = reinterpret_cast<const uint16_t*>(c);
#pragma unroll 8
            for (int k = 1; k < CB / 2; ++k) x ^= h[k];
          }
          const uint32_t sum = (x ^ (x >> 8)) & 0xFFu;
          const uint32_t recv = ((b0 & 0xFu) | (b1 << 4)) & 0xFFu;
          if (recv != sum) {
            st = kStChecksum;
          } else {
            ok = 1;
            st = kStOk;
            sync = (start >> 15) & 1u;
            if (sync) st |= kStSync;
          }
        }
        sm.okflag[tid + 1] = ok;
        sm.start_q8[tid + 1] = (start & 0x7FFFu) << 2;
      }
      __syncthreads();
      // ---- does this capsule release its predecessor? ---------------------------------------------
      uint32_t emit = 0;
      int prev_q8 = 0, diff = 0;
      if (tid < live && ok) {
        const uint32_t prev_ok = sm.okflag[tid];
        if (sync) {
          if (prev_ok) st |= kStEncReset;
        } else if (prev_ok) {
          const int cur_q8 = (int)sm.start_q8[tid + 1];
          prev_q8 = (int)sm.start_q8[tid];
          diff = cur_q8 - prev_q8;
          if (prev_q8 > cur_q8) diff += (360 << 8);
          if (T::JUMP_CABINS && diff > thr_q8) {
            st |= kStDiscard;
          } else {
            emit = 1;
            st |= kStEmit;
          }
        }
      }
      const uint32_t inc_scan = warp_inclusive_scan(emit);
      if (lane == 31) sm.warp_a[warp] = inc_scan;
      // scan-start chain: transfer function of the flag through this capsule, f(s_in) = s_out
      unsigned long long raw = 0;
      uint32_t Fsync = 0x2;  // identity: f(0) = 0 (bit 0), f(1) = 1 (bit 1)
      if constexpr (T::SYNC_CHAIN) {
        uint32_t f = 0x2;
        if (emit) {
          const int inc_q16 = (diff << 8) / NODES;
          raw = raw_sync_mask<NODES>(prev_q8, inc_q16);
          if constexpr (DENSE) sm.inc_q16[tid] = inc_q16;  // the emission's step, once per capsule
          const uint32_t o0 = (uint32_t)(resolve_sync(raw, 0) >> (NODES - 1)) & 1u;
          const uint32_t o1 = (uint32_t)(resolve_sync(raw, 1) >> (NODES - 1)) & 1u;
          f = o0 | (o1 << 1);
        }
        // inclusive scan of the functions under composition: (g o f)(x) = g(f(x))
        Fsync = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t p = __shfl_up_sync(0xffffffffu, Fsync, o);
          if (lane >= (uint32_t)o) Fsync = ((Fsync >> (p & 1u)) & 1u) | (((Fsync >> ((p >> 1) & 1u)) & 1u) << 1);
        }
        if (lane == 31) sm.warp_b[warp] = Fsync;
      }
      __syncthreads();
      uint32_t base_off = 0, s_state = T::SYNC_CHAIN ? sm.carry_sync : 0u;
      for (uint32_t w = 0; w < warp; ++w) {
        base_off += sm.warp_a[w];
        if (T::SYNC_CHAIN) s_state = (sm.warp_b[w] >> s_state) & 1u;
      }
      const uint32_t my_off = base_off + inc_scan - emit;
      unsigned long long smask = 0;
      if constexpr (T::SYNC_CHAIN) {
        // flag entering this capsule: everything before it in the warp
        const uint32_t Fprev = __shfl_up_sync(0xffffffffu, Fsync, 1);
        const uint32_t s_in = (lane == 0) ? s_state : ((Fprev >> s_state) & 1u);
        if (emit) smask = resolve_sync(raw, s_in);
        if (tid < live) sm.smask[tid] = smask;
      }
      if (tid < live) {
        const uint32_t node_off = sm.carry_nodes + (uint32_t)NODES * my_off;
        if (emit) sm.emit_list[my_off] = tid;
        if (st_out) st_out[c0 + tid] = st;
        if (off_out) off_out[c0 + tid] = node_off;
        // this capsule's scan-start nodes (a few per revolution), for the assembler.  Only the dense entry points
        // offer the list: compiled into ultra-dense, the loop alone takes that kernel from 40 to 32 registers and
        // makes it slower
        if (DENSE && starts) {
          for (; smask; smask &= smask - 1) {
            const uint32_t idx = atomicAdd(&sm.n_starts, 1u);
            if (idx < a.starts_stride) starts[idx] = node_off + (uint32_t)(__ffsll((long long)smask) - 1);
          }
        }
      }
      if (tid == DT - 1) {
        uint32_t tot = 0, st2 = T::SYNC_CHAIN ? sm.carry_sync : 0u;
        for (uint32_t w = 0; w < DT / 32; ++w) {
          tot += sm.warp_a[w];
          if (T::SYNC_CHAIN) st2 = (sm.warp_b[w] >> st2) & 1u;
        }
        sm.tile_nodes = (uint32_t)NODES * tot;
        if (T::SYNC_CHAIN) sm.red_sync = st2;
      }
      // first sample position from which this capsule's smoothed distances no longer depend on the value that
      // enters the capsule (the nine candidates have merged): step 1 stores those directly, step 3 replays only
      // the positions before it
      uint32_t ud_pm = 64;
      if constexpr (T::SMOOTH_CHAIN) {
        // ---- smoothing chain, step 1: the nine outcomes of this capsule's 64 samples ------------------
        if (emit) {
          const uint8_t* pc = (tid == 0) ? sm.carry : tile + (tid - 1) * CB;
          uint32_t sc, q;
          const int r0 = ud_sample(pc, 0, sc, q);
          const uint32_t sc_first = sc;
          int cand[9];
#pragma unroll
          for (int k = 0; k < 9; ++k) cand[k] = (sc == 0) ? (r0 - 4 + k) : r0;
          bool merged = (sc != 0);
          if (merged) {
            ud_pm = 0;
            sm.ud_dist[tid][0] = (uint16_t)r0;
          }
          // two loops: with nine candidates until they merge (usually at once), then the plain recurrence, unrolled
          // so that the decodes of the next samples overlap the dependent smoothing steps
          uint32_t pos = 1;
          for (; pos < 64 && !merged; ++pos) {
            const int r = ud_sample(pc, pos, sc, q);
            int lo = 0x7fffffff, hi = -0x7fffffff;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
              cand[k] = ud_smooth(r, sc, cand[k]);
              lo = min(lo, cand[k]);
              hi = max(hi, cand[k]);
            }
            merged = (lo == hi);
            if (merged) {
              ud_pm = pos;
              sm.ud_dist[tid][pos] = (uint16_t)cand[0];
            }
          }
          int last = cand[0];
#pragma unroll 8
          for (; pos < 64; ++pos) {
            uint32_t s2, q2;
            const int r = ud_sample(pc, pos, s2, q2);
            last = ud_smooth(r, s2, last);
            sm.ud_dist[tid][pos] = (uint16_t)last;  // only read back for scale-0 samples (< 8192)
          }
          if (merged) cand[0] = last;
#pragma unroll
          for (int k = 0; k < 9; ++k) sm.ud_out[tid][k] = (uint32_t)(merged ? cand[0] : cand[k]);
          sm.ud_out[tid][9] = (uint32_t)r0;
          sm.ud_first_scale[tid] = sc_first | (merged ? 0x80000000u : 0u);
        }
      }
      __syncthreads();
      if constexpr (T::SMOOTH_CHAIN) {
        // ---- step 2: the value entering every releasing capsule.  A capsule whose nine outcomes agree
        // (any far sample inside it) is a constant: each thread walks back to the nearest such capsule (or
        // to the tile's input) and applies the tables from there -- usually one or two steps.
        {
          const uint32_t E = sm.tile_nodes / NODES;
          auto apply = [&](uint32_t j, int last) -> int {
            const uint32_t fs = sm.ud_first_scale[j];
            const int r0 = (int)sm.ud_out[j][9];
            int k = 4;
            if ((fs & 3u) == 0 && last && abs(r0 - last) <= 8) k = ((r0 + last) >> 1) - (r0 - 4);
            return (int)sm.ud_out[j][k];
          };
          if (tid < E) {
            int e0 = (int)tid - 1;  // last capsule before this one whose outcome is known without its input
            while (e0 >= 0 && !(sm.ud_first_scale[sm.emit_list[e0]] & 0x80000000u)) --e0;
            int last = (e0 >= 0) ? (int)sm.ud_out[sm.emit_list[e0]][0] : (int)sm.carry_last;
            for (int e = e0 + 1; e < (int)tid; ++e) last = apply(sm.emit_list[e], last);
            const uint32_t j = sm.emit_list[tid];
            sm.ud_last_in[j] = (uint32_t)last;
            if (tid == E - 1) sm.red_last = (uint32_t)apply(j, last);
          }
          __syncthreads();
          if (tid == 0 && E > 0) sm.carry_last = sm.red_last;
        }
        __syncthreads();
        // ---- step 3: replay the samples that do depend on the input, keep the smoothed distances ------
        if (emit) {
          const uint8_t* pc = (tid == 0) ? sm.carry : tile + (tid - 1) * CB;
          int last = (int)sm.ud_last_in[tid];
          for (uint32_t pos = 0; pos < ud_pm; ++pos) {
            uint32_t sc, q;
            const int r = ud_sample(pc, pos, sc, q);
            last = ud_smooth(r, sc, last);
            sm.ud_dist[tid][pos] = (uint16_t)last;  // only read back for scale-0 samples (< 8192)
          }
        }
        __syncthreads();
      }
      // ---- node-parallel emission: one contiguous run of NODES * E nodes -------------------------------
      if constexpr (F == kUltra) {
        const uint32_t E = sm.tile_nodes / (uint32_t)NODES;
        uint2* o = out + sm.carry_nodes;
        for (uint32_t e = warp; e < E; e += DT / 32) {
          const uint32_t j = sm.emit_list[e];
          const uint8_t* pc = (j == 0) ? sm.carry : tile + (j - 1) * CB;
          const int pq8 = (int)sm.start_q8[j];
          int d = (int)sm.start_q8[j + 1] - pq8;
          if (pq8 > (int)sm.start_q8[j + 1]) d += (360 << 8);
          ultra_cabin(pc, tile + j * CB, pq8, d, lane, sm.ultra_off, sm.wstage[warp]);
          __syncwarp();
          uint2* dst = o + (size_t)e * NODES;
#pragma unroll
          for (uint32_t k = 0; k < 3; ++k) dst[lane + 32u * k] = sm.wstage[warp][lane + 32u * k];
          __syncwarp();
        }
      } else if constexpr (F == kUltraDense) {
        // one warp per released capsule, one lane per 5-byte cabin (two samples): the cabin bytes, the capsule's
        // scan-start mask and the pair of smoothed distances are read once, and a lane stores its two nodes as
        // one 16-byte word -- the warp writes the capsule's 64 nodes as 512 contiguous bytes
        const uint32_t E = sm.tile_nodes / (uint32_t)NODES;
        uint2* o = out + sm.carry_nodes;
        const bool wide = (reinterpret_cast<uintptr_t>(o) & 15u) == 0;
        for (uint32_t e = warp; e < E; e += DT / 32) {
          const uint32_t j = sm.emit_list[e];
          const uint8_t* pc = (j == 0) ? sm.carry : tile + (j - 1) * CB;
          const int pq8 = (int)sm.start_q8[j];
          int d = (int)sm.start_q8[j + 1] - pq8;
          if (pq8 > (int)sm.start_q8[j + 1]) d += (360 << 8);
          const int inc = (d << 8) / 64;
          const uint8_t* cab = pc + 10 + 5 * lane;
          const uint32_t hi = cab[4];
          const uint32_t qa = ld16(cab) | ((hi & 0xFu) << 16), qb = ld16(cab + 2) | ((hi >> 4) << 16);
          uint32_t sa, sb, qua, qub;
          int da = ud_decode(qa, sa, qua), db = ud_decode(qb, sb, qub);
          const uint32_t sm2 = *reinterpret_cast<const uint32_t*>(&sm.ud_dist[j][2 * lane]);  // smoothed pair
          if (sa == 0) da = (int)(sm2 & 0xFFFFu);
          if (sb == 0) db = (int)(sm2 >> 16);
          const uint32_t sy = (uint32_t)(sm.smask[j] >> (2 * lane)) & 3u;
          const int ang = (pq8 << 8) + (int)(2 * lane) * inc;
          const uint2 na = pack_node(ang >> 10, (uint32_t)da, sy & 1u, qua);
          const uint2 nb = pack_node((ang + inc) >> 10, (uint32_t)db, sy >> 1, qub);
          uint2* dst = o + (size_t)e * NODES + 2 * lane;
          if (wide) {
            *reinterpret_cast<uint4*>(dst) = make_uint4(na.x, na.y, nb.x, nb.y);
          } else {
            dst[0] = na;
            dst[1] = nb;
          }
        }
      } else {
        // express, dense: a thread handles one pair of samples (an express cabin, a dense distance word): the
        // capsule look-ups and the capsule bytes are shared and the two nodes leave as one 16-byte store (a
        // capsule's run starts on a multiple of 256 / 320 bytes)
        constexpr uint32_t kPairs = NODES / 2;
        const uint32_t n_pairs = sm.tile_nodes / 2u;
        uint2* o = out + sm.carry_nodes;
        const bool wide = (reinterpret_cast<uintptr_t>(o) & 15u) == 0;
        for (uint32_t p = tid; p < n_pairs; p += DT) {
          const uint32_t e = p / kPairs, pair = p - e * kPairs;
          const uint32_t j = sm.emit_list[e];
          const uint8_t* pc = (j == 0) ? sm.carry : tile + (j - 1) * CB;
          const int pq8 = (int)sm.start_q8[j];
          uint2 na, nb;
          if constexpr (F == kExpress) {
            int d = (int)sm.start_q8[j + 1] - pq8;
            if (pq8 > (int)sm.start_q8[j + 1]) d += (360 << 8);
            cabin_express(pc, pq8, d, pair, na, nb);
          } else {
            pair_dense(pc, pq8, sm.inc_q16[j], pair, (uint32_t)(sm.smask[j] >> (2 * pair)) & 3u, na, nb);
          }
          if (wide) {
            *reinterpret_cast<uint4*>(o + 2u * p) = make_uint4(na.x, na.y, nb.x, nb.y);
          } else {
            o[2u * p] = na;
            o[2u * p + 1u] = nb;
          }
        }
      }
      __syncthreads();
      // ---- carry into the next tile -----------------------------------------------------------------
      for (uint32_t b = tid; b < (uint32_t)CB; b += DT) sm.carry[b] = tile[(live - 1) * CB + b];
      if (tid == 0) {
        sm.okflag[0] = sm.okflag[live];
        sm.start_q8[0] = sm.start_q8[live];
        sm.carry_nodes += sm.tile_nodes;
        if (T::SYNC_CHAIN) sm.carry_sync = sm.red_sync;
      }
      __syncthreads();
    }
    if (tid == 0) {
      if (a.node_counts) a.node_counts[s] = sm.carry_nodes;
      if (a.state_out) {
        uint32_t* state_out = a.state_out + (size_t)s * a.state_words;
        state_out[0] = T::SYNC_CHAIN ? sm.carry_sync : 0u;
        if (a.state_words == 2) state_out[1] = T::SMOOTH_CHAIN ? sm.carry_last : 0u;
      }
      if (DENSE && a.scan_start_counts) a.scan_start_counts[s] = sm.n_starts;
      if constexpr (STREAM) {
        uint32_t* held = a.held + (size_t)s * kHeldWords;
        held[kHeldOk] = sm.okflag[0];
        held[kHeldStart] = sm.start_q8[0];
        if constexpr (T::SYNC_CHAIN) held[kHeldSync] = sm.carry_sync;
        if constexpr (T::SMOOTH_CHAIN) held[kHeldLast] = sm.carry_last;
      }
    }
    // the last capsule is held for the next push (a stream without capsules writes back what it read)
    if constexpr (STREAM)
      for (uint32_t w = tid; w < kCarryWords; w += DT)
        a.held[(size_t)s * kHeldWords + w] = reinterpret_cast<const uint32_t*>(sm.carry)[w];
    __syncthreads();
  }
}

// ---- HQ capsules (handler_hqnode.cpp:93-172): CRC32 + pass-through -----------------------------------
// The CRC (reflected 0x04C11DB7 over the 777 message bytes + the SDK's zero padding to 780, sl_crc.cpp:52-69) is a
// chain of dependent table look-ups.  Two things shorten it: eight bytes per step (slicing-by-8: eight independent
// look-ups + one XOR tree), and FOUR threads per capsule -- the register of a table-driven CRC is linear in (state,
// message), so  raw(s, A || B) = advance_|B|(raw(s, A)) ^ raw(0, B):  the threads take the byte ranges [0,192),
// [192,384), [384,576), [576,780), the first with the initial value 0xFFFFFFFF and the others with 0, and one of them
// combines  advance_204(advance_192(advance_192(r0) ^ r1) ^ r2) ^ r3.  "Advance by N zero bytes" is four look-ups in
// a 4 x 256 table per N, built on the host (hq_tables_init).  A capsule starts at any byte offset (781 bytes apart):
// message words come from aligned words by funnel shift.
constexpr int HC = 32;          // capsules per tile (small tiles: five CTAs per SM, so a few hundred streams are all in flight at once)
constexpr int HT = 4 * HC;      // threads: four per capsule
constexpr int kHqBytes = 781;   // 1 sync + 8 timestamp + 96 * 8 nodes + 4 crc
__device__ uint32_t g_hq_advance[2][4][256];  // [0]: 192 zero bytes, [1]: 204
struct HqSmem {
  uint8_t cap[(HC * kHqBytes + 15) & ~15];
  uint32_t table[8][256];    // slicing-by-8: table[k][b] = CRC register after byte b and k zero bytes
  uint32_t advance[2][4][256];
  uint32_t emit_list[HC];
  uint32_t status[HC], emit[HC];
  uint32_t warp_a[HC / 32];
  uint32_t carry_nodes, tile_nodes;
};

// STREAM: a stream session's instantiation.  HQ capsules carry nothing across capsules (handler_hqnode.cpp:93-172), so
// it differs only in where the nodes go (behind the session's carry slots).
template <bool STREAM>
__global__ void __launch_bounds__(HT) decode_hq_kernel(CapsuleDecodeArgs a RPL_LIST_PARAM) {
  extern __shared__ __align__(16) unsigned char capsule_smem_raw[];
  HqSmem& sm = *reinterpret_cast<HqSmem*>(capsule_smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t i = tid; i < 256; i += HT) {
    uint32_t c = i;
#pragma unroll
    for (int j = 0; j < 8; ++j) c = (c & 1u) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
    sm.table[0][i] = c;
  }
  for (uint32_t i = tid; i < 2 * 4 * 256; i += HT) (&sm.advance[0][0][0])[i] = (&g_hq_advance[0][0][0])[i];
  __syncthreads();
  for (uint32_t i = tid; i < 256; i += HT) {
    uint32_t c = sm.table[0][i];
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      c = (c >> 8) ^ sm.table[0][c & 0xFFu];
      sm.table[k][i] = c;
    }
  }
  __syncthreads();
  auto advance = [&](uint32_t which, uint32_t v) {
    return sm.advance[which][0][v & 0xFFu] ^ sm.advance[which][1][(v >> 8) & 0xFFu] ^ sm.advance[which][2][(v >> 16) & 0xFFu] ^
           sm.advance[which][3][v >> 24];
  };
  RPL_FOR_STREAMS(s) {
    const uint32_t n = STREAM ? min(a.counts[s], a.stride_capsules) : a.counts[s];
    const uint8_t* src = a.capsules + RPL_STREAM_CAPSULES(s, kHqBytes);
    uint2* out = STREAM ? a.nodes_out + (size_t)s * a.node_stride + a.node_first
                        : a.nodes_out + (size_t)s * a.stride_capsules * 96;
    uint32_t* st_out = a.capsule_status ? a.capsule_status + (size_t)s * a.stride_capsules : nullptr;
    uint32_t* off_out = a.capsule_node_offset ? a.capsule_node_offset + (size_t)s * a.stride_capsules : nullptr;
    if (tid == 0) sm.carry_nodes = 0;
    __syncthreads();
    for (uint32_t c0 = 0; c0 < n; c0 += HC) {
      const uint32_t live = min((uint32_t)HC, n - c0);
      const uint32_t bytes = live * kHqBytes;
      const uint8_t* g = src + (size_t)c0 * kHqBytes;
      uint32_t done = 0;
      if ((reinterpret_cast<uintptr_t>(g) & 15u) == 0) {
        const uint32_t quads = bytes >> 4;
        for (uint32_t q = tid; q < quads; q += HT) cp_async16(&sm.cap[16 * q], g + 16 * q);
        done = quads << 4;
      }
      for (uint32_t w = done + tid; w < bytes; w += HT) sm.cap[w] = __ldg(g + w);
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      // ---- CRC: thread (capsule cj, range seg) ---------------------------------------------------------------
      const uint32_t cj = tid >> 2, seg = tid & 3u;
      const uint8_t* c = sm.cap + cj * kHqBytes;
      uint32_t part = 0;
      bool framed = false;
      if (cj < live) {
        framed = (c[0] == 0xA5);
        if (framed) {
          uint32_t crc = (seg == 0) ? 0xFFFFFFFFu : 0u;
          const uintptr_t addr = reinterpret_cast<uintptr_t>(c + 192u * seg);
          const uint32_t* w = reinterpret_cast<const uint32_t*>(addr & ~uintptr_t(3));
          const uint32_t sh = (uint32_t)(addr & 3u) * 8u;
          const int steps = (seg == 3) ? 25 : 24;  // 8 bytes each: 192 bytes, the last range 200 + the tail below
          uint32_t w0 = w[0];
#pragma unroll 2
          for (int k = 0; k < steps; ++k) {
            const uint32_t w1 = w[2 * k + 1], w2 = w[2 * k + 2];
            const uint32_t one = __funnelshift_r(w0, w1, sh) ^ crc, two = __funnelshift_r(w1, w2, sh);
            w0 = w2;
            crc = sm.table[7][one & 0xFFu] ^ sm.table[6][(one >> 8) & 0xFFu] ^ sm.table[5][(one >> 16) & 0xFFu] ^
                  sm.table[4][one >> 24] ^ sm.table[3][two & 0xFFu] ^ sm.table[2][(two >> 8) & 0xFFu] ^
                  sm.table[1][(two >> 16) & 0xFFu] ^ sm.table[0][two >> 24];
          }
          if (seg == 3) {  // byte 776 and three zero bytes
            const uint32_t one = (uint32_t)c[776] ^ crc;
            crc = sm.table[3][one & 0xFFu] ^ sm.table[2][(one >> 8) & 0xFFu] ^ sm.table[1][(one >> 16) & 0xFFu] ^
                  sm.table[0][one >> 24];
          }
          part = crc;
        }
      }
      // the four ranges of a capsule sit in neighbouring lanes
      const uint32_t l0 = lane & ~3u;
      const uint32_t r1 = __shfl_sync(0xffffffffu, part, l0 + 1), r2 = __shfl_sync(0xffffffffu, part, l0 + 2),
                     r3 = __shfl_sync(0xffffffffu, part, l0 + 3);
      if (seg == 0 && cj < live) {
        uint32_t st = kStBadFrame, emit = 0;
        if (framed) {
          uint32_t crc = advance(0, part) ^ r1;
          crc = advance(0, crc) ^ r2;
          crc = advance(1, crc) ^ r3;
          crc ^= 0xFFFFFFFFu;
          if (crc == ld32(c + kHqBytes - 4)) {
            st = kStOk | kStEmit;
            emit = 1;
          } else {
            st = kStChecksum;
          }
        }
        sm.status[cj] = st;
        sm.emit[cj] = emit;
      }
      __syncthreads();
      // ---- node offsets: exclusive scan of the release flags over the tile's capsules (the first two warps) ----
      uint32_t emit = 0, inc_scan = 0;
      if (tid < HC) {
        emit = (tid < live) ? sm.emit[tid] : 0u;
        inc_scan = warp_inclusive_scan(emit);
        if (lane == 31) sm.warp_a[warp] = inc_scan;
      }
      __syncthreads();
      if (tid < HC) {
        uint32_t base_off = 0;
        for (uint32_t w = 0; w < warp; ++w) base_off += sm.warp_a[w];
        const uint32_t my_off = base_off + inc_scan - emit;
        if (tid < live) {
          if (emit) sm.emit_list[my_off] = tid;
          if (st_out) st_out[c0 + tid] = sm.status[tid];
          if (off_out) off_out[c0 + tid] = sm.carry_nodes + 96u * my_off;
        }
        if (tid == HC - 1) sm.tile_nodes = 96u * (base_off + inc_scan);
      }
      __syncthreads();
      const uint32_t n_nodes = sm.tile_nodes;
      uint2* o = out + sm.carry_nodes;
      for (uint32_t q = tid; q < n_nodes; q += HT) {
        const uint32_t e = q / 96u, pos = q - e * 96u;
        const uint8_t* p = sm.cap + sm.emit_list[e] * kHqBytes + 9 + 8 * pos;
        const uintptr_t pa = reinterpret_cast<uintptr_t>(p);
        const uint32_t* pw = reinterpret_cast<const uint32_t*>(pa & ~uintptr_t(3));  // (w2 stays inside the capsule)
        const uint32_t psh = (uint32_t)(pa & 3u) * 8u;
        const uint32_t w0 = pw[0], w1 = pw[1], w2 = pw[2];
        o[q] = make_uint2(__funnelshift_r(w0, w1, psh), __funnelshift_r(w1, w2, psh));
      }
      __syncthreads();
      if (tid == 0) sm.carry_nodes += sm.tile_nodes;
      __syncthreads();
    }
    if (tid == 0) {
      if (a.node_counts) a.node_counts[s] = sm.carry_nodes;
      if (a.state_out) a.state_out[2 * s] = a.state_out[2 * s + 1] = 0u;
    }
    __syncthreads();
  }
}

// ---- standard nodes (handler_normalnode.cpp:88-141): 5-state byte machine ----------------------------
constexpr int NT = 256;       // threads
constexpr int kChunk = 30;    // bytes per thread per tile (a multiple of 5; the replay keeps one bit per byte in a u32)
constexpr int kNormTile = NT * kChunk;
struct NormalSmem {
  uint8_t raw[12 + 4 + kNormTile + 12];  // [12 pad][4 bytes of the previous tile][tile]: the tile starts 16-byte aligned
  uint32_t warp_f[NT / 32], warp_c[NT / 32];
  uint16_t ends[kNormTile / 5 + 8];   // tile-relative index of each record's last byte
  uint32_t carry_state, carry_nodes, tile_nodes, red_state;
};
// packed state->state map: 3 bits per entry, entry s = image of state s
constexpr uint32_t kIdentityMap = 0 | (1 << 3) | (2 << 6) | (3 << 9) | (4 << 12);
__device__ __forceinline__ uint32_t byte_map(uint32_t b) {
  const uint32_t t0 = (((b >> 1) ^ b) & 1u);      // state 0: sync bit and its inverse
  const uint32_t t1 = (b & 1u) ? 2u : 0u;         // state 1: check bit
  return t0 | (t1 << 3) | (3u << 6) | (4u << 9);  // 2 -> 3, 3 -> 4, 4 -> 0
}
// (g o f)(s) = g(f(s))
__device__ __forceinline__ uint32_t compose_map(uint32_t g, uint32_t f) {
  uint32_t r = 0;
#pragma unroll
  for (int s = 0; s < 5; ++s) r |= ((g >> (3u * ((f >> (3 * s)) & 7u))) & 7u) << (3 * s);
  return r;
}

// STREAM: a stream session's instantiation (NormalDecodeArgs::node_stride != 0).  The held record's state and last four
// bytes take the place of a previous tile's (carry_state and the halo), so a record begun in an earlier push completes
// in this one's first bytes, read through the halo like a record spanning two tiles.
// STARTS (a stamped session push, STREAM only): node_end [n_streams][node_stride - node_first] gets the push-relative
// index of the last byte of the scan-start records alone, at their node index (a few stores per revolution)
template <bool STREAM, bool STARTS>
__device__ __forceinline__ void decode_normal_body(const NormalDecodeArgs& a RPL_LIST_PARAM) {
  static_assert(STREAM || !STARTS, "the scan-start ends are a stream session's");
  __shared__ __align__(16) NormalSmem sm;
  uint8_t* const sm_bytes = sm.raw + 12;  // bytes[0..3] = halo, bytes + 4 = the tile
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  RPL_FOR_STREAMS(s) {
    const uint32_t n = STREAM ? min(a.byte_counts[s], a.stride_bytes) : a.byte_counts[s];
    const uint8_t* src = a.bytes + (size_t)s * a.stride_bytes;
    uint2* out = STREAM ? a.nodes_out + (size_t)s * a.node_stride + a.node_first
                        : a.nodes_out + (size_t)s * (a.stride_bytes / 5u);
    uint32_t* end_out = STARTS ? a.node_end + (size_t)s * (a.node_stride - a.node_first)
                        : (!STREAM && a.node_end) ? a.node_end + (size_t)s * (a.stride_bytes / 5u) : nullptr;
    uint32_t held_in = 0;  // STREAM, thread 0: bytes of the unfinished record entering the push
    if constexpr (STREAM) {
      // all zero (a fresh stream): state 0, whose first record ends at byte 5 at the earliest, never reading the halo
      if (tid == 0) {
        const uint32_t* held = a.held + (size_t)s * kHeldWords;
        held_in = held[kHeldOk];
        sm.carry_state = held_in;
        sm.carry_nodes = 0;
        *reinterpret_cast<uint32_t*>(sm_bytes) = held[0];
      }
    } else {
      if (tid == 0) {
        sm.carry_state = 0;
        sm.carry_nodes = 0;
      }
      if (tid < 4) sm_bytes[tid] = 0;
    }
    __syncthreads();
    for (uint32_t t0 = 0; t0 < n; t0 += kNormTile) {
      const uint32_t live = min((uint32_t)kNormTile, n - t0);
      {  // stage the tile: 16-byte loads where the stream is aligned (tiles are multiples of 16 bytes long)
        uint32_t done = 0;
        if ((reinterpret_cast<uintptr_t>(src + t0) & 15u) == 0) {
          const uint4* g4 = reinterpret_cast<const uint4*>(src + t0);
          uint4* d128 = reinterpret_cast<uint4*>(sm_bytes + 4);
          const uint32_t quads = live >> 4;
          for (uint32_t q = tid; q < quads; q += NT) d128[q] = __ldg(g4 + q);
          done = quads << 4;
        }
        for (uint32_t i = done + tid; i < live; i += NT) sm_bytes[4 + i] = __ldg(src + t0 + i);
      }
      __syncthreads();
      // ---- fast path: the tile is entered between records and holds only whole, well-formed records.
      // Then the byte machine accepts every record where it lies (state 0 -> 1 -> 2 -> 3 -> 4 -> 0), so
      // record q is bytes [5q, 5q+5) and the nodes can be written without the scans below.
      {
        const uint32_t n_rec = live / 5u;
        int ok = (sm.carry_state == 0 && n_rec * 5u == live) ? 1 : 0;
        // one sweep: every record is read as two aligned words (5 bytes never span three), checked and turned into
        // its node in registers; the nodes are written once the whole block agrees that the tile is clean
        constexpr uint32_t kRecPerThread = (kNormTile / 5 + NT - 1) / NT;
        const uint32_t* W = reinterpret_cast<const uint32_t*>(sm_bytes + 4);  // 16-byte aligned
        uint2 nd[kRecPerThread];
#pragma unroll
        for (uint32_t j = 0; j < kRecPerThread; ++j) {
          const uint32_t q = tid + j * NT;
          nd[j] = make_uint2(0u, 0u);
          if (q < n_rec) {
            const uint32_t off = 5u * q, w = off >> 2, sh = (off & 3u) * 8u;
            const uint32_t w0 = W[w], w1 = W[w + 1];
            const uint32_t lo = __funnelshift_r(w0, w1, sh);  // bytes 0..3 of the record
            const uint32_t b4 = (w1 >> sh) & 0xFFu;           // byte 4
            const uint32_t sq = lo & 0xFFu, angle_chk = (lo >> 8) & 0xFFFFu, dist = (lo >> 24) | (b4 << 8);
            ok &= (int)(((sq >> 1) ^ sq) & angle_chk & 1u);
            nd[j].x = ((((angle_chk >> 1) << 8) / 90u) & 0xFFFFu) | (dist << 16);
            nd[j].y = (((sq >> 2) << 2) << 16) | ((sq & 1u) << 24);
          }
        }
        if (__syncthreads_and(ok)) {
          uint2* o = out + sm.carry_nodes;
#pragma unroll
          for (uint32_t j = 0; j < kRecPerThread; ++j) {
            const uint32_t q = tid + j * NT;
            if (q < n_rec) {
              o[q] = nd[j];
              if (end_out && (!STARTS || ((nd[j].y >> 24) & 1u))) end_out[sm.carry_nodes + q] = t0 + 5 * q + 4;
            }
          }
          __syncthreads();
          if (tid < 4) sm_bytes[tid] = sm_bytes[live + tid];
          if (tid == 0) sm.carry_nodes += n_rec;
          __syncthreads();
          continue;
        }
      }
      // fold this thread's bytes into one map
      const uint32_t b0 = tid * kChunk;
      uint32_t f = kIdentityMap;
      for (uint32_t i = 0; i < (uint32_t)kChunk; ++i) {
        if (b0 + i < live) f = compose_map(byte_map(sm_bytes[4 + b0 + i]), f);
      }
      uint32_t Fm = f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t p = __shfl_up_sync(0xffffffffu, Fm, o);
        if (lane >= (uint32_t)o) Fm = compose_map(Fm, p);
      }
      if (lane == 31) sm.warp_f[warp] = Fm;
      __syncthreads();
      uint32_t state = sm.carry_state;
      for (uint32_t w = 0; w < warp; ++w) state = (sm.warp_f[w] >> (3u * state)) & 7u;
      const uint32_t Fprev = __shfl_up_sync(0xffffffffu, Fm, 1);
      if (lane != 0) state = (Fprev >> (3u * state)) & 7u;
      // replay from the known entry state: which bytes complete a record?
      uint32_t ends = 0, cnt = 0, st = state;
      for (uint32_t i = 0; i < (uint32_t)kChunk; ++i) {
        if (b0 + i < live) {
          if (st == 4) {
            ends |= 1u << i;
            ++cnt;
          }
          st = (byte_map(sm_bytes[4 + b0 + i]) >> (3u * st)) & 7u;
        }
      }
      const uint32_t inc_scan = warp_inclusive_scan(cnt);
      if (lane == 31) sm.warp_c[warp] = inc_scan;
      __syncthreads();
      uint32_t off = inc_scan - cnt;
      for (uint32_t w = 0; w < warp; ++w) off += sm.warp_c[w];
      while (ends) {
        const uint32_t i = __ffs(ends) - 1;
        ends &= ends - 1;
        sm.ends[off++] = (uint16_t)(b0 + i);
      }
      if (tid == NT - 1) {
        uint32_t tot = 0, st2 = sm.carry_state;
        for (uint32_t w = 0; w < NT / 32; ++w) {
          tot += sm.warp_c[w];
          st2 = (sm.warp_f[w] >> (3u * st2)) & 7u;
        }
        sm.tile_nodes = tot;
        sm.red_state = st2;
      }
      __syncthreads();
      const uint32_t n_nodes = sm.tile_nodes;
      uint2* o = out + sm.carry_nodes;
      for (uint32_t q = tid; q < n_nodes; q += NT) {
        const uint8_t* r = sm_bytes + sm.ends[q];  // record = bytes[end-4 .. end], shifted by the 4-byte halo
        const uint32_t sq = r[0];
        const uint32_t angle_chk = ld16(r + 1), dist = ld16(r + 3);
        const uint32_t key = (((angle_chk >> 1) << 8) / 90u) & 0xFFFFu;
        uint2 nd;
        nd.x = key | (dist << 16);
        nd.y = (((sq >> 2) << 2) << 16) | ((sq & 1u) << 24);
        o[q] = nd;
        if (end_out && (!STARTS || ((nd.y >> 24) & 1u))) end_out[sm.carry_nodes + q] = t0 + sm.ends[q];
      }
      __syncthreads();
      if constexpr (STREAM) {
        // the next push reads the halo, and a last tile of live < 4 bytes shifts it onto itself: every read lands
        // before any write
        uint8_t last = 0;
        if (tid < 4) last = sm_bytes[live + tid];
        __syncwarp();
        if (tid < 4) sm_bytes[tid] = last;
      } else {
        if (tid < 4) sm_bytes[tid] = sm_bytes[live + tid];  // last four bytes of this tile (live >= 4 or stream ends)
      }
      if (tid == 0) {
        sm.carry_nodes += sm.tile_nodes;
        sm.carry_state = sm.red_state;
      }
      __syncthreads();
    }
    if (tid == 0) {
      if (a.node_counts) a.node_counts[s] = sm.carry_nodes;
      if constexpr (STREAM) {  // a stream without bytes writes back what it read
        uint32_t* held = a.held + (size_t)s * kHeldWords;
        held[kHeldOk] = sm.carry_state;
        held[0] = *reinterpret_cast<const uint32_t*>(sm_bytes);
        // every byte entering (held + pushed) is in a decoded record, held for the next push, or skipped
        StreamCounters& sc = a.counters[s];
        sc.bytes_in += n;
        sc.frames += sm.carry_nodes;
        sc.skipped_bytes += held_in + n - 5u * sm.carry_nodes - sm.carry_state;
      } else {
        if (a.fsm_state_out) a.fsm_state_out[s] = sm.carry_state;
      }
    }
    __syncthreads();
  }
}

template <bool STREAM>
__global__ void __launch_bounds__(NT, 5) decode_normal_kernel(NormalDecodeArgs a RPL_LIST_PARAM) {
  decode_normal_body<STREAM, false>(a RPL_LIST_ARG);
}

__global__ void __launch_bounds__(NT, 5) decode_normal_starts_kernel(NormalDecodeArgs a RPL_LIST_PARAM) {
  decode_normal_body<true, true>(a RPL_LIST_ARG);
}

// the decoders' tables, in this translation unit's device memory
cudaError_t upload_tables() {
  cudaError_t e;
  {  // handler_capsules.cpp:546-556, evaluated exactly as written there (double arithmetic, truncation)
    int table[493];
    for (int k2 = 0; k2 < 492; ++k2) {
      const int off_q16 = (int)(8 * 3.1415926535 * (1 << 16) / 180) - (k2 << 6) - (k2 * k2 * k2) / 98304;
      table[k2] = int(off_q16 * 180 / 3.14159265);
    }
    const int off_default = (int)(7.5 * 3.1415926535 * (1 << 16) / 180.0);
    table[492] = int(off_default * 180 / 3.14159265);
    e = cudaMemcpyToSymbol(g_ultra_offset, table, sizeof(table));
    if (e != cudaSuccess) return e;
  }
  {  // HQ: "advance the CRC register by N zero bytes" as 4 x 256 tables, N = 192 and 204 (decode_hq_kernel)
    static uint32_t t0[256];
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int j = 0; j < 8; ++j) c = (c & 1u) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
      t0[i] = c;
    }
    static uint32_t adv[2][4][256];
    const int nbytes[2] = {192, 204};
    for (int w = 0; w < 2; ++w)
      for (int k = 0; k < 4; ++k)
        for (uint32_t b = 0; b < 256; ++b) {
          uint32_t v = b << (8 * k);
          for (int i = 0; i < nbytes[w]; ++i) v = (v >> 8) ^ t0[v & 0xFFu];
          adv[w][k][b] = v;
        }
    e = cudaMemcpyToSymbol(g_hq_advance, adv, sizeof(adv));
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

#ifndef RPL_DECODE_LIST
template <int F>
cudaError_t launch_fmt(const CapsuleDecodeArgs& a, int grid, cudaStream_t stream) {
  if (a.node_stride)
    decode_capsule_kernel<F, true><<<grid, Fmt<F>::DT, sizeof(CapsuleSmem<F>), stream>>>(a);
  else
    decode_capsule_kernel<F, false><<<grid, Fmt<F>::DT, sizeof(CapsuleSmem<F>), stream>>>(a);
  return cudaGetLastError();
}

template <int F>
cudaError_t configure_fmt() {
  cudaError_t e = cudaFuncSetAttribute(decode_capsule_kernel<F, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)sizeof(CapsuleSmem<F>));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(decode_capsule_kernel<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)sizeof(CapsuleSmem<F>));
}

}  // namespace

cudaError_t launch_decode_capsules(uint32_t ans_type, const CapsuleDecodeArgs& a, int grid, cudaStream_t stream,
                                   const StreamList* list) {
  if (a.n_streams == 0) return cudaSuccess;
  if (list) return launch_decode_capsules_list(ans_type, a, *list, grid, stream);
  switch (ans_type) {
    case 0x82: return launch_fmt<kExpress>(a, grid, stream);
    case 0x84: return launch_fmt<kUltra>(a, grid, stream);
    case 0x85: return launch_fmt<kDense>(a, grid, stream);
    case 0x86: return launch_fmt<kUltraDense>(a, grid, stream);
    case 0x83:
      if (a.node_stride)
        decode_hq_kernel<true><<<grid, HT, sizeof(HqSmem), stream>>>(a);
      else
        decode_hq_kernel<false><<<grid, HT, sizeof(HqSmem), stream>>>(a);
      return cudaGetLastError();
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_decode_normal(const NormalDecodeArgs& a, int grid, cudaStream_t stream, const StreamList* list) {
  if (a.n_streams == 0) return cudaSuccess;
  if (list) return launch_decode_normal_list(a, *list, grid, stream);
  if (a.node_stride && a.node_end)
    decode_normal_starts_kernel<<<grid, NT, 0, stream>>>(a);
  else if (a.node_stride)
    decode_normal_kernel<true><<<grid, NT, 0, stream>>>(a);
  else
    decode_normal_kernel<false><<<grid, NT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t decode_formats_configure() {
  cudaError_t e;
  if ((e = upload_tables()) != cudaSuccess) return e;
  if ((e = configure_fmt<kExpress>()) != cudaSuccess || (e = configure_fmt<kUltra>()) != cudaSuccess ||
      (e = configure_fmt<kDense>()) != cudaSuccess || (e = configure_fmt<kUltraDense>()) != cudaSuccess)
    return e;
  e = cudaFuncSetAttribute(decode_hq_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HqSmem));
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(decode_hq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HqSmem));
  if (e != cudaSuccess) return e;
  return decode_list_configure();
}
#else
template <int F>
cudaError_t launch_fmt(const CapsuleDecodeArgs& a, const StreamList& l, int grid, cudaStream_t stream) {
  decode_capsule_kernel<F, true><<<grid, Fmt<F>::DT, sizeof(CapsuleSmem<F>), stream>>>(a, l);
  return cudaGetLastError();
}

template <int F>
cudaError_t configure_fmt() {
  return cudaFuncSetAttribute(decode_capsule_kernel<F, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)sizeof(CapsuleSmem<F>));
}

}  // namespace

cudaError_t launch_decode_capsules_list(uint32_t ans_type, const CapsuleDecodeArgs& a, const StreamList& l, int grid,
                                        cudaStream_t stream) {
  switch (ans_type) {
    case 0x82: return launch_fmt<kExpress>(a, l, grid, stream);
    case 0x84: return launch_fmt<kUltra>(a, l, grid, stream);
    case 0x85: return launch_fmt<kDense>(a, l, grid, stream);
    case 0x86: return launch_fmt<kUltraDense>(a, l, grid, stream);
    case 0x83:
      decode_hq_kernel<true><<<grid, HT, sizeof(HqSmem), stream>>>(a, l);
      return cudaGetLastError();
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_decode_normal_list(const NormalDecodeArgs& a, const StreamList& l, int grid, cudaStream_t stream) {
  if (a.node_end)
    decode_normal_starts_kernel<<<grid, NT, 0, stream>>>(a, l);
  else
    decode_normal_kernel<true><<<grid, NT, 0, stream>>>(a, l);
  return cudaGetLastError();
}

cudaError_t decode_list_configure() {
  cudaError_t e;
  if ((e = upload_tables()) != cudaSuccess) return e;
  if ((e = configure_fmt<kExpress>()) != cudaSuccess || (e = configure_fmt<kUltra>()) != cudaSuccess ||
      (e = configure_fmt<kDense>()) != cudaSuccess || (e = configure_fmt<kUltraDense>()) != cudaSuccess)
    return e;
  return cudaFuncSetAttribute(decode_hq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(HqSmem));
}
#endif

}  // namespace rpl
