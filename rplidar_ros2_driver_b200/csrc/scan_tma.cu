// scan_tma.cu -- fast scan kernel v2: TMA-staged scan tiles (producer warp + mbarrier ring).
//
// Same contract and the same two passes as scan_fast.cu (mark keys, fold to a rank table,
// place by rank; ascendScanData_ + publish_scan, reference
// src/sdk/src/sl_lidar_driver.cpp:128-184 and src/rplidar_node.cpp:581-677), restructured so
// that no consumer warp ever waits on a global load:
//
//   * a dedicated producer warp streams the scan tile through a shared-memory ring with
//     1-D bulk TMA copies (cp.async.bulk, 8 KB chunks, mbarrier full/empty handshake).
//     The chunk sequence is [scan s pass 1][scan s pass 2][scan s+1 pass 1]...: the producer
//     runs ahead across pass and scan boundaries, so HBM/L2 latency is hidden behind the ring
//     depth instead of behind resident warps.  Pass-1 copies carry an L2 evict_last hint, the
//     pass-2 copies (L2 hits) and all output stores evict_first.
//   * marking keeps v1's 64 KB byte map (plain byte stores, ~10 instructions per node).  A
//     first version of this kernel ORed key bits into the bitmap with warp-aggregated
//     shared-memory atomics instead; it executed ~100 instructions per node in that loop, so it
//     was dropped.
//
// Serves launches without the ascended node buffer (that variant needs two more shared
// tables and stays on scan_fast.cu).  Requires every scan base to be 16-byte aligned (nodes
// pointer 16 B aligned, even stride); the host falls back to scan_fast.cu otherwise.
//
// LaserScan Mode B at strides in (8192, 32768] -- the shared-memory kernels of scan_small.cu take
// the smaller ones -- runs on the sibling scan_tma_cluster_kernel below instead: a cluster of two
// CTAs holds the whole scan, so every node is read from global memory once.
#include <type_traits>

#include "rpl_device.cuh"
#include "scan_args.h"
#include "scan_common.cuh"

namespace rpl {

namespace {

#ifndef RPL_TMA_TC
#define RPL_TMA_TC 512
#endif
#ifndef RPL_TMA_CTAS
#define RPL_TMA_CTAS 2
#endif
constexpr int TC = RPL_TMA_TC;         // consumer threads (512 or 1024)
constexpr int kCtasPerSm = RPL_TMA_CTAS;
constexpr int kCWarps = TC / 32;
constexpr uint32_t kRowBytes = kKeySpace / TC;   // byte-map bytes folded by one thread
constexpr uint32_t kCols = kRowBytes / 16;       // 16-byte columns per row
constexpr uint32_t kWordsPerThread = kWords / TC;
static_assert(TC == 512 || TC == 1024, "fold layout is written for 512 or 1024 consumer threads");
constexpr int kBlock = TC + 32;        // + one producer warp
#ifndef RPL_TMA_CH
#define RPL_TMA_CH 1024
#endif
#ifndef RPL_TMA_STAGES
#define RPL_TMA_STAGES 16
#endif
#ifndef RPL_TMA_STAGES_SHARED
#define RPL_TMA_STAGES_SHARED 4
#endif
constexpr uint32_t CH = RPL_TMA_CH;          // nodes per chunk (8 bytes each)
constexpr int kRounds = CH / TC;       // nodes per consumer thread per chunk
// Ring depth (CH * stages * 8 bytes).  LaserScan Mode B streams fastest with a 128 KB ring and one CTA per SM:
// 0.865 ms per 4096 x 32768-node launch against 1.08 ms with 32 KB rings in two CTAs per SM (H100 SXM, 400 W
// power limit; 8 and 12 stages lie in between).  Mode A keeps the 32 KB ring and its second CTA per SM: with the
// 128 KB ring it lost 7 %.  The PointCloud2 payload keeps it too (not measured with a deeper ring).
template <int MODE>
constexpr int kStagesOf = MODE == 0 ? RPL_TMA_STAGES : RPL_TMA_STAGES_SHARED;

template <int kStages>
struct __align__(128) TmaSmem {
  uint8_t bytemap[kKeySpace];                // presence map (swizzled)
  uint2 ring[kStages][CH];
  uint2 rankV[kWords];                       // {bits, exclusive prefix} over measured keys
  unsigned long long full[kStages];
  unsigned long long empty[kStages];
  uint32_t red[4 * kCWarps];
  uint32_t valid_count;
  uint32_t totV;
  uint32_t fallback;
};

// byte-map swizzle: within the row a thread folds, the 16-byte column is XORed with row bits so
// that the 128-bit reads of 8 neighbouring threads hit 8 different bank groups
__device__ __forceinline__ uint32_t swz_x(uint32_t x) {
  if (TC == 512) return (x ^ ((x >> 3) & 0x70u)) & 0xFFFFu;  // 128-byte rows: column ^= row & 7
  return (x ^ ((x >> 3) & 0x30u)) & 0xFFFFu;                 // 64-byte rows: column ^= (row >> 1) & 3
}
__device__ __forceinline__ uint32_t gather4(uint32_t x) { return (x * 0x10204080u) >> 28; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// producer-side wait: the ring is usually full, so let the hardware park the thread (suspend
// time hint, ns) instead of spinning through issue slots the consumer warps need
__device__ __forceinline__ void mbar_wait_relaxed(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(20000u)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// 1-D bulk TMA copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, void* bar,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC) : "memory"); }

// which scans run through the ring (producer and consumers must agree)
__device__ __forceinline__ bool scan_is_streamed(uint32_t n, uint32_t stride, uint32_t max_nodes) {
  return n != 0 && n <= stride && n <= max_nodes && n <= kMaxFastNodes;
}

// fold: consumer thread t gathers the presence bytes of keys [kRowBytes t, kRowBytes (t+1)) into
// its kWordsPerThread bitmap words
__device__ __forceinline__ void fold_row(const uint8_t* bytemap, uint32_t tid, uint32_t (&wv)[kWordsPerThread]) {
#pragma unroll
  for (uint32_t j = 0; j < kWordsPerThread; ++j) wv[j] = 0;
  const uint4* bm = reinterpret_cast<const uint4*>(bytemap);
  const uint32_t colx = (TC == 512) ? (tid & 7u) : ((tid >> 1) & 3u);
#pragma unroll
  for (uint32_t c = 0; c < kCols; ++c) {
    const uint4 q = bm[tid * kCols + (c ^ colx)];  // physical column of logical chunk c
    const uint32_t x[4] = {q.x, q.y, q.z, q.w};
    uint32_t bv = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) bv |= gather4(x[j] & 0x01010101u) << (4 * j);
    wv[c >> 1] |= bv << (16 * (c & 1));
  }
}

// MODE: 0 = LaserScan Mode B, 1 = LaserScan Mode A, 2 = PointCloud2 (window + polar->xyz)
template <int MODE>
__global__ void __launch_bounds__(kBlock, kCtasPerSm) scan_tma_kernel(ScanBatchArgs a, FastWorkspace ws) {
  constexpr int kStages = kStagesOf<MODE>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TmaSmem<kStages>& sm = *reinterpret_cast<TmaSmem<kStages>*>(smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&sm.full[i], 1);         // the producer's arrive.expect_tx
      mbar_init(&sm.empty[i], kCWarps);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // =========================== producer warp ===========================================
  if (warp == kCWarps) {
    if (lane == 0) {
      const uint64_t pol_keep = l2_policy_evict_last();
      const uint64_t pol_stream = l2_policy_evict_first();
      uint32_t stage = 0, parity = 1;  // empty-barrier parity: first round passes at once
      for (uint32_t s = blockIdx.x; s < a.n_scans; s += gridDim.x) {
        const uint32_t n = a.counts[s];
        if (!scan_is_streamed(n, a.stride, ws.max_nodes)) continue;
        const uint2* base = a.nodes + (size_t)s * a.stride;
        const uint32_t nch = (n + CH - 1) / CH;
        for (int pass = 0; pass < 2; ++pass) {
          for (uint32_t c = 0; c < nch; ++c) {
            mbar_wait_relaxed(&sm.empty[stage], parity);
            // an odd tail is rounded up to a whole 16 bytes; the extra node lies inside the
            // scan's stride (even stride, n odd => n + 1 <= stride) and is masked by consumers
            const uint32_t cn = min(CH, n - c * CH);
            const uint32_t bytes = ((cn + 1u) & ~1u) * 8u;
            mbar_expect_tx(&sm.full[stage], bytes);
            tma_load_1d(&sm.ring[stage][0], base + (size_t)c * CH, bytes, &sm.full[stage],
                        pass == 0 ? pol_keep : pol_stream);
            if (++stage == kStages) {
              stage = 0;
              parity ^= 1u;
            }
          }
        }
      }
    }
    return;
  }

  // =========================== consumer warps ==========================================
  const bool new_proto = a.is_new_protocol != 0;
  const bool inverted = a.inverted != 0;
  const uint64_t pol_stream = l2_policy_evict_first();
  const uint32_t q_shift = new_proto ? 16u : 18u, q_mask = new_proto ? 0xFFu : 0x3Fu;
  constexpr bool MODE_A = (MODE == 1);
  constexpr bool CLOUD = (MODE == 2);
  const float w_rmin = a.range_min, w_rmax = a.range_max, w_imin = a.intensity_min;
  // intensity straight from word y without the conversion pipe (exact for values < 2^23)
  auto intensity_of = [&](uint32_t y) {
    return __fsub_rn(__uint_as_float(((y >> q_shift) & q_mask) | 0x4B000000u), 8388608.0f);
  };
  uint32_t stage = 0, parity = 0;  // ring position of the next chunk to consume
  using Checked = std::integral_constant<bool, true>;
  using Unchecked = std::integral_constant<bool, false>;
  auto advance = [&]() {
    if (++stage == kStages) {
      stage = 0;
      parity ^= 1u;
    }
  };

  // hand the current ring slot back to the producer.  Called after the memory operations
  // (byte-map / output stores) whose addresses depend on the values loaded from the slot, so
  // the arrive cannot issue before those loads have returned.
  auto release = [&]() {
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[stage]);
  };
  auto drain = [&](uint32_t nch) {  // consume chunks without looking at them
    for (uint32_t c = 0; c < nch; ++c) {
      mbar_wait(&sm.full[stage], parity);
      release();
      advance();
    }
  };

  for (uint32_t s = blockIdx.x; s < a.n_scans; s += gridDim.x) {
    const uint32_t n = a.counts[s];

    if (n > a.stride || n > ws.max_nodes) {  // caller error: report, touch nothing
      if (tid == 0) {
        if (a.status) a.status[s] = 0x80008000u;  // SL_RESULT_INVALID_DATA
        if (a.path) a.path[s] = 0u;
        if (a.beam_counts) a.beam_counts[s] = 0u;
        if (a.angle_inc) a.angle_inc[s] = 0.0f;
      }
      continue;
    }
    if (n > kMaxFastNodes) {  // cannot be tie-free: general kernel
      if (tid == 0) a.fallback_list[atomicAdd(a.fallback_count, 1u)] = s;
      continue;
    }
    if (n == 0) {  // ascendScanData: OPERATION_FAIL; publish_scan: nodes.empty() -> return
      if (tid == 0) {
        if (a.status) a.status[s] = a.apply_ascend ? kResultOperationFail : kResultOk;
        if (a.path) a.path[s] = 0u;
        if (a.beam_counts) a.beam_counts[s] = 0u;
        if (a.angle_inc) a.angle_inc[s] = 0.0f;
      }
      continue;
    }
    const uint32_t nch = (n + CH - 1) / CH;

    // ---- phase 0: clear the presence map ------------------------------------------------
    {
      uint4* bm = reinterpret_cast<uint4*>(sm.bytemap);
      const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
      for (uint32_t j = 0; j < kKeySpace / 16 / TC; ++j) bm[j * TC + tid] = z;
      if (tid == 0) {
        sm.fallback = 0;
      }
    }
    consumer_sync();

    // ---- phase 1 (mark): one byte store per measured key ---------------------------------
    uint32_t cnt = 0;
    uint8_t* const bmap = sm.bytemap;
    auto mark_chunk = [&](auto checked, uint32_t c) {
      mbar_wait(&sm.full[stage], parity);
      const uint2* slot = sm.ring[stage];
      uint2 v[kRounds];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) v[r] = slot[r * TC + tid];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        const uint32_t dist = __funnelshift_r(v[r].x, v[r].y, 16);
        bool valid = dist != 0;
        if (CLOUD) valid = valid && cloud_keep(dist_to_m(dist), intensity_of(v[r].y), w_rmin, w_rmax, w_imin);
        if (decltype(checked)::value && c * CH + r * TC + tid >= n) valid = false;
        if (valid) bmap[swz_x(v[r].x)] = 1;
        cnt += valid ? 1u : 0u;
      }
      release();
      advance();
    };
    const uint32_t nfull = n / CH;
    for (uint32_t c = 0; c < nfull; ++c) mark_chunk(Unchecked{}, c);
    if (nfull < nch) mark_chunk(Checked{}, nfull);
    cnt = warp_sum(cnt);
    if (lane == 0) sm.red[warp] = cnt;
    consumer_sync();

    // ---- fold: byte map -> bitmap + exclusive popcount prefix ------------------------------
    {
      // thread t owns keys [kRowBytes t, kRowBytes (t+1)) = kWordsPerThread bitmap words
      uint32_t wv[kWordsPerThread];
      fold_row(sm.bytemap, tid, wv);
      uint32_t sv = 0;
#pragma unroll
      for (uint32_t j = 0; j < kWordsPerThread; ++j) sv += __popc(wv[j]);
      const uint32_t iv = warp_inclusive_scan(sv);
      if (lane == 31) sm.red[2 * kCWarps + warp] = iv;
      consumer_sync();
      if (warp == 0) {
        uint32_t tv = lane < kCWarps ? sm.red[2 * kCWarps + lane] : 0u;
        uint32_t cc = lane < kCWarps ? sm.red[lane] : 0u;
        const uint32_t cv = warp_inclusive_scan(tv);
        cc = warp_sum(cc);
        if (lane < kCWarps) sm.red[2 * kCWarps + lane] = cv - tv;
        if (lane == 31) {
          sm.totV = cv;
          sm.valid_count = cc;
        }
      }
      consumer_sync();
      uint32_t pv = sm.red[2 * kCWarps + warp] + iv - sv;
#pragma unroll
      for (uint32_t j = 0; j < kWordsPerThread; ++j) {
        sm.rankV[tid * kWordsPerThread + j] = make_uint2(wv[j], pv);
        pv += __popc(wv[j]);
      }
    }
    consumer_sync();
    const uint32_t M = sm.valid_count;

    if (M == 0) {
      // ascendScanData: OPERATION_FAIL, buffer untouched; publish_scan: nothing to publish
      if (tid == 0) {
        if (a.status) a.status[s] = a.apply_ascend ? kResultOperationFail : kResultOk;
        if (a.path) a.path[s] = 0u;
        if (a.beam_counts) a.beam_counts[s] = 0u;
        if (a.angle_inc) a.angle_inc[s] = 0.0f;
      }
      drain(nch);
      consumer_sync();
      continue;
    }
    // duplicate keys (fewer distinct keys than measured nodes) -> general kernel (stable rule);
    // so do Mode A scans too large for the shared-memory index map
    if (sm.totV != M || (MODE_A && M > kModeASmemMaxPoints)) {
      if (tid == 0) a.fallback_list[atomicAdd(a.fallback_count, 1u)] = s;
      drain(nch);
      consumer_sync();
      continue;
    }

    // ---- phase 2 (place): rank and place --------------------------------------------------
    float* ranges = CLOUD ? nullptr : a.ranges + (size_t)s * a.stride;
    float* intens = CLOUD ? nullptr : a.intensities + (size_t)s * a.stride;
    float4* cloud = CLOUD ? a.xyzi + (size_t)s * a.stride : nullptr;
    uint16_t* sidx = reinterpret_cast<uint16_t*>(sm.bytemap);  // Mode A: u-rank -> node index (map is dead)
    const uint2* base = a.nodes + (size_t)s * a.stride;
    const float inc = angle_increment(M, MODE_A);
    const bool has0 = (sm.rankV[0].x & 1u) != 0;
    // Mode B output slot = ob + os * rank in wrapping u32 arithmetic (reference
    // rplidar_node.cpp:673); intensities[] sits at a fixed byte distance from ranges[]
    const uint32_t ob = inverted ? M - 1u : 0u, os = inverted ? 0xFFFFFFFFu : 1u;
    const ptrdiff_t i_minus_r = reinterpret_cast<char*>(intens) - reinterpret_cast<char*>(ranges);

    auto place_chunk = [&](auto checked, uint32_t c) {
      mbar_wait(&sm.full[stage], parity);
      const uint2* slot = sm.ring[stage];
      uint2 v[kRounds];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) v[r] = slot[r * TC + tid];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        const uint2 nd = v[r];
        const uint32_t k = nd.x & 0xFFFFu;
        const uint32_t dist = __funnelshift_r(nd.x, nd.y, 16);
        uint32_t measured = dist != 0 ? 1u : 0u;
        if (decltype(checked)::value && c * CH + r * TC + tid >= n) measured = 0;
        const uint32_t rk = rank_of(sm.rankV, k);
        const float dm = dist_to_m(dist);
        if (CLOUD) {  // polar -> xyz at the rank among kept points (oracle/cloud_oracle.cpp 1-3)
          const float it = intensity_of(nd.y);
          if (!cloud_keep(dm, it, w_rmin, w_rmax, w_imin)) measured = 0;
          const float2 cs = __ldg(a.trig + k);
          st_f32x4_if(cloud + rk, make_float4(__fmul_rn(dm, cs.x), __fmul_rn(dm, cs.y), 0.0f, it), pol_stream,
                      measured);
        } else if (!MODE_A) {  // Mode B: reference rplidar_node.cpp:661-677
          const uint32_t o = ob + os * rk;
          const float it = intensity_of(nd.y);
          float* pr = ranges + o;
          st_f32_if(pr, dm, pol_stream, measured);
          st_f32_if(reinterpret_cast<float*>(reinterpret_cast<char*>(pr) + i_minus_r), it, pol_stream, measured);
        } else if (measured) {  // Mode A: remember which node sits at this u-rank (mode_a_emit_smem)
          sidx[mode_a_urank(k, rk, M, inverted, has0)] = (uint16_t)(c * CH + r * TC + tid);
        }
      }
      release();
      advance();
    };
    for (uint32_t c = 0; c < nfull; ++c) place_chunk(Unchecked{}, c);
    if (nfull < nch) place_chunk(Checked{}, nfull);
    consumer_sync();

    // ---- phase 3 (Mode A): resolve bins that hold several points --------------------------
    if (MODE_A) {
      ModeAOut mo;
      mo.ranges = ranges;
      mo.intens = intens;
      mo.angle = a.angle;
      mo.M = M;
      mo.inc = inc;
      mo.inverted = inverted;
      mo.new_proto = new_proto;
      mo.policy = pol_stream;
      // the rank table is dead by now: each warp stages a batch of bins in its own slice of it
      static_assert(kEmit2Stage * 2 * kCWarps <= sizeof(sm.rankV), "bin staging must fit the rank table");
      mode_a_emit_smem(mo, sidx, base, warp, kCWarps,
                       reinterpret_cast<uint16_t*>(sm.rankV) + warp * ((kEmit2Stage + 7u) & ~7u));
    }
    consumer_sync();
    if (tid == 0) {
      if (sm.fallback) {
        a.fallback_list[atomicAdd(a.fallback_count, 1u)] = s;
      } else {
        if (a.status) a.status[s] = kResultOk;
        if (a.path) a.path[s] = 0u;
        if (a.beam_counts) a.beam_counts[s] = M;
        if (a.angle_inc) a.angle_inc[s] = inc;
      }
    }
    consumer_sync();
  }
}

// =========================== two-CTA cluster kernel (LaserScan Mode B) ===========================
// A scan of up to 32768 nodes does not fit one SM's shared memory next to its byte map, but it fits two.
// scan_tma_cluster_kernel stages the whole scan across a cluster of two CTAs and reads every node from
// global memory once: chunk c (CH nodes) goes to CTA c & 1, slot c >> 1, filled by one bulk copy with an
// evict_first hint.  Each CTA marks its own nodes in its own byte map and folds it to bit-words; the CTAs
// swap words and measured counts through distributed shared memory, both build the same rank table, and
// each places its own slots from shared memory.  The ring kernel's second pass over global memory (an L2
// re-read of 8 B per node, and the 34 MB of evict_last lines it keeps live) is gone.
//
// Exchange: CTA r writes its words and count into the PEER's inbox with st.async, whose bytes complete on
// the peer's inbox_full barrier; the peer arms that barrier for the scan with one arrive.expect_tx of
// kInboxBytes.  Its phase completes once the arrive and all the bytes are in, in either order.  The data
// is visible to every thread that waits on the phase.  No fence and no block barrier come before the
// signal: a first version stored plainly and signalled with a fence.acq_rel.cluster + remote arrive, and
// that fence alone made the kernel no faster than the ring kernel.  After reading its own inbox, a CTA
// arrives on the peer's peer_free barrier (release, cluster scope): the peer waits there before it writes
// this inbox for the next scan, so neither barrier can run more than one phase ahead of its waiter.  Both
// barriers complete one phase per streamed scan.
//
// Why this cannot deadlock: only the consumer threads touch the exchange barriers, and both CTAs walk
// the same scans in the same order and take the same branches (every decision -- invalid, empty, no
// measured node, duplicate key -- depends on counts[s] or on the exchanged totals, identical on both
// sides).  In scan s a CTA publishes after its own mark pass, which waits only on its own producer; the
// producer waits only on slots its own consumers release after the place pass of scan s - 1, which in
// turn needs the peer's publish of s - 1 and the peer's read of the inbox of s - 1 -- both done before the
// peer could start scan s.  The producer warp never takes part in a cluster barrier while the loop runs;
// the whole cluster, producer warps included, meets in barrier.cluster exactly twice: after the barrier
// init (no remote arrive may reach an uninitialised barrier) and before exit (no CTA may exit while the
// peer can still store to its inbox or arrive on its barriers).
constexpr int kClusterSlots = 16;
constexpr uint32_t kClusterMaxNodes = 2u * kClusterSlots * CH;  // 32768
static_assert(kClusterMaxNodes <= kMaxFastNodes, "every scan the cluster kernel serves must be streamable");

struct __align__(128) ClusterSmem {
  uint8_t bytemap[kKeySpace];                // presence map of this CTA's nodes (swizzled)
  uint2 tile[kClusterSlots][CH];             // this CTA's half of the scan: chunk 2 j + rank in slot j
  uint2 rankV[kWords];                       // {bits, exclusive prefix} over the whole scan's measured keys
  uint4 inbox[kWords / 4];                   // the peer's bit-words of the current scan (written remotely)
  unsigned long long full[kClusterSlots];
  unsigned long long empty[kClusterSlots];
  unsigned long long inbox_full;             // the peer wrote inbox and inbox_count
  unsigned long long peer_free;              // the peer read the words this CTA wrote into its inbox
  uint32_t red[4 * kCWarps];
  uint32_t inbox_count;                      // the peer's measured-node count (written remotely)
  uint32_t valid_count;
  uint32_t totV;
};
static_assert(sizeof(ClusterSmem) <= 232448, "one CTA per SM: at most 227 KB of dynamic shared memory");
constexpr uint32_t kInboxBytes = sizeof(ClusterSmem::inbox) + sizeof(uint32_t);  // words + count per scan

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// all threads of both CTAs (exited threads would never arrive: call it with the whole block)
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// shared::cluster address of `p`'s counterpart in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t peer_addr(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
// asynchronous store into a peer CTA's shared memory that counts its bytes on the peer's mbarrier `bar`:
// once the barrier's phase completes, the data is visible to the threads that waited on it
__device__ __forceinline__ void st_async_v4(uint32_t addr, uint4 v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(addr),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void st_async_u32(uint32_t addr, uint32_t v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(addr), "r"(v),
               "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(addr) : "memory");
}
// wait for a phase completed by the peer's remote arrive: acquire at cluster scope, so that the peer's
// shared-memory accesses before its arrive are visible (or complete) here
__device__ __forceinline__ void mbar_wait_cluster(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// serves Mode B without the ascended buffer for strides in (kSmallMaxNodes, kClusterMaxNodes], 16-byte
// aligned scan bases; launched with cluster dims (2, 1, 1) and an even grid
__global__ void __launch_bounds__(kBlock, 1) scan_tma_cluster_kernel(ScanBatchArgs a, FastWorkspace ws) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  ClusterSmem& sm = *reinterpret_cast<ClusterSmem*>(smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
  const uint32_t s0 = blockIdx.x >> 1, s_step = gridDim.x >> 1;

  if (tid == 0) {
    for (int i = 0; i < kClusterSlots; ++i) {
      mbar_init(&sm.full[i], 1);         // the producer's arrive.expect_tx
      mbar_init(&sm.empty[i], kCWarps);  // one arrive per consumer warp (after the place pass)
    }
    mbar_init(&sm.inbox_full, 1);        // this CTA's arrive.expect_tx per scan + the peer's st.async bytes
    mbar_init(&sm.peer_free, 1);         // one remote arrive by the peer per scan
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  cluster_sync_all();

  if (warp == kCWarps) {
    // =========================== producer warp =========================================
    if (lane == 0) {
      const uint64_t pol_stream = l2_policy_evict_first();
      uint32_t eph = 0xFFFFFFFFu;  // empty-barrier parity per slot: the first fill passes at once
      for (uint32_t s = s0; s < a.n_scans; s += s_step) {
        const uint32_t n = a.counts[s];
        if (!scan_is_streamed(n, a.stride, ws.max_nodes)) continue;
        const uint2* base = a.nodes + (size_t)s * a.stride;
        const uint32_t nch = (n + CH - 1) / CH;
        const uint32_t mine = (nch + 1u - rank) >> 1;  // chunks c < nch with c & 1 == rank
        for (uint32_t j = 0; j < mine; ++j) {
          mbar_wait_relaxed(&sm.empty[j], (eph >> j) & 1u);
          eph ^= 1u << j;
          const uint32_t c = 2u * j + rank;
          // an odd tail is rounded up to a whole 16 bytes as in scan_tma_kernel (masked by consumers)
          const uint32_t cn = min(CH, n - c * CH);
          const uint32_t bytes = ((cn + 1u) & ~1u) * 8u;
          mbar_expect_tx(&sm.full[j], bytes);
          tma_load_1d(&sm.tile[j][0], base + (size_t)c * CH, bytes, &sm.full[j], pol_stream);
        }
      }
    }
    __syncwarp();
  } else {
    // =========================== consumer warps ========================================
    const bool new_proto = a.is_new_protocol != 0;
    const bool inverted = a.inverted != 0;
    const uint64_t pol_stream = l2_policy_evict_first();
    const uint32_t q_shift = new_proto ? 16u : 18u, q_mask = new_proto ? 0xFFu : 0x3Fu;
    auto intensity_of = [&](uint32_t y) {
      return __fsub_rn(__uint_as_float(((y >> q_shift) & q_mask) | 0x4B000000u), 8388608.0f);
    };
    const bool writer = rank == 0 && tid == 0;  // per-scan outputs come from cluster rank 0
    const uint32_t peer_inbox = peer_addr(sm.inbox, peer);
    const uint32_t peer_count = peer_addr(&sm.inbox_count, peer);
    const uint32_t peer_inbox_full = peer_addr(&sm.inbox_full, peer);
    const uint32_t peer_peer_free = peer_addr(&sm.peer_free, peer);
    uint32_t fph = 0;                         // full-barrier parity per slot
    uint32_t in_par = 0, free_par = 1;        // exchange barriers: peer_free's first wait passes at once
    using Checked = std::integral_constant<bool, true>;
    using Unchecked = std::integral_constant<bool, false>;
    auto release = [&](uint32_t j) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[j]);
    };

    for (uint32_t s = s0; s < a.n_scans; s += s_step) {
      const uint32_t n = a.counts[s];
      if (n > a.stride || n > ws.max_nodes) {  // caller error: report, touch nothing
        if (writer) {
          if (a.status) a.status[s] = 0x80008000u;  // SL_RESULT_INVALID_DATA
          if (a.path) a.path[s] = 0u;
          if (a.beam_counts) a.beam_counts[s] = 0u;
          if (a.angle_inc) a.angle_inc[s] = 0.0f;
        }
        continue;
      }
      if (n == 0) {  // ascendScanData: OPERATION_FAIL; publish_scan: nodes.empty() -> return
        if (writer) {
          if (a.status) a.status[s] = a.apply_ascend ? kResultOperationFail : kResultOk;
          if (a.path) a.path[s] = 0u;
          if (a.beam_counts) a.beam_counts[s] = 0u;
          if (a.angle_inc) a.angle_inc[s] = 0.0f;
        }
        continue;
      }
      const uint32_t nch = (n + CH - 1) / CH, nfull = n / CH;
      const uint32_t mine = (nch + 1u - rank) >> 1;

      // ---- clear the presence map (while this scan's copies are still in flight) --------------
      {
        uint4* bm = reinterpret_cast<uint4*>(sm.bytemap);
        const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (uint32_t j = 0; j < kKeySpace / 16 / TC; ++j) bm[j * TC + tid] = z;
      }
      consumer_sync();

      // ---- mark this CTA's chunks (they stay in their slots for the place pass) ------------
      uint32_t cnt = 0;
      uint8_t* const bmap = sm.bytemap;
      auto mark_chunk = [&](auto checked, uint32_t j) {
        mbar_wait(&sm.full[j], (fph >> j) & 1u);
        fph ^= 1u << j;
        const uint32_t c = 2u * j + rank;
        const uint2* slot = sm.tile[j];
        uint2 v[kRounds];
#pragma unroll
        for (int r = 0; r < kRounds; ++r) v[r] = slot[r * TC + tid];
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          const uint32_t dist = __funnelshift_r(v[r].x, v[r].y, 16);
          bool valid = dist != 0;
          if (decltype(checked)::value && c * CH + r * TC + tid >= n) valid = false;
          if (valid) bmap[swz_x(v[r].x)] = 1;
          cnt += valid ? 1u : 0u;
        }
      };
      // the partial chunk (c == nfull < nch) is the last of this CTA's chunks if it is this CTA's at all
      const bool tail = nfull < nch && (nfull & 1u) == rank;
      const uint32_t mine_full = tail ? mine - 1u : mine;
      for (uint32_t j = 0; j < mine_full; ++j) mark_chunk(Unchecked{}, j);
      if (tail) mark_chunk(Checked{}, mine_full);
      cnt = warp_sum(cnt);
      if (lane == 0) sm.red[warp] = cnt;
      consumer_sync();

      // ---- fold, exchange with the peer, rank table -----------------------------------------
      {
        uint32_t wv[kWordsPerThread];
        static_assert(kWordsPerThread == 4, "the exchange moves one uint4 of bit-words per thread");
        fold_row(sm.bytemap, tid, wv);
        if (tid == 0) mbar_expect_tx(&sm.inbox_full, kInboxBytes);  // this scan's phase: the peer's words + count
        mbar_wait_cluster(&sm.peer_free, free_par);  // the peer has read what this CTA sent for the last scan
        free_par ^= 1u;
        st_async_v4(peer_inbox + tid * 16u, make_uint4(wv[0], wv[1], wv[2], wv[3]), peer_inbox_full);
        if (warp == 0) {
          const uint32_t own = warp_sum(lane < kCWarps ? sm.red[lane] : 0u);
          if (lane == 0) st_async_u32(peer_count, own, peer_inbox_full);
        }
        mbar_wait_cluster(&sm.inbox_full, in_par);
        in_par ^= 1u;
        const uint4 pw = sm.inbox[tid];
        const uint32_t other = sm.inbox_count;
        wv[0] |= pw.x;
        wv[1] |= pw.y;
        wv[2] |= pw.z;
        wv[3] |= pw.w;
        uint32_t sv = 0;
#pragma unroll
        for (uint32_t j = 0; j < kWordsPerThread; ++j) sv += __popc(wv[j]);
        const uint32_t iv = warp_inclusive_scan(sv);
        if (lane == 31) sm.red[2 * kCWarps + warp] = iv;
        consumer_sync();  // every thread has read its inbox entry: the peer may overwrite it
        if (tid == 0) mbar_arrive_remote(peer_peer_free);
        if (warp == 0) {
          uint32_t tv = lane < kCWarps ? sm.red[2 * kCWarps + lane] : 0u;
          uint32_t cc = lane < kCWarps ? sm.red[lane] : 0u;
          const uint32_t cv = warp_inclusive_scan(tv);
          cc = warp_sum(cc);
          if (lane < kCWarps) sm.red[2 * kCWarps + lane] = cv - tv;
          if (lane == 31) {
            sm.totV = cv;
            sm.valid_count = cc + other;
          }
        }
        consumer_sync();
        uint32_t pv = sm.red[2 * kCWarps + warp] + iv - sv;
#pragma unroll
        for (uint32_t j = 0; j < kWordsPerThread; ++j) {
          sm.rankV[tid * kWordsPerThread + j] = make_uint2(wv[j], pv);
          pv += __popc(wv[j]);
        }
      }
      consumer_sync();
      const uint32_t M = sm.valid_count;  // measured nodes of the whole scan, the same in both CTAs

      if (M == 0 || sm.totV != M) {
        if (writer) {
          if (M == 0) {  // ascendScanData: OPERATION_FAIL, buffer untouched; publish_scan: nothing to publish
            if (a.status) a.status[s] = a.apply_ascend ? kResultOperationFail : kResultOk;
            if (a.path) a.path[s] = 0u;
            if (a.beam_counts) a.beam_counts[s] = 0u;
            if (a.angle_inc) a.angle_inc[s] = 0.0f;
          } else {  // duplicate keys, within a half or across the halves -> general kernel (stable rule)
            a.fallback_list[atomicAdd(a.fallback_count, 1u)] = s;
          }
        }
        for (uint32_t j = 0; j < mine; ++j) release(j);
        continue;
      }

      // ---- place this CTA's chunks by rank, then hand the slots back ----------------------
      float* ranges = a.ranges + (size_t)s * a.stride;
      float* intens = a.intensities + (size_t)s * a.stride;
      // Mode B output slot = ob + os * rank in wrapping u32 arithmetic (reference
      // rplidar_node.cpp:673); intensities[] sits at a fixed byte distance from ranges[]
      const uint32_t ob = inverted ? M - 1u : 0u, os = inverted ? 0xFFFFFFFFu : 1u;
      const ptrdiff_t i_minus_r = reinterpret_cast<char*>(intens) - reinterpret_cast<char*>(ranges);
      auto place_chunk = [&](auto checked, uint32_t j) {
        const uint32_t c = 2u * j + rank;
        const uint2* slot = sm.tile[j];
        uint2 v[kRounds];
#pragma unroll
        for (int r = 0; r < kRounds; ++r) v[r] = slot[r * TC + tid];
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          const uint2 nd = v[r];
          const uint32_t k = nd.x & 0xFFFFu;
          const uint32_t dist = __funnelshift_r(nd.x, nd.y, 16);
          uint32_t measured = dist != 0 ? 1u : 0u;
          if (decltype(checked)::value && c * CH + r * TC + tid >= n) measured = 0;
          const uint32_t rk = rank_of(sm.rankV, k);
          const uint32_t o = ob + os * rk;
          float* pr = ranges + o;
          st_f32_if(pr, dist_to_m(dist), pol_stream, measured);
          st_f32_if(reinterpret_cast<float*>(reinterpret_cast<char*>(pr) + i_minus_r), intensity_of(nd.y), pol_stream,
                    measured);
        }
        release(j);
      };
      for (uint32_t j = 0; j < mine_full; ++j) place_chunk(Unchecked{}, j);
      if (tail) place_chunk(Checked{}, mine_full);
      if (writer) {
        if (a.status) a.status[s] = kResultOk;
        if (a.path) a.path[s] = 0u;
        if (a.beam_counts) a.beam_counts[s] = M;
        if (a.angle_inc) a.angle_inc[s] = angle_increment(M, false);
      }
    }
  }
  cluster_sync_all();
}

}  // namespace

template <int MODE>
constexpr size_t kSmemOf = sizeof(TmaSmem<kStagesOf<MODE>>);

cudaError_t launch_scan_tma(const ScanBatchArgs& a, const FastWorkspace& ws, int grid, cudaStream_t stream) {
  if (a.xyzi) scan_tma_kernel<2><<<grid, kBlock, kSmemOf<2>, stream>>>(a, ws);
  else if (a.mode_a) scan_tma_kernel<1><<<grid, kBlock, kSmemOf<1>, stream>>>(a, ws);
  else scan_tma_kernel<0><<<grid, kBlock, kSmemOf<0>, stream>>>(a, ws);
  return cudaGetLastError();
}

bool scan_tma_cluster_applies(uint32_t stride) { return stride > kSmallMaxNodes && stride <= kClusterMaxNodes; }

namespace {
// launch configuration of scan_tma_cluster_kernel: clusters of two CTAs along x
struct ClusterLaunch {
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t cfg{};
  ClusterLaunch(int grid, cudaStream_t stream) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kBlock);
    cfg.dynamicSmemBytes = sizeof(ClusterSmem);
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
};
}  // namespace

cudaError_t launch_scan_tma_cluster(const ScanBatchArgs& a, const FastWorkspace& ws, int grid, cudaStream_t stream) {
  if (grid <= 0 || (grid & 1) != 0) return cudaErrorInvalidValue;
  ClusterLaunch l(grid, stream);
  return cudaLaunchKernelEx(&l.cfg, scan_tma_cluster_kernel, a, ws);
}

int scan_tma_max_clusters() {
  ClusterLaunch l(2, nullptr);
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, scan_tma_cluster_kernel, &l.cfg) != cudaSuccess) return 0;
  return n;
}

cudaError_t scan_tma_configure() {
  cudaError_t e = cudaFuncSetAttribute(scan_tma_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOf<0>);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(scan_tma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOf<1>);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(scan_tma_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)sizeof(ClusterSmem));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(scan_tma_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOf<2>);
}

int scan_tma_max_ctas_per_sm(int mode) {
  int nb = 0;
  if (mode == 0) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, scan_tma_kernel<0>, kBlock, kSmemOf<0>);
  else if (mode == 1) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, scan_tma_kernel<1>, kBlock, kSmemOf<1>);
  else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, scan_tma_kernel<2>, kBlock, kSmemOf<2>);
  return nb;
}

}  // namespace rpl
