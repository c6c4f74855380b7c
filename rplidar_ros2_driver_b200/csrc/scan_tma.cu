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
//   * marking keeps scan_fast.cu's 64 KB byte map (plain byte stores, ~10 instructions per
//     node; the map, its fold and the rank table are in scan_common.cuh).  A first version of
//     this kernel ORed key bits into the bitmap with warp-aggregated shared-memory atomics
//     instead; it executed ~100 instructions per node in that loop, so it was dropped.
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
#include "sm90_async.cuh"

namespace rpl {

namespace {

constexpr int TC = kMapThreads;        // consumer threads
constexpr int kCWarps = TC / 32;
constexpr int kBlock = TC + 32;        // + one producer warp
constexpr uint32_t CH = 1024;          // nodes per chunk (8 KB)
constexpr int kRounds = CH / TC;       // nodes per consumer thread per chunk
// Ring depth (CH * stages * 8 bytes).  LaserScan Mode B streams fastest with a 128 KB ring and one CTA per SM:
// 0.865 ms per 4096 x 32768-node launch against 1.08 ms with 32 KB rings in two CTAs per SM (H100 SXM, 400 W
// power limit; 8 and 12 stages lie in between).  Mode A keeps the 32 KB ring and its second CTA per SM: with the
// 128 KB ring it lost 7 %.  The PointCloud2 payload keeps it too (not measured with a deeper ring).
template <int MODE>
constexpr int kStagesOf = MODE == 0 ? 16 : 4;

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
};

// which scans run through the ring (producer and consumers must agree)
__device__ __forceinline__ bool scan_is_streamed(uint32_t n, uint32_t stride, uint32_t max_nodes) {
  return n != 0 && n <= stride && n <= max_nodes && n <= kMaxFastNodes;
}

// ---- Mode A emit, shared-memory variant -------------------------------------------------------
// ncu on scan_fast.cu's mode_a_emit showed its global scratch doubling DRAM traffic (8 B written + 8 B read per
// point through a 76 MB working set).  Here the place pass only records WHICH node sits at each
// u-rank, as a u16 node index in the 64 KB the dead presence map leaves free (so M <= 32768),
// and the emit pass gathers the nodes from the tile again (L2 hits, coalesced for a sorted
// revolution).  Bins of a batch are staged per warp in the (equally dead) rank table.
constexpr uint32_t kEmit2Batch = 256;
constexpr uint32_t kEmit2Stage = kEmit2Batch + 33;  // staged bins: one entry before, 32 after
constexpr uint32_t kModeASmemMaxPoints = kKeySpace / 2;

__device__ __forceinline__ void mode_a_emit_smem(const ModeAOut& o, const uint16_t* sidx, const uint2* tile,
                                                 uint32_t warp, uint32_t nwarps, uint16_t* sb) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t M = o.M;
  const uint32_t len = ((M + nwarps - 1u) / nwarps + kEmit2Batch - 1u) & ~(kEmit2Batch - 1u);
  const uint32_t r_begin = min(M, warp * len), r_end = min(M, r_begin + len);
  if (r_begin >= r_end) return;
  const bool inverted = o.inverted;
  const float inc = o.inc;
  // integer quotient where the float chain provably agrees, else the exact chain in registers
  // (FP64, no memory access): this pass is bound by load latency, not by issue slots, so the
  // table lookup of mode_a_emit would only add a dependent L2 access per entry
  auto bin_of_key = [&](uint32_t key) { return (uint32_t)mode_a_bin_fast(key, M, inc, inverted); };
  const uint32_t kNoBin = 0xFFFFu, kBeforeFirst = 0xFFFEu;  // real bins are < 32768
  const float kInf = __int_as_float(0x7f800000);
  auto entry_of = [&](uint2 nd) {
    return mode_a_entry(dist_to_m(__funnelshift_r(nd.x, nd.y, 16)), nd.x & 0xFFFFu, (nd.y >> 16) & 0xFFu);
  };
  constexpr int kW = kEmit2Batch / 32;
  using Checked = std::integral_constant<bool, true>;
  using Unchecked = std::integral_constant<bool, false>;

  auto batch = [&](auto checked, uint32_t base) {
    constexpr bool CK = decltype(checked)::value;
    __syncwarp();
    // stage: this lane's own eight entries (kept in registers) plus one halo entry (the entry
    // before the batch for lane 0, the 32 after it for the others); all gathers issued together
    uint2 nd[kW];
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      const uint32_t r = base + w * 32 + lane;
      nd[w] = (!CK || r < M) ? tile[sidx[r]] : make_uint2(0, 0);
    }
    const uint32_t th = (lane == 0) ? 0u : (kEmit2Batch + lane);  // lane 0 -> before; 1..31 -> after
    const long long rh = (long long)base - 1 + th;
    const bool halo_ok = !CK || (rh >= 0 && rh < (long long)M);
    const uint2 ndh = halo_ok ? tile[sidx[halo_ok ? rh : 0]] : make_uint2(0, 0);
    const uint32_t r2 = base - 1 + kEmit2Batch + 32;  // last look-ahead slot (lane 31)
    const bool last_ok = (lane == 31) && (!CK || r2 < M);
    const uint2 nd2 = last_ok ? tile[sidx[last_ok ? r2 : 0]] : make_uint2(0, 0);
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      const uint32_t r = base + w * 32 + lane;
      sb[1 + w * 32 + lane] = (!CK || r < M) ? (uint16_t)bin_of_key(nd[w].x & 0xFFFFu) : (uint16_t)kNoBin;
    }
    {
      uint32_t b = (CK && rh < 0) ? kBeforeFirst : kNoBin;
      if (halo_ok) b = bin_of_key(ndh.x & 0xFFFFu);
      sb[th] = (uint16_t)b;
      if (lane == 31) sb[kEmit2Batch + 32] = last_ok ? (uint16_t)bin_of_key(nd2.x & 0xFFFFu) : (uint16_t)kNoBin;
    }
    __syncwarp();
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      const uint32_t i = 1 + w * 32 + lane;
      const uint32_t r = base + w * 32 + lane;
      const bool live = !CK || r < M;
      const uint32_t b = sb[i], bprev = sb[i - 1];
      const bool head = live && (b != bprev);
      unsigned long long v = entry_of(nd[w]);
      // the next entry's node sits in the neighbouring lane (or lane 0 of the next window):
      // a bin shared by two points -- the usual collision -- costs two shuffles, no memory access
      uint2 nxt;
      nxt.x = __shfl_down_sync(0xffffffffu, nd[w].x, 1);
      nxt.y = __shfl_down_sync(0xffffffffu, nd[w].y, 1);
      if (w + 1 < kW) {
        const uint32_t fx = __shfl_sync(0xffffffffu, nd[(w + 1) % kW].x, 0);
        const uint32_t fy = __shfl_sync(0xffffffffu, nd[(w + 1) % kW].y, 0);
        if (lane == 31) nxt = make_uint2(fx, fy);
      }
      if (head && sb[i + 1] == b) {
        if (w + 1 == kW && lane == 31) nxt = tile[sidx[r + 1]];  // first entry of the next batch
        v = min(v, entry_of(nxt));
        if (sb[i + 2] == b) {  // three or more points in the bin: walk on (rare: M points, M bins)
          for (uint32_t rr = r + 2; rr < M; ++rr) {
            const uint2 other = tile[sidx[rr]];
            if (bin_of_key(other.x & 0xFFFFu) != b) break;
            v = min(v, entry_of(other));
          }
        }
      }
      mode_a_store_bin(o, head ? (int)b : 0, v, head ? 1u : 0u);
      const int gap_from = (CK && bprev == kBeforeFirst) ? 0 : (int)bprev + 1;
      if (head && (int)b > gap_from) {  // empty bins in front of this run
        if ((int)b - gap_from == 1) {
          o.ranges[gap_from] = kInf;
          o.intens[gap_from] = 0.0f;
        } else {
          mode_a_fill_empty(o, gap_from, (int)b);
        }
      }
      if (CK && live && r == M - 1u) mode_a_fill_empty(o, (int)b + 1, (int)M);  // empty bins behind the last run
    }
  };
  for (uint32_t base = r_begin; base < r_end; base += kEmit2Batch) {
    // interior batches (entry before and all 256 + 32 look-ahead entries exist) skip every range check
    if (base >= 1u && base + kEmit2Batch + 32u <= M) batch(Unchecked{}, base);
    else batch(Checked{}, base);
  }
}

// MODE: 0 = LaserScan Mode B, 1 = LaserScan Mode A, 2 = PointCloud2 (window + polar->xyz)
template <int MODE>
__global__ void __launch_bounds__(kBlock, 2) scan_tma_kernel(ScanBatchArgs a, uint32_t max_nodes) {
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
        if (!scan_is_streamed(n, a.stride, max_nodes)) continue;
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
  const IntensityOf intensity_of(new_proto);
  constexpr bool MODE_A = (MODE == 1);
  constexpr bool CLOUD = (MODE == 2);
  const float w_rmin = a.range_min, w_rmax = a.range_max, w_imin = a.intensity_min;
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

    if (n > a.stride || n > max_nodes) {  // caller error: report, touch nothing
      if (tid == 0) write_outcome(a, s, kResultInvalidData, 0u, 0.0f);
      continue;
    }
    if (n > kMaxFastNodes) {  // cannot be tie-free: general kernel
      if (tid == 0) hand_to_general(a, s);
      continue;
    }
    if (n == 0) {  // ascendScanData: OPERATION_FAIL; publish_scan: nodes.empty() -> return
      if (tid == 0) write_outcome_empty(a, s);
      continue;
    }
    const uint32_t nch = (n + CH - 1) / CH;

    // ---- phase 0: clear the presence map ------------------------------------------------
    bytemap_clear(sm.bytemap, tid);
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
      uint32_t wv[kWordsPerThread];
      fold_row(sm.bytemap, tid, wv);
      rank_table(sm, wv, tid, 0u);
    }
    consumer_sync();
    const uint32_t M = sm.valid_count;

    if (M == 0) {
      if (tid == 0) write_outcome_empty(a, s);
      drain(nch);
      consumer_sync();
      continue;
    }
    // duplicate keys (fewer distinct keys than measured nodes) -> general kernel (stable rule);
    // so do Mode A scans too large for the shared-memory index map
    if (sm.totV != M || (MODE_A && M > kModeASmemMaxPoints)) {
      if (tid == 0) hand_to_general(a, s);
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
    const ModeBOut mode_b(ranges, intens, M, inverted);

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
        } else if (!MODE_A) {
          mode_b.store(rk, dm, intensity_of(nd.y), measured);
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
    if (tid == 0) write_outcome(a, s, kResultOk, M, inc);
    consumer_sync();
  }
}

// =========================== two-CTA cluster kernel (LaserScan Mode B) ===========================
// A scan of up to 32768 nodes does not fit one SM's shared memory next to its byte map, but it fits two.
// scan_tma_cluster_kernel stages the whole scan across a cluster of two CTAs and reads every node from
// global memory once: chunk c (CH nodes) goes to CTA c & 1, slot c >> 1, filled by one bulk copy.  Each
// CTA marks its own nodes in its own byte map and folds it to bit-words; the CTAs swap words and measured
// counts through distributed shared memory, both build the same rank table, and each places its own
// chunks.  The ring kernel's second pass over global memory (an L2 re-read of 8 B per node, and the 34 MB
// of evict_last lines it keeps live) is gone.
//
// L2 policy: the bulk copies and the output stores are marked evict_normal.  With nothing read twice there
// is nothing to protect, and on the H100 evict_normal on both took about 1 % off the launch, while
// evict_first on both (as in the ring kernel) or evict_normal on the stores alone were slower (DESIGN.md §5.1).
//
// Held slots: shared memory is full (216.6 KB), but the register file is not.  Each consumer thread keeps
// its kRounds nodes of the chunks in slots j < kHeld in registers (4 registers per chunk) and hands those
// slots back to its producer as soon as they are marked, so the producer loads the next scan's first
// chunks while this scan folds, exchanges and builds its rank table -- a stretch in which the SM would
// otherwise have no load in flight.  The other slots are handed back in the place pass, which takes them
// first, in ascending order, and then places the held chunks from registers.  Each filled slot still gets
// exactly one arrive per consumer warp per scan: held slots when they are marked, the others in the place
// pass, which hands them back without placing them for a scan handed on or with nothing measured.
//
// Pipeline: the consumer warps mark the cluster's next streamed scan s2 while they place scan s, so that the
// stretch with no stores in flight is only the fold, the exchange and the rank table.  After each of s's slots
// j >= kHeld is placed and handed back, a warp marks one chunk of s2: first its held chunks (slots the producer
// refilled during s's fold and exchange), then its slot j - kMarkLag, whose refill was asked for kMarkLag places
// ago.  Then s's held chunks are placed from registers and the rest of s2 is marked.  The byte map is free by then:
// s's fold has turned it into bit-words, and it is cleared for s2 right after that fold, behind rank_table's
// barriers and before the barrier that precedes the first mark of s2.  s2's measured count stays in a register
// until its fold, as sm.red holds s's counts until rank_table has read them.  Both sets of held chunks are live
// during the first places (96 registers per thread, no spills).
//
// Exchange: CTA r writes its words and count into the PEER's inbox with st.async, whose bytes complete on
// the peer's inbox_full barrier; the peer arms that barrier for the scan with one arrive.expect_tx of
// kInboxBytes.  Its phase completes once the arrive and all the bytes are in, in either order.  The data
// is visible to every thread that waits on the phase.  No fence and no block barrier come before the
// signal: a first version stored plainly and signalled with a fence.acq_rel.cluster + remote arrive, and
// that fence alone made the kernel no faster than the ring kernel.  Once every consumer thread has used what
// it read from its own inbox -- the words and count are folded into the rank table behind rank_table's
// barriers -- thread 0 arrives on the peer's peer_free barrier: the peer waits there before it writes this
// inbox for the next scan, so neither barrier can run more than one phase ahead of its waiter.  That arrive
// is a release at CTA scope (mbar_arrive_remote): the reads it hands back have returned their values
// before it issues, and the cluster-scope form put a MEMBAR.ALL.GPU in front of it that held every consumer
// warp for about 2 us per scan.  Both barriers complete one phase per streamed scan.
//
// Why this cannot deadlock: only the consumer threads touch the exchange barriers, and both CTAs walk
// the same scan sequence (see the comment above ClusterSmem; invalid and empty scans never enter it)
// and take the same branches (no measured node, duplicate key -- decided on the exchanged totals,
// identical on both sides).  The waits, for consecutive streamed scans s - 1, s and s + 1 of the cluster:
//   * The producer fills scan by scan and slot by slot and waits only on its own consumers' arrives: to load
//     chunk j of scan s + 1 into a held slot it waits for their mark of slot j of scan s; into any other slot,
//     for their place pass of scan s over slot j (a slot scan s does not use is free already).
//   * In the place pass of scan s, a consumer warp waits on slot j of scan s + 1 only after it has itself handed
//     back every slot of s up to j (held slots: all of them, at their mark; others: kMarkLag places before).
//     Take the lowest slot any warp waits on: every waiting warp has handed it back, and a warp that waits on
//     nothing runs on until it has handed back every slot of s -- no warp meets a barrier before it has marked
//     all of s + 1, so none can hold another up there.  All 16 arrives for that slot come, the producer, which
//     has filled every lower slot, fills it, and the wait ends.  By induction every mark of s + 1 ends.  There
//     is no block barrier between a warp's arrive on a slot and its wait on that slot's refill.
//   * The exchange of scan s + 1 comes after both CTAs have marked all of it, which needs nothing from the peer
//     past the rank table of s.  A CTA's rank table of s needs the peer's words of s, which the peer sends once
//     it has marked s (in its place pass of s - 1, or before its loop for the first scan), and the peer_free
//     arrive for s - 1, which the peer made in its rank table of s - 1 before it marked s.  Neither waits on
//     this CTA past the exchange of s - 1, which it has finished.  So no wait of either CTA closes a cycle.
// The producer warp never takes part in a cluster barrier while the loop runs;
// the whole cluster, producer warps included, meets in barrier.cluster exactly twice: after the barrier
// init (no remote arrive may reach an uninitialised barrier) and before exit (no CTA may exit while the
// peer can still store to its inbox or arrive on its barriers).
constexpr int kClusterSlots = 16;
constexpr uint32_t kClusterMaxNodes = 2u * kClusterSlots * CH;  // 32768
static_assert(kClusterMaxNodes <= kMaxFastNodes, "every scan the cluster kernel serves must be streamable");
// Slots per CTA whose chunks are held in registers from the mark to the place pass.  Timed on an H100 SXM (4096 x
// 32768-node Mode B launches): 0 / 4 / 6 / 8 / 10 / 12 held slots take 0.788 / 0.780 / 0.782 / 0.790 / 0.788 /
// 0.784-0.791 ms at 64 / 80 / 88 / 95 / 96 / 96 registers per thread, no spills (DESIGN.md §5.1).
constexpr int kHeld = 4;
static_assert(kHeld >= 0 && kHeld <= kClusterSlots, "held slots are a prefix of the tile");
// How many slots the next scan's mark trails the place front by, so that a slot's refill has landed by the time it
// is marked.  Timed on an H100 SXM at 700 W (4096 x 32768-node Mode B launches, three runs each, alternately):
// 2 / 4 / 6 slots take 0.744-0.745 / 0.744-0.745 / 0.752 ms (DESIGN.md §5.1).
constexpr uint32_t kMarkLag = 4;

// The scan sequence of a cluster.  A static round robin (cluster c takes scans c, c + C, c + 2 C, ... of C clusters)
// left the clusters ending up to 37 us apart on an H100 (DESIGN.md §5.1): clusters of the same work do not run at the
// same rate.  So rank 0's producer draws the scans at run time: the cluster's first two candidates are static (c and
// c + C), every later one comes from the call's ticket counter (2 C + atomicAdd(ticket, 1)), and without a ticket
// (single scans) the round robin goes on.  It reports the scans that are not streamed as the consumers' writer did,
// and keeps the streamed ones, in order, in a ring of kSeqSlots entries: seq[j % kSeqSlots] is the cluster's j-th
// scan, kSeqEnd once there is none.  It draws entry j + 2 once it has issued every load of entry j, so that both
// producers know each next scan while the current one still loads.  Rank 1 learns entries 0 and 1 from rank 0's ring
// after the first cluster barrier, and entry k + 2 with the exchange of entry k (inbox_next), which its consumer
// thread 0 then writes into its own ring.
//   Ring reuse.  Rank 0: its producer writes entry j + 2 after loading entry j's chunk 0 into slot 0, which needed
// every consumer warp's mark of entry j - 1's chunk 0, made after those threads had read entry j - 1 and so entry
// j - 2, the entry that slot (j + 2) % kSeqSlots held: no consumer can still be reading it.  Rank 1: its consumers read
// in order behind their own thread 0; its producer, which may run ahead through scans with no chunk of its own, frees
// each entry on seq_empty, and thread 0 waits there before it overwrites the entry.  That producer never waits on
// thread 0 for anything but entries already sent, so the wait ends.
constexpr int kSeqSlots = 4;
constexpr uint32_t kSeqEnd = 0xFFFFFFFFu;

struct __align__(128) ClusterSmem {
  uint8_t bytemap[kKeySpace];                // presence map of this CTA's nodes (swizzled)
  uint2 tile[kClusterSlots][CH];             // this CTA's half of the scan: chunk 2 j + rank in slot j
  uint2 rankV[kWords];                       // {bits, exclusive prefix} over the whole scan's measured keys
  uint4 inbox[kWords / 4];                   // the peer's bit-words of the current scan (written remotely)
  unsigned long long full[kClusterSlots];
  unsigned long long empty[kClusterSlots];
  unsigned long long inbox_full;             // the peer wrote inbox and inbox_count
  unsigned long long peer_free;              // the peer read the words this CTA wrote into its inbox
  unsigned long long seq_full[kSeqSlots];    // seq[j % kSeqSlots] holds the cluster's j-th scan
  unsigned long long seq_empty[kSeqSlots];   // rank 1: its producer has read the entry (rank 0 needs none, below)
  uint32_t seq[kSeqSlots];                   // the cluster's scan sequence (kSeqEnd after its last scan)
  uint32_t red[4 * kCWarps];
  uint32_t inbox_count;                      // the peer's measured-node count (written remotely)
  uint32_t inbox_next;                       // rank 1: the scan two places ahead in the sequence (written remotely)
  uint32_t valid_count;
  uint32_t totV;
};
static_assert(sizeof(ClusterSmem) <= 232448, "one CTA per SM: at most 227 KB of dynamic shared memory");
// words + count per scan; rank 1's inbox also takes the sequence entry rank 0 sends along
constexpr uint32_t kInboxBytes = sizeof(ClusterSmem::inbox) + sizeof(uint32_t);

// serves Mode B without the ascended buffer for strides in (kSmallMaxNodes, kClusterMaxNodes], 16-byte
// aligned scan bases; launched with cluster dims (2, 1, 1) and an even grid
__global__ void __launch_bounds__(kBlock, 1) scan_tma_cluster_kernel(ScanBatchArgs a, uint32_t max_nodes,
                                                                      uint32_t* ticket, unsigned long long* stamp) {
  stamp_start(stamp);
  extern __shared__ __align__(128) unsigned char smem_raw[];
  ClusterSmem& sm = *reinterpret_cast<ClusterSmem*>(smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
  const uint32_t s0 = blockIdx.x >> 1, s_step = gridDim.x >> 1;

  if (tid == 0) {
    for (int i = 0; i < kClusterSlots; ++i) {
      mbar_init(&sm.full[i], 1);         // the producer's arrive.expect_tx
      mbar_init(&sm.empty[i], kCWarps);  // one arrive per consumer warp (after the mark or the place pass)
    }
    mbar_init(&sm.inbox_full, 1);        // this CTA's arrive.expect_tx per scan + the peer's st.async bytes
    mbar_init(&sm.peer_free, 1);         // one remote arrive by the peer per scan
    for (int i = 0; i < kSeqSlots; ++i) {
      mbar_init(&sm.seq_full[i], 1);     // the entry's writer
      mbar_init(&sm.seq_empty[i], 1);    // rank 1's producer
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  // rank 0's producer: the next streamed scan of the cluster, or kSeqEnd; the others are reported here
  uint32_t drawn = 0;
  bool ended = false;
  auto claim = [&]() -> uint32_t {
    while (!ended) {
      const uint32_t k = drawn++;
      const uint32_t s = k < 2 || !ticket ? s0 + k * s_step : 2u * s_step + atomicAdd(ticket, 1u);
      if (s >= a.n_scans) break;
      const uint32_t n = a.counts[s];
      if (scan_is_streamed(n, a.stride, max_nodes)) return s;
      if (n == 0) write_outcome_empty(a, s);  // ascendScanData: OPERATION_FAIL; publish_scan: nodes.empty() -> return
      else write_outcome(a, s, kResultInvalidData, 0u, 0.0f);  // caller error: report, touch nothing
    }
    ended = true;
    return kSeqEnd;
  };
  auto seq_put = [&](uint32_t j, uint32_t v) {
    sm.seq[j % kSeqSlots] = v;
    mbar_arrive(&sm.seq_full[j % kSeqSlots]);
  };
  auto seq_get = [&](uint32_t j) {
    mbar_wait(&sm.seq_full[j % kSeqSlots], (j / kSeqSlots) & 1u);
    return *(volatile uint32_t*)&sm.seq[j % kSeqSlots];
  };
  if (rank == 0 && warp == kCWarps && lane == 0) {  // entries 0 and 1, published after the cluster barrier
    sm.seq[0] = claim();
    sm.seq[1] = claim();
  }
  cluster_sync_all();
  if (rank == 0 && warp == kCWarps && lane == 0) {
    mbar_arrive(&sm.seq_full[0]);
    mbar_arrive(&sm.seq_full[1]);
  }
  if (rank == 1 && tid == 0) {  // entries 0 and 1 from rank 0's ring (written before the cluster barrier)
    seq_put(0, ld_peer_u32(peer_addr(&sm.seq[0], 0)));
    seq_put(1, ld_peer_u32(peer_addr(&sm.seq[1], 0)));
  }

  if (warp == kCWarps) {
    // =========================== producer warp =========================================
    if (lane == 0) {
      const uint64_t pol_load = l2_policy_evict_normal();  // (see the L2 policy note above the kernel)
      uint32_t eph = 0xFFFFFFFFu;  // empty-barrier parity per slot: the first fill passes at once
      for (uint32_t js = 0;; ++js) {
        const uint32_t s = seq_get(js);
        if (rank == 1) mbar_arrive(&sm.seq_empty[js % kSeqSlots]);
        if (s == kSeqEnd) break;
        const uint32_t n = a.counts[s];
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
          tma_load_1d(&sm.tile[j][0], base + (size_t)c * CH, bytes, &sm.full[j], pol_load);
        }
        if (rank == 0) seq_put(js + 2, claim());
      }
    }
    __syncwarp();
  } else {
    // =========================== consumer warps ========================================
    const bool new_proto = a.is_new_protocol != 0;
    const bool inverted = a.inverted != 0;
    const IntensityOf intensity_of(new_proto);
    const bool writer = rank == 0 && tid == 0;  // per-scan outputs come from cluster rank 0
    const uint32_t peer_inbox = peer_addr(sm.inbox, peer);
    const uint32_t peer_count = peer_addr(&sm.inbox_count, peer);
    const uint32_t peer_inbox_full = peer_addr(&sm.inbox_full, peer);
    const uint32_t peer_next = peer_addr(&sm.inbox_next, peer);
    const uint32_t peer_peer_free = peer_addr(&sm.peer_free, peer);
    uint32_t fph = 0;                         // full-barrier parity per slot
    uint32_t in_par = 0, free_par = 1;        // exchange barriers: peer_free's first wait passes at once
    using Checked = std::integral_constant<bool, true>;
    using Unchecked = std::integral_constant<bool, false>;
    auto release = [&](uint32_t j) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[j]);
    };

    // this CTA's share of a streamed scan of n nodes (n = 0: no scan, no chunk)
    struct Half {
      uint32_t n, mine, mine_full, nheld;
    };
    auto half_of = [&](uint32_t n) {
      const uint32_t nch = (n + CH - 1) / CH, nfull = n / CH;
      Half h;
      h.n = n;
      h.mine = (nch + 1u - rank) >> 1;  // chunks c < nch with c & 1 == rank
      // the partial chunk (c == nfull < nch) is the last of this CTA's chunks if it is this CTA's at all
      h.mine_full = nfull < nch && (nfull & 1u) == rank ? h.mine - 1u : h.mine;
      h.nheld = min((uint32_t)kHeld, h.mine);
      return h;
    };

    uint32_t cnt = 0;  // measured nodes this thread has marked of the scan being marked
    uint8_t* const bmap = sm.bytemap;
    auto fetch = [&](uint32_t j, uint2 (&v)[kRounds]) {
      const uint2* slot = sm.tile[j];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) v[r] = slot[r * TC + tid];
    };
    auto wait_and_fetch = [&](uint32_t j, uint2 (&v)[kRounds]) {
      mbar_wait(&sm.full[j], (fph >> j) & 1u);
      fph ^= 1u << j;
      fetch(j, v);
    };
    auto mark_chunk = [&](auto checked, const uint2 (&v)[kRounds], uint32_t j, uint32_t n) {
      const uint32_t c = 2u * j + rank;
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        const uint32_t dist = __funnelshift_r(v[r].x, v[r].y, 16);
        bool valid = dist != 0;
        if (decltype(checked)::value && c * CH + r * TC + tid >= n) valid = false;
        if (valid) bmap[swz_x(v[r].x)] = 1;
        cnt += valid ? 1u : 0u;
      }
    };
    // held slot j: copied into registers, marked, and handed back at once (after the byte-map stores whose addresses
    // depend on the slot's values).  Every held chunk takes the tail mask, which is a no-op on the full ones.
    auto mark_held = [&](uint32_t j, const Half& h, uint2 (&v)[kRounds]) {
      wait_and_fetch(j, v);
      mark_chunk(Checked{}, v, j, h.n);
      release(j);
    };
    // any other slot: marked and left in shared memory for the place pass
    auto mark_resident = [&](uint32_t j, const Half& h) {
      uint2 v[kRounds];
      wait_and_fetch(j, v);
      if (j < h.mine_full) mark_chunk(Unchecked{}, v, j, h.n);
      else mark_chunk(Checked{}, v, j, h.n);
    };

    // The loop is software-pipelined over the cluster's streamed scans: an iteration starts with scan s marked
    // (its held chunks in held[]), folds, exchanges and ranks it, and places it while it marks the next streamed
    // scan s2 into the byte map, which is cleared right after s's fold.  Only constant indices into held[] and
    // next_held[] (no local memory).
    uint2 held[kHeld > 0 ? kHeld : 1][kRounds];
    uint2 next_held[kHeld > 0 ? kHeld : 1][kRounds];
    uint32_t js = 0;  // the sequence entry of s
    uint32_t s = seq_get(js);
    Half cur = half_of(s < a.n_scans ? a.counts[s] : 0u);
    if (s < a.n_scans) {  // the first scan is marked with no place pass to hide behind
      bytemap_clear(sm.bytemap, tid);
      consumer_sync();
#pragma unroll
      for (int j = 0; j < kHeld; ++j) {
        if (j < (int)cur.nheld) mark_held(j, cur, held[j]);
      }
      for (uint32_t j = cur.nheld; j < cur.mine; ++j) mark_resident(j, cur);
    }

    while (s < a.n_scans) {
      cnt = warp_sum(cnt);
      if (lane == 0) sm.red[warp] = cnt;
      // s2's counts stay in cnt until its fold: sm.red holds s's until rank_table has read them
      cnt = 0;
      consumer_sync();

      // ---- fold, exchange with the peer, rank table -----------------------------------------
      {
        uint32_t wv[kWordsPerThread];
        static_assert(kWordsPerThread == 4, "the exchange moves one uint4 of bit-words per thread");
        fold_row(sm.bytemap, tid, wv);
        // this scan's phase: the peer's words + count (+ rank 1: sequence entry js + 2)
        if (tid == 0) mbar_expect_tx(&sm.inbox_full, kInboxBytes + (rank == 1 ? 4u : 0u));
        mbar_wait_cluster(&sm.peer_free, free_par);  // the peer has read what this CTA sent for the last scan
        free_par ^= 1u;
        st_async_v4(peer_inbox + tid * 16u, make_uint4(wv[0], wv[1], wv[2], wv[3]), peer_inbox_full);
        if (warp == 0) {
          const uint32_t own = warp_sum(lane < kCWarps ? sm.red[lane] : 0u);
          if (lane == 0) st_async_u32(peer_count, own, peer_inbox_full);
          if (lane == 0 && rank == 0) st_async_u32(peer_next, seq_get(js + 2), peer_inbox_full);
        }
        mbar_wait_cluster(&sm.inbox_full, in_par);
        in_par ^= 1u;
        const uint4 pw = sm.inbox[tid];
        const uint32_t other = sm.inbox_count;
        if (rank == 1 && tid == 0) {  // entry js + 2 into this CTA's ring, once its producer has read entry js - 2
          const uint32_t jn = js + 2;
          mbar_wait(&sm.seq_empty[jn % kSeqSlots], ((jn / kSeqSlots) & 1u) ^ 1u);
          seq_put(jn, sm.inbox_next);
        }
        wv[0] |= pw.x;
        wv[1] |= pw.y;
        wv[2] |= pw.z;
        wv[3] |= pw.w;
        rank_table(sm, wv, tid, other);
        // every thread has used its inbox entry (rank_table's barriers): the peer may overwrite it
        if (tid == 0) mbar_arrive_remote(peer_peer_free);
        // every thread has folded its row (rank_table's barriers), and the fold maps threads to bytes unlike the
        // clear: clear the map for the next scan, whose first mark comes after the barrier below
        bytemap_clear(sm.bytemap, tid);
      }
      consumer_sync();
      const uint32_t M = sm.valid_count;  // measured nodes of the whole scan, the same in both CTAs

      const bool placing = M != 0 && sm.totV == M;
      if (writer && !placing) {
        if (M == 0) write_outcome_empty(a, s);
        else hand_to_general(a, s);  // duplicate keys, within a half or across the halves
      }
      const uint32_t s2 = seq_get(js + 1);
      const Half nx = half_of(s2 < a.n_scans ? a.counts[s2] : 0u);

      // ---- place this CTA's chunks of s by rank and mark those of s2 ----------------------------------------
      // s's slots still in shared memory go first, in ascending order, each handed back once placed (or at once if
      // s is not placed), so that the producer's next wait (on slot kHeld) is the first one met.  After each of
      // them one chunk of s2 is marked: its held chunks first, which the producer loaded during s's fold and
      // exchange, then its other chunks kMarkLag slots behind the place front, so that their refill has had time
      // to land.  Then s's held chunks are placed from registers, and the rest of s2 is marked.
      const ModeBOut mode_b(a.ranges + (size_t)s * a.stride, a.intensities + (size_t)s * a.stride, M, inverted,
                            l2_policy_evict_normal());
      auto place_chunk = [&](auto checked, const uint2 (&v)[kRounds], uint32_t j) {
        const uint32_t c = 2u * j + rank;
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          const uint2 nd = v[r];
          const uint32_t k = nd.x & 0xFFFFu;
          const uint32_t dist = __funnelshift_r(nd.x, nd.y, 16);
          uint32_t measured = dist != 0 ? 1u : 0u;
          if (decltype(checked)::value && c * CH + r * TC + tid >= cur.n) measured = 0;
          mode_b.store(rank_of(sm.rankV, k), dist_to_m(dist), intensity_of(nd.y), measured);
        }
      };
      auto place_resident = [&](uint32_t j) {
        if (placing) {
          uint2 v[kRounds];
          fetch(j, v);
          if (j < cur.mine_full) place_chunk(Unchecked{}, v, j);
          else place_chunk(Checked{}, v, j);
        }
        release(j);  // the held slots went back in the mark pass
      };
      uint32_t j = cur.nheld;  // s's next slot to place
#pragma unroll
      for (int h = 0; h < kHeld; ++h) {
        if (j < cur.mine) place_resident(j++);
        if (h < (int)nx.nheld) mark_held(h, nx, next_held[h]);
      }
      uint32_t jm = nx.nheld;  // s2's next slot to mark
      for (; j < cur.mine; ++j) {
        place_resident(j);
        if (jm + kMarkLag <= j && jm < nx.mine) mark_resident(jm++, nx);
      }
      if (placing) {
#pragma unroll
        for (int h = 0; h < kHeld; ++h) {
          if (h < (int)cur.nheld) place_chunk(Checked{}, held[h], h);
        }
        if (writer) write_outcome(a, s, kResultOk, M, angle_increment(M, false));
      }
      for (; jm < nx.mine; ++jm) mark_resident(jm, nx);

#pragma unroll
      for (int h = 0; h < kHeld; ++h) {
#pragma unroll
        for (int r = 0; r < kRounds; ++r) held[h][r] = next_held[h][r];
      }
      cur = nx;
      s = s2;
      ++js;
    }
  }
  // this CTA has no scan left: the general kernel, launched as this kernel's programmatic dependent, may be scheduled
  // onto the SMs the finished CTAs free (it waits for this whole kernel before it reads anything)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  cluster_sync_all();
  stamp_end(stamp);
}

}  // namespace

template <int MODE>
constexpr size_t kSmemOf = sizeof(TmaSmem<kStagesOf<MODE>>);

cudaError_t launch_scan_tma(const ScanBatchArgs& a, uint32_t max_nodes, int grid, cudaStream_t stream) {
  if (a.xyzi) scan_tma_kernel<2><<<grid, kBlock, kSmemOf<2>, stream>>>(a, max_nodes);
  else if (a.mode_a) scan_tma_kernel<1><<<grid, kBlock, kSmemOf<1>, stream>>>(a, max_nodes);
  else scan_tma_kernel<0><<<grid, kBlock, kSmemOf<0>, stream>>>(a, max_nodes);
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

cudaError_t launch_scan_tma_cluster(const ScanBatchArgs& a, uint32_t max_nodes, int grid, uint32_t* ticket,
                                    unsigned long long* stamp, cudaStream_t stream) {
  if (grid <= 0 || (grid & 1) != 0) return cudaErrorInvalidValue;
  ClusterLaunch l(grid, stream);
  return cudaLaunchKernelEx(&l.cfg, scan_tma_cluster_kernel, a, max_nodes, ticket, stamp);
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
