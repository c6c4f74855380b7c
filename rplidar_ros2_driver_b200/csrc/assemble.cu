// assemble.cu -- scan assembly on the GPU (SURVEY.md 8(f) rank 2): cuts decoded node streams into
// scans, the bridge between the decoders and the scan kernels without a host round trip.
//
// Replaces ScanDataHolder::pushScanNodeData / rewindCurrentScanData (reference
// src/sdk/src/sl_lidar_driver.cpp:272-315) as a pure function of the node stream and the
// scan-reset requests (one per scan-start capsule, SlamtecLidarDriver::onHQNodeScanResetReq
// :1651-1653):
//   * a node with flag bit 0 opens a scan and publishes the scan in progress if it holds anything;
//     nodes before the first such node are dropped; the last, unfinished scan is not published;
//   * a reset empties the scan in progress: the scan [s, e) between two scan-start nodes is
//     published iff no reset position r satisfies s < r <= e;
//   * a scan longer than max_nodes (8192 in the SDK) keeps overwriting its last entry.
// One CTA per stream.  Scan starts are rare (one per revolution), so the flag pass just appends
// their positions to a small shared-memory list (unordered, one atomic per scan start) and rank-sorts
// it; reset counts come from a prefix over the capsule flags + binary search; published scans are
// compacted into descriptors and then copied coalesced.  A stream with more scan starts than the
// list holds takes the chunked block-scan path instead (same result, more barriers).
#include "decode_args.h"
#include "delay_model.cuh"
#include "rpl_device.cuh"

namespace rpl {

namespace {

constexpr int AT = 512;
constexpr uint32_t kListCap = 4096, kResetCap = 1024;  // scan starts per stream handled by the list path
constexpr uint32_t kStSync = 2, kStDiscard = 8, kStChecksum = 16, kStEncReset = 32, kStBadFrame = 64;

// STREAM: the counters this push adds to a stream's StreamCounters (s_ct, summed over the CTA)
enum : uint32_t { kCtChecksum, kCtEncReset, kCtDiscard, kCtBadFrame, kCtUnopened, kCtOverwritten, kCtN };
__device__ __forceinline__ void block_count(uint32_t* s_ct, uint32_t i, uint32_t v) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(s_ct + i, v);
}

__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* warp_tot, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t inc = warp_inclusive_scan(v);
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < AT / 32; ++w) {
    const uint32_t t = warp_tot[w];
    if ((uint32_t)w < warp) base += t;
    tot += t;
  }
  __syncthreads();
  *total = tot;
  return base + inc - v;
}

// ascending rank sort of a short list (duplicates keep their list order)
__device__ __forceinline__ void rank_sort(const uint32_t* in, uint32_t* out, uint32_t k) {
  for (uint32_t e = threadIdx.x; e < k; e += AT) {
    const uint32_t v = in[e];
    uint32_t r = 0;
    for (uint32_t j = 0; j < k; ++j) {
      const uint32_t w = in[j];
      r += (w < v || (w == v && j < e)) ? 1u : 0u;
    }
    out[r] = v;
  }
}

// STREAM: a stream session's instantiation, any capsule format (AssembleArgs::carry_len): positions count from the first
// node of the revolution carried in front of the new nodes, which is a scan start like any other -- listed first when
// the decoder hands a scan-start list over (dense), found by the flag pass like the others when it does not.
// STAMPED (a stamped session push, STREAM only): also the stamp of every published scan's scan-start node and of the
// open revolution's first node, computed for those nodes alone (sa, and the delay model m0 or, with a per-stream table,
// the stream's own)
// LIST (a mixed byte session, STREAM only): CTA slot i serves stream list.streams[i] of the chunk
template <bool STREAM, bool STAMPED, bool LIST>
__device__ __forceinline__ void assemble_body(const AssembleArgs& a, const AssembleStampArgs& sa, const DelayModel& m0,
                                              const StreamList& list) {
  static_assert(STREAM || !STAMPED, "stamps are a stream session's");
  static_assert(STREAM || !LIST, "stream lists are a stream session's");
  __shared__ uint32_t s_list[kListCap], s_sorted[kListCap];      // scan-start positions
  __shared__ uint32_t s_rlist[kResetCap], s_rsorted[kResetCap];  // reset positions
  __shared__ uint32_t s_cnt, s_rcnt;
  __shared__ uint32_t s_warp[AT / 32];
  __shared__ int s_wmax[AT / 32];
  __shared__ int s_last_sync;       // position of the latest scan-start node seen so far (-1: none)
  __shared__ uint32_t s_published;  // scans published so far
  __shared__ int s_open;            // STREAM: first node of the revolution left open (-1: none, or a reset emptied it)
  __shared__ uint32_t s_ct[kCtN];   // STREAM: this push's counts (block_count)
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (uint32_t i = blockIdx.x; i < a.n_streams; i += gridDim.x) {
    const uint32_t s = LIST ? list.streams[i] : i;
    DelayModel m = m0;
    if constexpr (STAMPED)
      if (sa.lidars) m = delay_model(sa.ans_type, sa.lidars[s].timing);
    const uint32_t L = STREAM ? a.carry_len[s] : 0u;           // carried nodes
    const uint32_t base = STREAM ? a.max_nodes - L : 0u;        // position 0 within the stream's region
    const uint32_t n = a.node_counts[s] + L;
    const uint2* nodes = a.nodes + (size_t)s * a.stride_nodes + base;
    const bool have_resets = a.capsule_status != nullptr;
    const uint32_t ncap = !have_resets ? 0u : STREAM ? min(a.capsule_counts[s], a.stride_capsules) : a.capsule_counts[s];
    const uint32_t* cst = have_resets ? a.capsule_status + (size_t)s * a.stride_capsules : nullptr;
    const uint32_t* coff = have_resets ? a.capsule_node_offset + (size_t)s * a.stride_capsules : nullptr;
    uint32_t* rs = a.reset_prefix + (size_t)s * a.stride_capsules;  // inclusive count of reset capsules
    uint2* desc = a.desc + (size_t)s * a.max_scans;                 // (start, length) of published scans
    uint2* out = a.scans_out + (size_t)s * a.max_scans * a.scan_stride;
    uint32_t* out_len = a.scan_len + (size_t)s * a.max_scans;
    // STAMPED: the stamp of the scan-start node at position x (ScanDataHolder::_scan_begin_timestamp_uS), what the
    // timestamp kernels would have written for it.  The only scan start among the carried nodes is the carried
    // revolution's first, at 0.  A capsule-format node was released by the last capsule whose node offset is <= its
    // index (a capsule that releases nothing shares the next release's offset); a 0x81 node takes the receive time of
    // the chunk its record's last byte came in.
    unsigned long long open_in = 0, held_rx_in = kRxUnknown;
    if constexpr (STAMPED) {
      if (sa.prev_stamped) {
        open_in = sa.open_ts_in[s];
        if (m.prev_base) held_rx_in = sa.held_rx[s];
      }
    }
    const unsigned long long* crx = STAMPED && have_resets ? sa.capsule_rx_us + (size_t)s * a.stride_capsules : nullptr;
    auto stamp_at = [&](uint32_t x) -> unsigned long long {
      if constexpr (!STAMPED) {
        return 0ull;
      } else {
        if (x < L) return open_in;
        const uint32_t y = x - L;
        if (!have_resets) {  // 0x81
          const uint32_t e = sa.node_end[(size_t)s * sa.stride_ends + y];
          return sa.chunk_rx_us[(size_t)s * sa.stride_chunks + e / sa.chunk_bytes] - m.base;
        }
        uint32_t lo = 0, hi = ncap;  // first capsule with offset > y (>= 1: node y was released)
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (coff[mid] <= y) lo = mid + 1;
          else hi = mid;
        }
        const uint32_t j = lo - 1;
        // express, ultra: the released capsule's own receive time, the held one's for capsule 0
        if (m.prev_base && j == 0 && held_rx_in == kRxUnknown) return 0ull;
        const unsigned long long rx = !m.prev_base ? crx[j] : j ? crx[j - 1] : held_rx_in;
        unsigned long long d = m.base;
        if (m.group >= 0) d += (unsigned long long)(m.group - (int)(y - coff[j])) * m.sd;
        return rx - d;
      }
    };

    if (tid == 0) {
      s_cnt = 0;
      s_rcnt = 0;
      s_last_sync = -1;
      s_published = 0;
    }
    if constexpr (STREAM)
      if (tid < kCtN) s_ct[tid] = 0;
    __syncthreads();
    // ---- flag pass: positions of the scan-start nodes and of the reset requests -----------------------
    uint32_t n_chk = 0, n_enc = 0, n_disc = 0, n_bad = 0;  // STREAM: the capsule reports' events
    for (uint32_t j = tid; j < ncap; j += AT) {
      const uint32_t v = cst[j];
      if (v & kStSync) {
        const uint32_t idx = atomicAdd(&s_rcnt, 1u);
        if (idx < kResetCap) s_rlist[idx] = coff[j] + L;
      }
      if constexpr (STREAM) {
        n_chk += (v & kStChecksum) ? 1u : 0u;
        n_enc += (v & kStEncReset) ? 1u : 0u;
        n_disc += (v & kStDiscard) ? 1u : 0u;
        n_bad += (v & kStBadFrame) ? 1u : 0u;
      }
    }
    if constexpr (STREAM) {
      block_count(s_ct, kCtChecksum, n_chk);
      block_count(s_ct, kCtEncReset, n_enc);
      block_count(s_ct, kCtDiscard, n_disc);
      block_count(s_ct, kCtBadFrame, n_bad);
    }
    // the decoder may have handed the scan-start positions over (rpl_decode_dense_batch_starts_dev): then the node
    // stream is not read again at all
    const uint32_t n_listed = (a.scan_starts && a.scan_start_counts) ? a.scan_start_counts[s] : 0xFFFFFFFFu;
    const uint32_t lead = (STREAM && L > 0) ? 1u : 0u;  // the carried revolution's scan start, at 0
    if (n_listed <= a.starts_stride && n_listed + lead <= kListCap) {
      const uint32_t* lst = a.scan_starts + (size_t)s * a.starts_stride;
      for (uint32_t e = tid; e < n_listed; e += AT) s_list[e + lead] = lst[e] + L;
      if (tid == 0) {
        if (lead) s_list[0] = 0;
        s_cnt = n_listed + lead;
      }
    } else {
      const uint32_t* flags = reinterpret_cast<const uint32_t*>(nodes) + 1;  // word 1 of every node
      uint32_t i = tid;
      for (; i + 3 * AT < n; i += 4 * AT) {
        const uint32_t y0 = __ldg(flags + 2 * (size_t)i), y1 = __ldg(flags + 2 * (size_t)(i + AT));
        const uint32_t y2 = __ldg(flags + 2 * (size_t)(i + 2 * AT)), y3 = __ldg(flags + 2 * (size_t)(i + 3 * AT));
        if (((y0 | y1 | y2 | y3) >> 24) & 1u) {
          const uint32_t yy[4] = {y0, y1, y2, y3};
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if ((yy[u] >> 24) & 1u) {
              const uint32_t idx = atomicAdd(&s_cnt, 1u);
              if (idx < kListCap) s_list[idx] = i + u * AT;
            }
          }
        }
      }
      for (; i < n; i += AT) {
        if ((__ldg(flags + 2 * (size_t)i) >> 24) & 1u) {
          const uint32_t idx = atomicAdd(&s_cnt, 1u);
          if (idx < kListCap) s_list[idx] = i;
        }
      }
    }
    __syncthreads();
    const uint32_t K = s_cnt, RK = s_rcnt;
    if (K <= kListCap && RK <= kResetCap) {
      // ---- list path ---------------------------------------------------------------------------------
      rank_sort(s_list, s_sorted, K);
      rank_sort(s_rlist, s_rsorted, RK);
      __syncthreads();
      auto resets_upto = [&](uint32_t x) -> uint32_t {  // number of reset positions <= x
        uint32_t lo = 0, hi = RK;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (s_rsorted[mid] <= x) lo = mid + 1;
          else hi = mid;
        }
        return lo;
      };
      for (uint32_t k0 = 0; k0 + 1 < K; k0 += AT) {
        const uint32_t k = k0 + tid;
        uint32_t publish = 0, st = 0, en = 0;
        if (k + 1 < K) {
          st = s_sorted[k];
          en = s_sorted[k + 1];
          publish = (resets_upto(en) == resets_upto(st)) ? 1u : 0u;
        }
        uint32_t tot = 0;
        const uint32_t ex = block_excl_scan(publish, s_warp, &tot);
        if (publish) {
          const uint32_t slot = s_published + ex;
          if (slot < a.max_scans) desc[slot] = make_uint2(st, en - st);
        }
        __syncthreads();
        if (tid == 0) s_published += tot;
        __syncthreads();
      }
      if constexpr (STREAM) {
        // the holder's losses per revolution [start, end): the first reset after its start empties it, and the nodes
        // from there to the next scan start find no scan open; the nodes it kept past max_nodes overwrote its last
        // entry.  The nodes in front of the first scan start (none behind a carried revolution) find none either.
        uint32_t unopened = (tid == 0) ? (K ? s_sorted[0] : n) : 0u, overwritten = 0;
        for (uint32_t k = tid; k < K; k += AT) {
          const uint32_t st = s_sorted[k], en = k + 1 < K ? s_sorted[k + 1] : n;
          const uint32_t ri = resets_upto(st);
          const uint32_t cut = ri < RK ? min(s_rsorted[ri], en) : en;
          unopened += en - cut;
          overwritten += cut - st > a.max_nodes ? cut - st - a.max_nodes : 0u;
        }
        block_count(s_ct, kCtUnopened, unopened);
        block_count(s_ct, kCtOverwritten, overwritten);
      }
      // the revolution after the last scan start stays open unless a reset follows its start
      if (STREAM && tid == 0) s_open = (K > 0 && resets_upto(s_sorted[K - 1]) == RK) ? (int)s_sorted[K - 1] : -1;
    } else {
      // ---- many scan starts: chunked block scans over the flags ---------------------------------------
      uint32_t carry = 0;
      for (uint32_t c0 = 0; c0 < ncap; c0 += AT) {
        const uint32_t j = c0 + tid;
        const uint32_t v = (j < ncap && (cst[j] & kStSync)) ? 1u : 0u;
        uint32_t tot = 0;
        const uint32_t ex = block_excl_scan(v, s_warp, &tot);
        if (j < ncap) rs[j] = carry + ex + v;
        carry += tot;
      }
      __syncthreads();
      auto resets_upto = [&](uint32_t x) -> uint32_t {
        if (!have_resets || ncap == 0) return 0u;
        uint32_t lo = 0, hi = ncap;  // first capsule with offset > x
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (coff[mid] + L <= x) lo = mid + 1;
          else hi = mid;
        }
        return lo ? rs[lo - 1] : 0u;
      };
      for (uint32_t c0 = 0; c0 < n; c0 += AT) {
        const uint32_t i = c0 + tid;
        const bool sync = i < n && ((nodes[i].y >> 24) & 1u);
        // previous scan-start position: exclusive running maximum of the sync positions
        int m = sync ? (int)i : -1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, m, o);
          if (lane >= (uint32_t)o) m = max(m, t);
        }
        if (lane == 31) s_wmax[warp] = m;
        __syncthreads();
        int prev = __shfl_up_sync(0xffffffffu, m, 1);
        if (lane == 0) prev = -1;
        int before = s_last_sync;
        for (uint32_t w = 0; w < warp; ++w) before = max(before, s_wmax[w]);
        prev = max(prev, before);
        uint32_t publish = 0;
        if (sync && prev >= 0) publish = (resets_upto(i) == resets_upto((uint32_t)prev)) ? 1u : 0u;
        if constexpr (STREAM) {
          // the holder's losses node by node: a node finds no scan open when no scan start precedes it or a reset
          // came after that start; one kept max_nodes or more behind its scan start overwrote the last entry
          uint32_t unopened = 0, overwritten = 0;
          if (i < n && !sync) {
            if (prev < 0 || resets_upto(i) != resets_upto((uint32_t)prev)) unopened = 1;
            else if (i - (uint32_t)prev >= a.max_nodes) overwritten = 1;
          }
          block_count(s_ct, kCtUnopened, unopened);
          block_count(s_ct, kCtOverwritten, overwritten);
        }
        uint32_t tot = 0;
        const uint32_t ex = block_excl_scan(publish, s_warp, &tot);  // syncs
        if (publish) {
          const uint32_t k = s_published + ex;
          if (k < a.max_scans) desc[k] = make_uint2((uint32_t)prev, i - (uint32_t)prev);
        }
        __syncthreads();
        if (tid == 0) {
          int last = s_last_sync;
          for (int w = 0; w < AT / 32; ++w) last = max(last, s_wmax[w]);
          s_last_sync = last;
          s_published += tot;
        }
        __syncthreads();
      }
      if (STREAM && tid == 0) {
        const int ls = s_last_sync;
        s_open = (ls >= 0 && resets_upto((uint32_t)ls) == carry) ? ls : -1;
      }
    }
    __syncthreads();
    const uint32_t total = s_published;
    if (tid == 0) a.scans_per_stream[s] = total;
    if constexpr (STREAM) {
      if (tid == 0) {
        // K counts every scan start (the lists keep counting past their capacity): each closes the revolution before
        // it, published unless a reset emptied it, and a reset after the last one empties the open revolution
        StreamCounters& c = a.counters[s];
        if (a.counted_capsule_bytes) {
          c.frames += ncap;
          c.bytes_in += (unsigned long long)ncap * a.counted_capsule_bytes;
        }
        c.bad_frames += s_ct[kCtBadFrame];
        c.checksum_errors += s_ct[kCtChecksum];
        c.encoder_resets += s_ct[kCtEncReset];
        c.scan_resets += RK;
        c.discarded_capsules += s_ct[kCtDiscard];
        c.nodes += a.node_counts[s];
        c.nodes_unopened += s_ct[kCtUnopened];
        c.nodes_overwritten += s_ct[kCtOverwritten];
        c.scans_rewound += K ? K - 1 - total + (s_open < 0 ? 1u : 0u) : 0u;
        c.scans_published += total;
        c.scans_unreturned += total > a.max_scans ? total - a.max_scans : 0u;
      }
    }
    // ---- copy the published scans (descriptors were written by this CTA: visible after the barrier) ---
    const uint32_t stored = min(total, a.max_scans);
    if (a.views_out) {
      // view mode: no copy.  A published scan is handed on as (first node, count) into the node buffer itself;
      // a scan that hit the holder's capacity gets the holder's "replace the last entry" applied in place
      // (the nodes behind the cap are dropped either way).
      uint2* vout = a.views_out + (size_t)s * a.max_scans;
      for (uint32_t k = tid; k < a.max_scans; k += AT) {
        uint2 v = make_uint2(0u, 0u);
        if (k < stored) {
          const uint2 d = desc[k];
          const uint32_t cnt = min(d.y, a.max_nodes);
          if (d.y > cnt) a.nodes_mut[(size_t)s * a.stride_nodes + base + d.x + cnt - 1] = nodes[d.x + d.y - 1];
          v = make_uint2((uint32_t)((size_t)s * a.stride_nodes + base + d.x), cnt);
          if constexpr (!STAMPED) {
            if (a.scan_begin_ts_us)
              a.scan_begin_ts_us[(size_t)s * a.max_scans + k] =
                  a.node_ts_us ? a.node_ts_us[(size_t)s * a.stride_nodes + base + d.x] : 0ull;
          }
        }
        if constexpr (STAMPED) {
          // the end: the closing scan-start node at desc.x + desc.y, also for the last stored slot of a stream that
          // published more than max_scans (the first dropped scan's begin)
          const size_t o = (size_t)s * a.max_scans + k;
          const unsigned long long b = k < stored ? stamp_at(desc[k].x) : 0ull;
          a.scan_begin_ts_us[o] = b;
          sa.slot_begin_us[o] = b;
          sa.slot_end_us[o] = k < stored ? stamp_at(desc[k].x + desc[k].y) : 0ull;
        }
        vout[k] = v;
        out_len[k] = v.y;
      }
      if constexpr (STREAM) {
        // the open revolution, capped by the holder's rule, right-aligned into the other arena's carry slots (none of
        // its nodes is a published scan's, so the in-place cap above never touches them)
        const int ls = s_open;
        const uint32_t t = ls >= 0 ? n - (uint32_t)ls : 0u, tc = min(t, a.max_nodes);
        const uint2* src = nodes + (ls >= 0 ? ls : 0);
        uint2* dst = a.carry_out + (size_t)s * a.stride_nodes + a.max_nodes - tc;
        const uint32_t ncopy = t > tc ? tc - 1 : tc;
        for (uint32_t q = tid; q < ncopy; q += AT) dst[q] = src[q];
        if (tid == 0) {
          if (t > tc) dst[tc - 1] = src[t - 1];
          a.carry_len_out[s] = tc;
          if constexpr (STAMPED) {
            // every thread has read held_rx_in (before the first barrier of this stream)
            sa.open_ts_out[s] = ls >= 0 ? stamp_at((uint32_t)ls) : 0ull;
            if (m.prev_base) sa.held_rx[s] = ncap ? crx[ncap - 1] : held_rx_in;
          }
        }
      }
      __syncthreads();
      continue;
    }
    for (uint32_t k = 0; k < stored; ++k) {
      const uint2 d = desc[k];
      const uint32_t cnt = min(d.y, a.max_nodes);
      uint2* o = out + (size_t)k * a.scan_stride;
      const uint2* src = nodes + d.x;
      // a scan that hit the cap kept overwriting its last entry: its last slot takes the scan's last node.
      // The copy leaves that slot alone (one writer per output element, no ordering between threads needed).
      const bool capped = d.y > cnt;
      const uint32_t ncopy = capped ? cnt - 1 : cnt;
      uint32_t q = tid;
      for (; q + 3 * AT < ncopy; q += 4 * AT) {  // four independent loads in flight per thread
        const uint2 v0 = ld_hint_v2(src + q, l2_policy_evict_first()), v1 = ld_hint_v2(src + q + AT, l2_policy_evict_first());
        const uint2 v2 = ld_hint_v2(src + q + 2 * AT, l2_policy_evict_first()), v3 = ld_hint_v2(src + q + 3 * AT, l2_policy_evict_first());
        o[q] = v0;
        o[q + AT] = v1;
        o[q + 2 * AT] = v2;
        o[q + 3 * AT] = v3;
      }
      for (; q < ncopy; q += AT) o[q] = src[q];
      if (tid == 0) {
        if (capped) o[cnt - 1] = src[d.y - 1];
        out_len[k] = cnt;
        // the scan-start node's stamp (ScanDataHolder::_scan_begin_timestamp_uS, sl_lidar_driver.cpp:293)
        if (a.scan_begin_ts_us)
          a.scan_begin_ts_us[(size_t)s * a.max_scans + k] =
              a.node_ts_us ? a.node_ts_us[(size_t)s * a.stride_nodes + d.x] : 0ull;
      }
    }
    __syncthreads();
  }
}

template <bool STREAM>
__global__ void __launch_bounds__(AT) assemble_kernel(AssembleArgs a) {
  assemble_body<STREAM, false, false>(a, AssembleStampArgs{}, DelayModel{}, StreamList{});
}

__global__ void __launch_bounds__(AT) assemble_stamped_kernel(AssembleArgs a, AssembleStampArgs sa, DelayModel m) {
  assemble_body<true, true, false>(a, sa, m, StreamList{});
}

template <bool STAMPED>
__global__ void __launch_bounds__(AT) assemble_list_kernel(AssembleArgs a, AssembleStampArgs sa, DelayModel m,
                                                           StreamList l) {
  assemble_body<true, STAMPED, true>(a, sa, m, l);
}

}  // namespace

cudaError_t launch_assemble(const AssembleArgs& a, int grid, cudaStream_t stream, const StreamList* list) {
  if (a.n_streams == 0) return cudaSuccess;
  if (list)
    assemble_list_kernel<false><<<grid, AT, 0, stream>>>(a, AssembleStampArgs{}, DelayModel{}, *list);
  else if (a.carry_len)
    assemble_kernel<true><<<grid, AT, 0, stream>>>(a);
  else
    assemble_kernel<false><<<grid, AT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_assemble_stamped(const AssembleArgs& a, const AssembleStampArgs& sa, int grid, cudaStream_t stream,
                                    const StreamList* list) {
  if (a.n_streams == 0) return cudaSuccess;
  if (list)
    assemble_list_kernel<true><<<grid, AT, 0, stream>>>(a, sa, delay_model(sa.ans_type, sa.timing), *list);
  else
    assemble_stamped_kernel<<<grid, AT, 0, stream>>>(a, sa, delay_model(sa.ans_type, sa.timing));
  return cudaGetLastError();
}

}  // namespace rpl
