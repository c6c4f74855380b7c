// scan_fast.cu -- the hot kernel: fused ascendScanData + publish_scan for tie-free scans.
//
// Replaces, per scan (one CTA per scan, persistent over the batch):
//   ascendScanData_            reference src/sdk/src/sl_lidar_driver.cpp:128-184
//   publish_scan compute body  reference src/rplidar_node.cpp:581-677
//
// Idea: the sort key is the 16-bit angle_z_q14 (angle_rad is strictly monotonic in it), so
// for a scan whose keys are distinct the two std::sort calls collapse into a RANK LOOKUP:
//   mark    stream the packed nodes once from HBM (128-bit loads, L2 evict_last), mark a
//           65536-entry presence map in shared memory with plain byte stores (no atomics),
//   fold    turn the byte map into a bitmap + per-word exclusive popcount prefix,
//   place   stream the nodes again (L2 hits: the tile was just read; evict_first) and put
//           every point at rank(key) = prefix[key>>5] + popc(bits[key>>5] & below(key)).
// Mode B writes ranges[rank]; Mode A derives bin ownership (head / tail / empty-bin gaps)
// from the same bitmap; the ascended node buffer is a second rank over all nodes' final keys.
// A scan with duplicate keys (detected as popcount != count) is handed to the general
// radix-sort kernel through a device-side list -- results there follow the stable tie rule.
//
// HBM traffic per node: 8 B read + 4 B ranges + 4 B intensities (+8 B ascended node).
#include <type_traits>

#include "rpl_device.cuh"
#include "scan_args.h"
#include "scan_common.cuh"

namespace rpl {

namespace {

constexpr int T = kFastThreads;                 // 512 threads = 16 warps
constexpr int kWarps = T / 32;
constexpr int kUnroll = 8;
constexpr uint32_t kDummySlot = kKeySpace;      // where unmeasured nodes "mark"
static_assert(T == kMapThreads, "the byte-map fold is laid out for the whole block");

struct __align__(16) FastSmem {
  uint8_t bytemap[kKeySpace];      // presence map (swizzled)
  uint8_t dummy[16];
  uint2 rankV[kWords];             // {bits, exclusive prefix} over measured keys
  uint2 rankA[kWords];             // same over all nodes' final keys (ascended buffer)
  uint32_t vbits[kKeySpace / 32];  // measured flag per node index (ascended buffer only)
  uint32_t red[4 * kWarps];
  uint32_t valid_count;
  uint32_t first_valid;
  uint32_t front_key;
  uint32_t totV;
  uint32_t totA;
};

// ---- Mode A emit: the packed entries of the place pass, from a per-CTA global scratch ----------
// One warp of `nwarps`; E = entries in u-order.  Call with all 32 lanes converged.
//
// Ownership: a run (maximal stretch of equal bins) belongs to the warp whose slice holds its
// first entry.  The owner writes the run's bin and the empty bins in front of it; the owner of
// the last run also writes the empty bins behind it.  A warp therefore may read past the end of
// its slice to finish a run it owns, and skips leading entries that continue a run of the
// previous slice.
constexpr uint32_t kEmitBatch = 256;                 // entries a warp stages per batch
constexpr uint32_t kEmitStage = kEmitBatch + 33;     // + the entry before and 32 after (look-ahead)
constexpr uint32_t kEmitStageBytes = (kEmitStage * 12 + 15) & ~15u;  // u64 entry + i32 bin per staged entry

// Every entry is handled by one lane, independently of all others: the lane that holds the
// first entry of a run (bin differs from the previous entry's) takes the run's minimum by
// looking ahead, writes the bin, and fills the empty bins in front of it; the lane holding the
// very last entry fills the empty bins behind it.  A warp stages 256 entries (+ one before,
// 32 after) and their bins in its private slice of shared memory, so all loads and bin
// evaluations of a batch are in flight together and the per-entry work reads shared memory.
// `stage`: kEmitStageBytes of shared memory private to this warp.  Call converged.
__device__ __forceinline__ void mode_a_emit(const ModeAOut& o, const unsigned long long* E, uint32_t warp,
                                            uint32_t nwarps, unsigned char* stage) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t M = o.M;
  const uint32_t len = ((M + nwarps - 1u) / nwarps + kEmitBatch - 1u) & ~(kEmitBatch - 1u);  // whole batches
  const uint32_t r_begin = min(M, warp * len), r_end = min(M, r_begin + len);
  if (r_begin >= r_end) return;
  unsigned long long* se = reinterpret_cast<unsigned long long*>(stage);
  int* sb = reinterpret_cast<int*>(stage + kEmitStage * 8);
  // (int)((angle - angle_min) / angle_increment) with the reference's own float angle from the
  // table: exact, no double precision, no divergence
  auto bin_of = [&](unsigned long long e) {
    const float2 a = __ldg(o.angle + ((uint32_t)(e >> 8) & 0xFFFFu));
    return __float2int_rz(__fdiv_rn(o.inverted ? a.y : a.x, o.inc));
  };
  const int kNoBin = 0x7fffffff;
  const float kInf = __int_as_float(0x7f800000);

  for (uint32_t base = r_begin; base < r_end; base += kEmitBatch) {
    __syncwarp();
    for (uint32_t t = lane; t < kEmitStage; t += 32) {  // staged index t <-> rank base - 1 + t
      const long long r = (long long)base - 1 + t;
      unsigned long long e = ~0ull;
      int b = (r < 0) ? -1 : kNoBin;
      if (r >= 0 && r < (long long)M) {
        e = E[r];
        b = bin_of(e);
      }
      se[t] = e;
      sb[t] = b;
    }
    __syncwarp();
#pragma unroll 2
    for (uint32_t w = 0; w < kEmitBatch / 32; ++w) {
      const uint32_t i = 1 + w * 32 + lane;
      const uint32_t r = base + w * 32 + lane;
      const bool live = r < M;
      const int b = sb[i], bprev = sb[i - 1];
      const bool head = live && (b != bprev);
      unsigned long long v = se[i];
      if (head && sb[i + 1] == b) {
        v = min(v, se[i + 1]);
        if (sb[i + 2] == b) {  // a run of three or more: walk it (rare with M points in M bins)
          uint32_t j = i + 2;
          while (j < kEmitStage && sb[j] == b) {
            v = min(v, se[j]);
            ++j;
          }
          if (j == kEmitStage) {
            for (uint32_t rr = base - 1 + j; rr < M; ++rr) {
              const unsigned long long ee = E[rr];
              if (bin_of(ee) != b) break;
              v = min(v, ee);
            }
          }
        }
      }
      mode_a_store_bin(o, head ? b : 0, v, head ? 1u : 0u);
      if (head && b - bprev > 1) {  // empty bins in front of this run
        if (b - bprev == 2) {
          o.ranges[b - 1] = kInf;
          o.intens[b - 1] = 0.0f;
        } else {
          mode_a_fill_empty(o, bprev + 1, b);
        }
      }
      if (live && r == M - 1u) mode_a_fill_empty(o, b + 1, (int)M);  // empty bins behind the last run
    }
  }
}

template <bool EMIT, bool MODE_A>
__global__ void __launch_bounds__(T, 2) scan_fast_kernel(ScanBatchArgs a, FastWorkspace ws) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FastSmem& sm = *reinterpret_cast<FastSmem*>(smem_raw);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool new_proto = a.is_new_protocol != 0;
  const bool inverted = a.inverted != 0;
  // launches without the ascended buffer always produce the LaserScan (host guarantees it)
  const bool want_scan = EMIT ? (a.ranges != nullptr) : true;
  unsigned long long* gscratch = ws.group + (size_t)blockIdx.x * ws.max_nodes;
  const uint64_t pol_keep = l2_policy_evict_last();
  const uint64_t pol_stream = l2_policy_evict_first();
  const IntensityOf intensity_of(new_proto);
  using Checked = std::integral_constant<bool, true>;
  using Unchecked = std::integral_constant<bool, false>;

  for (uint32_t s = blockIdx.x; s < a.n_scans; s += gridDim.x) {
    const uint32_t n = a.counts[s];
    const uint2* base = a.nodes + (size_t)s * a.stride;

    if (n > a.stride || n > ws.max_nodes) {  // caller error: report, touch nothing
      if (tid == 0) write_outcome(a, s, kResultInvalidData, 0u, 0.0f);
      continue;
    }
    if (n > kMaxFastNodes) {  // cannot be tie-free: general kernel
      if (tid == 0) hand_to_general(a, s);
      continue;
    }

    // ---- phase 0: clear the presence map ------------------------------------------------
    bytemap_clear(sm.bytemap, tid);
    if (EMIT)
      for (uint32_t w = tid; w < kKeySpace / 32; w += T) sm.vbits[w] = 0;
    __syncthreads();

    // ---- phase 1 (mark): stream the scan from HBM, mark measured keys --------------------
    uint32_t cnt = 0;
    auto mark = [&](uint32_t x, uint32_t y) -> uint32_t {
      const uint32_t valid = __funnelshift_r(x, y, 16) != 0 ? 1u : 0u;
      sm.bytemap[valid ? swz_x(x) : kDummySlot] = 1;
      cnt += valid;
      return valid;
    };
    if (!EMIT) {
      // 128-bit loads, two nodes per lane; peel one node when the scan starts mid-16-bytes
      const uint32_t head = (n != 0 && (reinterpret_cast<uintptr_t>(base) & 8u)) ? 1u : 0u;
      const uint4* b4 = reinterpret_cast<const uint4*>(base + head);
      const uint32_t npairs = (n - head) >> 1;
      if (tid == 0) {
        if (head) {
          const uint2 nd = ld_hint_v2(base, pol_keep);
          mark(nd.x, nd.y);
        }
        if ((n - head) & 1u) {
          const uint2 nd = ld_hint_v2(base + n - 1, pol_keep);
          mark(nd.x, nd.y);
        }
      }
      auto block = [&](auto checked, uint32_t p0) {
        uint4 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint32_t p = p0 + u * T + tid;
          if (!decltype(checked)::value || p < npairs) v[u] = ld_hint_v4(b4 + p, pol_keep);
          else v[u] = make_uint4(0, 0, 0, 0);  // dist 0: marks the dummy slot
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          mark(v[u].x, v[u].y);
          mark(v[u].z, v[u].w);
        }
      };
      uint32_t p0 = 0;
      for (; p0 + T * kUnroll <= npairs; p0 += T * kUnroll) block(Unchecked{}, p0);
      if (p0 < npairs) block(Checked{}, p0);
    } else {
      // one node per lane so that a ballot is the measured mask of 32 consecutive nodes
      auto block = [&](auto checked, uint32_t i0) {
        uint2 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint32_t i = i0 + u * T + tid;
          if (!decltype(checked)::value || i < n) v[u] = ld_hint_v2(base + i, pol_keep);
          else v[u] = make_uint2(0, 0);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint32_t i = i0 + u * T + tid;
          const uint32_t valid = mark(v[u].x, v[u].y);
          const uint32_t bal = __ballot_sync(0xffffffffu, valid != 0);
          if (lane == 0 && (i >> 5) < kKeySpace / 32) sm.vbits[i >> 5] = bal;
        }
      };
      uint32_t i0 = 0;
      for (; i0 + T * kUnroll <= n; i0 += T * kUnroll) block(Unchecked{}, i0);
      if (i0 < n) block(Checked{}, i0);
    }
    cnt = warp_sum(cnt);
    if (lane == 0) sm.red[warp] = cnt;
    __syncthreads();
    if (warp == 0) {
      uint32_t c = lane < kWarps ? sm.red[lane] : 0u;
      c = warp_sum(c);
      uint32_t f = 0xFFFFFFFFu;
      if (EMIT) {  // first measured node = first set bit of vbits
        const uint32_t nw = (n + 31) >> 5;
        for (uint32_t w0 = 0; w0 < nw; w0 += 32) {
          const uint32_t w = w0 + lane;
          const uint32_t bits = w < nw ? sm.vbits[w] : 0u;
          const uint32_t any = __ballot_sync(0xffffffffu, bits != 0);
          if (any) {
            const uint32_t src = __ffs(any) - 1;
            const uint32_t b = __shfl_sync(0xffffffffu, bits, src);
            f = ((w0 + src) << 5) + __ffs(b) - 1;
            break;
          }
        }
      }
      if (lane == 0) {
        sm.valid_count = c;
        sm.first_valid = f;
        if (EMIT) {
          // head tune: serial, only node 0's result survives (reference :133-147)
          uint32_t fk = 0;
          if (c != 0) fk = ascend_head_key(node_key(ld_stream_v2(base + f)), f, ascend_step(n));
          sm.front_key = fk;
        }
      }
    }
    __syncthreads();
    const uint32_t M = sm.valid_count;

    if (M == 0) {
      if (tid == 0) write_outcome_empty(a, s);
      if (a.nodes_out) {
        uint2* out = a.nodes_out + (size_t)s * a.stride;
        for (uint32_t i = tid; i < n; i += T) out[i] = ld_stream_v2(base + i);
      }
      __syncthreads();
      continue;
    }

    const float step = ascend_step(n);
    const uint32_t front_key = EMIT ? sm.front_key : 0u;
    const float front_deg = key_to_deg(front_key);

    // ---- phase 1c (ascended buffer): mark the filled keys of unmeasured nodes -----------
    if (EMIT) {
      const uint32_t nw = (n + 31) >> 5;
      for (uint32_t w = tid; w < nw; w += T) {
        const uint32_t left = n - (w << 5);
        const uint32_t live = left >= 32 ? 0xFFFFFFFFu : ((1u << left) - 1u);
        uint32_t inv = ~sm.vbits[w] & live;
        while (inv) {
          const uint32_t b = __ffs(inv) - 1;
          inv &= inv - 1;
          const uint32_t i = (w << 5) + b;
          const uint32_t fk = (i == 0) ? front_key : ascend_fill_key(front_deg, i, step);
          sm.bytemap[swz_x(fk)] = 2;
        }
      }
      __syncthreads();
    }

    // ---- fold: byte map -> bitmaps + exclusive popcount prefix --------------------------
    {
      // thread t owns keys [128 t, 128 t + 128) = 4 bitmap words = 8 16-byte chunks
      uint32_t wv[4] = {0, 0, 0, 0}, wa[4] = {0, 0, 0, 0};
      const uint4* bm = reinterpret_cast<const uint4*>(sm.bytemap);
#pragma unroll
      for (uint32_t c = 0; c < 8; ++c) {
        const uint4 q = bm[tid * 8 + (c ^ (tid & 7u))];  // physical column of logical chunk c
        const uint32_t x[4] = {q.x, q.y, q.z, q.w};
        uint32_t bv = 0, bi = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          bv |= gather4(x[j] & 0x01010101u) << (4 * j);
          if (EMIT) bi |= gather4((x[j] >> 1) & 0x01010101u) << (4 * j);
        }
        wv[c >> 1] |= bv << (16 * (c & 1));
        if (EMIT) wa[c >> 1] |= (bv | bi) << (16 * (c & 1));
      }
      uint32_t sv = 0, sa = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sv += __popc(wv[j]);
        sa += __popc(wa[j]);
      }
      const uint32_t iv = warp_inclusive_scan(sv);
      const uint32_t ia = EMIT ? warp_inclusive_scan(sa) : 0u;
      if (lane == 31) {
        sm.red[2 * kWarps + warp] = iv;
        sm.red[3 * kWarps + warp] = ia;
      }
      __syncthreads();
      if (warp == 0) {
        uint32_t tv = lane < kWarps ? sm.red[2 * kWarps + lane] : 0u;
        uint32_t ta = lane < kWarps ? sm.red[3 * kWarps + lane] : 0u;
        const uint32_t cv = warp_inclusive_scan(tv), ca = warp_inclusive_scan(ta);
        if (lane < kWarps) {
          sm.red[2 * kWarps + lane] = cv - tv;
          sm.red[3 * kWarps + lane] = ca - ta;
        }
        if (lane == 31) {
          sm.totV = cv;
          sm.totA = ca;
        }
      }
      __syncthreads();
      uint32_t pv = sm.red[2 * kWarps + warp] + iv - sv;
      uint32_t pa = sm.red[3 * kWarps + warp] + ia - sa;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sm.rankV[tid * 4 + j] = make_uint2(wv[j], pv);
        pv += __popc(wv[j]);
        if (EMIT) {
          sm.rankA[tid * 4 + j] = make_uint2(wa[j], pa);
          pa += __popc(wa[j]);
        }
      }
    }
    __syncthreads();

    // duplicate keys -> general kernel (stable tie rule)
    const bool tie = (sm.totV != M) || (EMIT && sm.totA != n);
    if (tie) {
      if (tid == 0) hand_to_general(a, s);
      __syncthreads();
      continue;
    }

    // ---- phase 2 (place): stream again (L2), rank and place -------------------------------
    float* ranges = want_scan ? a.ranges + (size_t)s * a.stride : nullptr;
    float* intens = want_scan ? a.intensities + (size_t)s * a.stride : nullptr;
    uint2* nodes_out = EMIT ? a.nodes_out + (size_t)s * a.stride : nullptr;
    const float inc = angle_increment(M, MODE_A);
    const bool has0 = (sm.rankV[0].x & 1u) != 0;
    const ModeBOut mode_b(ranges, intens, M, inverted);
    auto place = [&](uint2 nd, uint32_t i, bool live) {
      const uint32_t k = nd.x & 0xFFFFu;
      const uint32_t dist = __funnelshift_r(nd.x, nd.y, 16);
      const uint32_t measured = (live && dist != 0) ? 1u : 0u;
      if (EMIT && live) {
        const uint32_t fk = measured ? k : (i == 0 ? front_key : ascend_fill_key(front_deg, i, step));
        st_hint_v2(nodes_out + rank_of(sm.rankA, fk), node_with_key(nd, fk), pol_stream);
      }
      if (!want_scan) return;
      const uint32_t r = rank_of(sm.rankV, k);
      const float dm = dist_to_m(dist);
      if (!MODE_A) {
        mode_b.store(r, dm, intensity_of(nd.y), measured);
      } else if (measured) {  // Mode A: packed entry at the u-rank, resolved by mode_a_emit
        gscratch[mode_a_urank(k, r, M, inverted, has0)] = mode_a_entry(dm, k, (nd.y >> 16) & 0xFFu);
      }
    };
    {
      auto block = [&](auto checked, uint32_t i0) {
        uint2 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint32_t i = i0 + u * T + tid;
          if (!decltype(checked)::value || i < n) v[u] = ld_hint_v2(base + i, pol_stream);
          else v[u] = make_uint2(0, 0);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const uint32_t i = i0 + u * T + tid;
          place(v[u], i, !decltype(checked)::value || i < n);
        }
      };
      uint32_t i0 = 0;
      for (; i0 + T * kUnroll <= n; i0 += T * kUnroll) block(Unchecked{}, i0);
      if (i0 < n) block(Checked{}, i0);
    }
    __syncthreads();

    // ---- phase 3 (Mode A): resolve bins that hold several points --------------------------
    if (MODE_A && want_scan) {
      ModeAOut mo;
      mo.ranges = ranges;
      mo.intens = intens;
      mo.angle = a.angle;
      mo.M = M;
      mo.inc = inc;
      mo.inverted = inverted;
      mo.new_proto = new_proto;
      mo.policy = pol_stream;
      // the presence map is dead by now: each warp stages entries in its own 3.4 KB of it
      static_assert(kEmitStageBytes * kWarps <= kKeySpace, "stage buffers must fit the byte map");
      mode_a_emit(mo, gscratch, warp, kWarps, sm.bytemap + warp * kEmitStageBytes);
    }
    __syncthreads();
    if (tid == 0) write_outcome(a, s, kResultOk, M, inc);
    __syncthreads();
  }
}

}  // namespace

size_t scan_fast_smem_bytes() { return sizeof(FastSmem); }

cudaError_t launch_scan_fast(const ScanBatchArgs& a, const FastWorkspace& ws, int grid,
                             cudaStream_t stream) {
  const bool emit = a.nodes_out != nullptr && a.apply_ascend != 0;
  const bool mode_a = a.mode_a != 0;
  const size_t sh = sizeof(FastSmem);
  if (emit && mode_a) scan_fast_kernel<true, true><<<grid, T, sh, stream>>>(a, ws);
  else if (emit) scan_fast_kernel<true, false><<<grid, T, sh, stream>>>(a, ws);
  else if (mode_a) scan_fast_kernel<false, true><<<grid, T, sh, stream>>>(a, ws);
  else scan_fast_kernel<false, false><<<grid, T, sh, stream>>>(a, ws);
  return cudaGetLastError();
}

cudaError_t scan_fast_configure() {
  const int sh = (int)sizeof(FastSmem);
  cudaError_t e;
  e = cudaFuncSetAttribute(scan_fast_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sh);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(scan_fast_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sh);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(scan_fast_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sh);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(scan_fast_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sh);
}

int scan_fast_max_ctas_per_sm() {
  int nb = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, scan_fast_kernel<false, false>, T, sizeof(FastSmem));
  return nb;
}

}  // namespace rpl
