// session_migrate.cu -- a stream session's carried state in and out of records (rpl_capsule_stream_export / _import):
// the pack kernel gathers each listed stream's held and framer records, stamps, counters and open revolution into its
// record in a device staging buffer, the unpack kernel scatters validated records back into a session.  One CTA serves
// one record at a time; every part of a record is 16-byte aligned, and so is every per-stream array it mirrors, so the
// fixed part moves in 16-byte words, the open nodes too when the revolution starts on an even arena slot.
#include <algorithm>

#include "session_migrate_args.h"

namespace rpl {
namespace {

constexpr int MT = 256;

__device__ __forceinline__ void copy16(uint4* dst, const uint4* src, uint32_t n16) {
  for (uint32_t w = threadIdx.x; w < n16; w += MT) dst[w] = src[w];
}

// the open revolution: arena slots [max_nodes - L, max_nodes) of the stream's region <-> the record's node part
template <bool PACK>
__device__ __forceinline__ void copy_nodes(uint2* arena_tail, uint2* rec_nodes, uint32_t L) {
  if ((reinterpret_cast<uintptr_t>(arena_tail) & 15u) == 0) {
    uint4* a4 = reinterpret_cast<uint4*>(arena_tail);
    uint4* r4 = reinterpret_cast<uint4*>(rec_nodes);
    for (uint32_t w = threadIdx.x; w < L / 2; w += MT) {
      if (PACK) r4[w] = a4[w];
      else a4[w] = r4[w];
    }
    if ((L & 1u) && threadIdx.x == 0) {
      if (PACK) rec_nodes[L - 1] = arena_tail[L - 1];
      else arena_tail[L - 1] = rec_nodes[L - 1];
    }
  } else {
    for (uint32_t i = threadIdx.x; i < L; i += MT) {
      if (PACK) rec_nodes[i] = arena_tail[i];
      else arena_tail[i] = rec_nodes[i];
    }
  }
}

__global__ void __launch_bounds__(MT) stream_pack_kernel(MigrateArgs a) {
  for (uint32_t i = blockIdx.x; i < a.n; i += gridDim.x) {
    const uint32_t s = a.streams[i];
    const uint32_t type = a.types[i];
    const bool framer = a.framer && a.kind && type != 0x81u;
    uint8_t* rec = a.records + a.offsets[i];
    const uint32_t L = a.carry_len[s];
    uint8_t* p = rec + kRecHeaderBytes;
    copy16(reinterpret_cast<uint4*>(p), reinterpret_cast<const uint4*>(a.held + (size_t)s * kHeldWords), kRecHeldBytes / 16);
    p += kRecHeldBytes;
    if (framer) {
      copy16(reinterpret_cast<uint4*>(p), reinterpret_cast<const uint4*>(a.framer + (size_t)s * kFramerWords),
             kRecFramerBytes / 16);
      p += kRecFramerBytes;
    }
    if (threadIdx.x == 0) {
      const unsigned long long open = a.stamps_known ? a.open_ts[s] : 0ull;
      const unsigned long long rx = a.stamps_known ? a.held_rx[s] : kRxUnknown;
      const uint32_t flags = (open != 0ull ? kRecOpenKnown : 0u) | (rx != kRxUnknown ? kRecRxKnown : 0u);
      uint32_t* h = reinterpret_cast<uint32_t*>(rec);
      h[kRecWordMagic] = kRecMagic;
      h[kRecWordVersion] = kRecVersion;
      h[kRecWordKind] = a.kind;
      h[kRecWordType] = type;
      h[kRecWordMaxNodes] = a.max_nodes;
      h[kRecWordOpen] = L;
      h[kRecWordFlags] = flags;
      h[kRecWordReserved] = 0u;
      unsigned long long* st = reinterpret_cast<unsigned long long*>(p);
      st[0] = open;
      st[1] = (flags & kRecRxKnown) ? rx : 0ull;
    }
    p += kRecStampBytes;
    copy16(reinterpret_cast<uint4*>(p), reinterpret_cast<const uint4*>(a.counters + s), kRecCounterBytes / 16);
    p += kRecCounterBytes;
    copy_nodes<true>(a.arena + (size_t)s * a.stride_nodes + a.max_nodes - L, reinterpret_cast<uint2*>(p), L);
  }
}

__global__ void __launch_bounds__(MT) stream_unpack_kernel(MigrateArgs a) {
  for (uint32_t i = blockIdx.x; i < a.n; i += gridDim.x) {
    const uint32_t s = a.streams[i];
    uint8_t* rec = a.records + a.offsets[i];
    const uint32_t* h = reinterpret_cast<const uint32_t*>(rec);
    const uint32_t L = h[kRecWordOpen], flags = h[kRecWordFlags];
    const bool framer = h[kRecWordKind] && h[kRecWordType] != 0x81u;
    uint8_t* p = rec + kRecHeaderBytes;
    copy16(reinterpret_cast<uint4*>(a.held + (size_t)s * kHeldWords), reinterpret_cast<const uint4*>(p), kRecHeldBytes / 16);
    p += kRecHeldBytes;
    if (a.framer) {  // a 0x81 stream of a mixed session keeps a fresh framer record, as a reset leaves it
      uint4* f = reinterpret_cast<uint4*>(a.framer + (size_t)s * kFramerWords);
      for (uint32_t w = threadIdx.x; w < kRecFramerBytes / 16; w += MT)
        f[w] = framer ? reinterpret_cast<const uint4*>(p)[w] : make_uint4(0u, 0u, 0u, 0u);
    }
    if (framer) p += kRecFramerBytes;
    if (threadIdx.x == 0) {
      const unsigned long long* st = reinterpret_cast<const unsigned long long*>(p);
      a.open_ts[s] = (flags & kRecOpenKnown) ? st[0] : 0ull;
      a.held_rx[s] = (flags & kRecRxKnown) ? st[1] : kRxUnknown;
      a.carry_len[s] = L;
    }
    p += kRecStampBytes;
    copy16(reinterpret_cast<uint4*>(a.counters + s), reinterpret_cast<const uint4*>(p), kRecCounterBytes / 16);
    p += kRecCounterBytes;
    copy_nodes<false>(a.arena + (size_t)s * a.stride_nodes + a.max_nodes - L, reinterpret_cast<uint2*>(p), L);
  }
}

}  // namespace

cudaError_t launch_stream_pack(const MigrateArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  const int grid = (int)std::min<uint32_t>(a.n, (uint32_t)num_sms * 8u);
  stream_pack_kernel<<<grid, MT, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_stream_unpack(const MigrateArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n == 0) return cudaSuccess;
  const int grid = (int)std::min<uint32_t>(a.n, (uint32_t)num_sms * 8u);
  stream_unpack_kernel<<<grid, MT, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rpl
