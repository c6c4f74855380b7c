// frame.cu -- byte-level framing of raw capsule streams with the SDK's resynchronisation.
//
// The capsule unpackers of the SDK do not receive framed capsules: they hunt for the two sync nibbles byte by
// byte (reference src/sdk/src/dataunpacker/unpacker/handler_capsules.cpp:107-135 express, :324-353 ultra,
// :639-668 dense, :852-880 ultra-dense -- the same little machine four times, only the frame size differs):
//   waiting for byte 0:  high nibble 0xA -> byte 1;  anything else is skipped and `_is_previous_capsuledataRdy`
//                        is cleared
//   waiting for byte 1:  high nibble 0x5 -> collect; anything else (that byte is consumed, not looked at again)
//                        goes back to byte 0 and clears the flag as well
//   collecting:          bytes 2 .. size-1 are taken blindly; the frame is then checked (checksum) and decoded
// As a function of the stream this is a chain of jumps from one "waiting for byte 0" position to the next:
// +1, +2 or +frame size.  This kernel walks that chain and writes the frames it visits back to back
// ([capsules][frame size], the input format of decode_formats.cu); every stretch of skipped bytes
// becomes ONE all-zero capsule in the output.  The decoders report such a capsule as RPL_CAPSULE_BAD_FRAME and
// forget the capsule before it -- precisely the effect the skipped bytes have in the SDK -- so framing + decoding
// reproduces the SDK's node stream on damaged input (dropped, inserted, corrupted bytes), pinned against the
// SDK's own unpacker in tests/test_framing_vs_ref.py.
//
// One CTA per stream, tiles of 16 KB staged through shared memory.  A tile whose frames all sit where the chain
// expects them (the normal case) is recognised by one marker test per frame, in parallel, and copied as a block;
// only a tile with a broken marker is walked serially by one thread (a dependent shared-memory load per jump).
//
// STREAM: a byte session's instantiation (rpl_capsule_stream_push_bytes*).  The handlers keep their search across
// calls, so each stream's framer record (kFramer*, decode_args.h) carries the search position, the bytes of the
// unfinished frame and a skipped stretch not yet reported from one push to the next.  A push is framed as the held
// bytes followed by the push's bytes (the first tile is staged from both), so a frame spanning two pushes is completed
// as one spanning two tiles is, and the lost bit becomes the all-zero capsule in front of the next frame, in whichever
// push that comes.  The capsules of all pushes, concatenated, are those of the unsplit stream.  HQ (0x83) is framed
// here only: UnpackerHandler_HQNode::onData (handler_hqnode.cpp:95-172) skips any byte but 0xA5 while waiting, takes
// the 780 bytes after a 0xA5 blindly, and a skipped byte changes nothing in it (no all-zero capsule).  With receive
// times, each frame gets the time of the push chunk holding its last byte (when the handler completes it).
#include "decode_args.h"
#include "rpl_device.cuh"

namespace rpl {

namespace {

constexpr int FT = 256;
constexpr uint32_t kTileBytes = 16384;
constexpr uint32_t kMaxFrame = 176;
constexpr uint32_t kMaxEntries = 2 * (kTileBytes / 84) + 8;
constexpr uint32_t kDummy = 0xFFFFFFFFu;
constexpr uint32_t kHqFrame = 781;  // HQ capsule: 0xA5, then 780 bytes

template <bool STREAM>
struct FrameSmem {
  uint32_t words[(kTileBytes + (STREAM ? kHqFrame : kMaxFrame) + 8) / 4 + 2];
  uint32_t entry[kMaxEntries];  // tile offset of a frame, or kDummy
  uint32_t n_entries, new_pos, lost, done;
};

// LIST (a mixed byte session, STREAM only): CTA slot i serves stream list.streams[i] of the chunk, whose framed
// capsules start list.capsule_stride bytes apart
template <bool STREAM, bool LIST>
__device__ __forceinline__ void frame_capsules_body(FrameArgs a, FrameStreamArgs f, StreamList list) {
  static_assert(STREAM || !LIST, "stream lists are a byte session's");
  __shared__ FrameSmem<STREAM> sm;
  const uint32_t tid = threadIdx.x;
  const uint32_t cb = a.capsule_bytes;
  const bool hq = STREAM && cb == kHqFrame;
  uint8_t* sb = reinterpret_cast<uint8_t*>(sm.words);
  for (uint32_t i = blockIdx.x; i < a.n_streams; i += gridDim.x) {
    const uint32_t s = LIST ? list.streams[i] : i;
    // session: stream positions count from the first held byte; the push's byte i is position k + i
    uint32_t* rec = STREAM ? f.framer + (size_t)s * kFramerWords : nullptr;
    const uint32_t k = STREAM ? rec[kFramerPos] : 0u;
    const uint8_t* in = a.bytes + (size_t)s * a.stride_bytes;
    const uint32_t n = STREAM ? k + min(a.byte_counts[s], a.stride_bytes) : a.byte_counts[s];
    uint8_t* out = a.capsules_out + (LIST ? (size_t)s * list.capsule_stride : (size_t)s * a.stride_capsules * cb);
    const unsigned long long* rx_in = STREAM && f.chunk_rx_us ? f.chunk_rx_us + (size_t)s * f.stride_chunks : nullptr;
    unsigned long long* rx_out = STREAM ? f.capsule_rx_out + (size_t)s * a.stride_capsules : nullptr;
    uint32_t pos = 0, count = 0, tile = 0;
    uint32_t zeros = 0;  // STREAM, thread 0: all-zero capsules among the `count` emitted
    bool lost = STREAM ? rec[kFramerLost] != 0u : false, done = false;
    const uint8_t* t = sb;
    while (!done && pos < n) {
      // ---- stage [pos, pos + L) (word loads from the aligned-down address) -----------------------------
      const uint32_t L = min(kTileBytes + cb, n - pos);
      const uintptr_t addr = reinterpret_cast<uintptr_t>(in + pos - k);
      uint32_t sh = (uint32_t)(addr & 3u);
      const uint32_t* gw = reinterpret_cast<const uint32_t*>(addr - sh);
      const uint32_t nwords = (sh + L + 3u) >> 2;
      __syncthreads();  // the previous tile's readers are done
      if (STREAM && pos < k) {  // the push's first tile: the held bytes, then the push's
        const uint8_t* held = reinterpret_cast<const uint8_t*>(rec + kFramerBytes);
        for (uint32_t i = tid; i < L; i += FT) sb[i] = i < k ? held[i] : __ldg(in + (i - k));
        sh = 0;
      } else {
        for (uint32_t w = tid; w < nwords; w += FT) sm.words[w] = __ldg(gw + w);
      }
      __syncthreads();
      t = sb + sh;  // t[i] = stream byte pos + i
      tile = pos;
      // ---- fast path: every frame of the tile where the chain expects it --------------------------------
      const uint32_t K = min(kTileBytes / cb, L / cb);
      int ok = 1;
      for (uint32_t j = tid; j < K; j += FT)
        ok = ok && (hq ? t[j * cb] == 0xA5u : ((t[j * cb] >> 4) == 0xAu) && ((t[j * cb + 1] >> 4) == 0x5u));
      const int all_ok = __syncthreads_and(ok);
      if (K > 0 && all_ok) {
        const uint32_t first = count + (lost ? 1u : 0u);
        const uint32_t room = first < a.stride_capsules ? a.stride_capsules - first : 0u;
        const uint32_t kw = min(K, room);
        if (lost && count < a.stride_capsules)
          for (uint32_t i = tid; i < cb; i += FT) out[(size_t)count * cb + i] = 0;
        uint8_t* dst = out + (size_t)first * cb;
        const uint32_t bytes = kw * cb;
        if (sh == 0 && (reinterpret_cast<uintptr_t>(dst) & 3u) == 0 && (bytes & 3u) == 0) {
          uint32_t* d4 = reinterpret_cast<uint32_t*>(dst);
          for (uint32_t w = tid; w < (bytes >> 2); w += FT) d4[w] = sm.words[w];
        } else if (STREAM && (reinterpret_cast<uintptr_t>(dst) & 3u) == 0 && (bytes & 3u) == 0) {
          // a session's held bytes shift its stream off the word grid (sh != 0): whole words from two staged ones
          uint32_t* d4 = reinterpret_cast<uint32_t*>(dst);
          for (uint32_t w = tid; w < (bytes >> 2); w += FT) d4[w] = __funnelshift_r(sm.words[w], sm.words[w + 1], 8u * sh);
        } else {
          for (uint32_t i = tid; i < bytes; i += FT) dst[i] = t[i];
        }
        if (rx_in) {  // a frame's receive time: the chunk of its last byte (a placeholder takes the next frame's)
          for (uint32_t j = tid; j < kw; j += FT) rx_out[first + j] = rx_in[(pos + (j + 1) * cb - 1 - k) / f.chunk_bytes];
          if (lost && count < a.stride_capsules && tid == 0) rx_out[count] = rx_in[(pos + cb - 1 - k) / f.chunk_bytes];
        }
        if (STREAM && lost) ++zeros;
        count = first + K;
        lost = false;
        pos += K * cb;
        continue;
      }
      // ---- a marker is broken (or the stream ends inside this tile): walk the chain ------------------------
      if (tid == 0) {
        uint32_t q = 0, ne = 0, l = lost ? 1u : 0u, fin = 0;
        const uint32_t lim = min(kTileBytes, L);
        while (q < lim) {
          if (hq ? t[q] != 0xA5u : (t[q] >> 4) != 0xAu) {
            if (!hq) l = 1;
            q += 1;
            continue;
          }
          if (!hq) {
            if (q + 1 >= L) {  // the stream ends on a lone first marker byte
              fin = 1;
              break;
            }
            if ((t[q + 1] >> 4) != 0x5u) {
              l = 1;
              q += 2;
              continue;
            }
          }
          if (q + cb > L) {  // unfinished frame at the end of the stream
            fin = 1;
            break;
          }
          if (l) {
            sm.entry[ne++] = kDummy;
            l = 0;
            if (STREAM) ++zeros;
          }
          sm.entry[ne++] = q;
          q += cb;
        }
        // L < tile + frame means the stream ends in this tile: whatever is left over is an unfinished frame
        if (!fin && pos + q >= n) fin = 1;
        sm.n_entries = ne;
        sm.new_pos = pos + min(q, L);
        sm.lost = l;
        sm.done = fin;
      }
      __syncthreads();
      const uint32_t ne = sm.n_entries;
      for (uint32_t e = 0; e < ne; ++e) {
        if (count + e >= a.stride_capsules) break;
        const uint32_t off = sm.entry[e];
        uint8_t* dst = out + (size_t)(count + e) * cb;
        if (off == kDummy) {
          for (uint32_t i = tid; i < cb; i += FT) dst[i] = 0;
        } else {
          for (uint32_t i = tid; i < cb; i += FT) dst[i] = t[off + i];
        }
        if (rx_in && tid == 0)
          rx_out[count + e] = rx_in[((off == kDummy ? sm.entry[e + 1] : off) + pos + cb - 1 - k) / f.chunk_bytes];
      }
      count += ne;
      pos = sm.new_pos;
      lost = sm.lost != 0;
      done = sm.done != 0;
    }
    if constexpr (STREAM) {
      // the unfinished frame at the end is still staged: hold it, and the lost bit, for the next push
      __syncthreads();  // every thread has read the record (a push that completes nothing stages no tile)
      const uint32_t left = n - min(pos, n);
      uint8_t* held = reinterpret_cast<uint8_t*>(rec + kFramerBytes);
      for (uint32_t i = tid; i < left; i += FT) held[i] = t[pos - tile + i];
      if (tid == 0) {
        rec[kFramerPos] = left;
        rec[kFramerLost] = lost ? 1u : 0u;
        // every byte entering (held + pushed) is in a completed frame, held for the next push, or skipped
        const uint32_t frames = count - zeros;
        StreamCounters& sc = f.counters[s];
        sc.bytes_in += n - k;
        sc.frames += frames;
        sc.skipped_bytes += n - left - frames * cb;
      }
    }
    if (tid == 0) {
      a.capsule_counts_out[s] = count;  // > stride_capsules: the output overflowed (frames past it were dropped)
      if (a.bytes_left_out) a.bytes_left_out[s] = n - min(pos, n);
    }
    __syncthreads();
  }
}

template <bool STREAM>
__global__ void __launch_bounds__(FT) frame_capsules_kernel(FrameArgs a, FrameStreamArgs f) {
  frame_capsules_body<STREAM, false>(a, f, StreamList{});
}

__global__ void __launch_bounds__(FT) frame_capsules_list_kernel(FrameArgs a, FrameStreamArgs f, StreamList l) {
  frame_capsules_body<true, true>(a, f, l);
}

}  // namespace

cudaError_t launch_frame_capsules(const FrameArgs& a, int grid, cudaStream_t stream) {
  if (a.n_streams == 0) return cudaSuccess;
  frame_capsules_kernel<false><<<grid, FT, 0, stream>>>(a, FrameStreamArgs{});
  return cudaGetLastError();
}

cudaError_t launch_frame_capsules_stream(const FrameArgs& a, const FrameStreamArgs& f, int grid, cudaStream_t stream,
                                         const StreamList* list) {
  if (a.n_streams == 0) return cudaSuccess;
  if (list)
    frame_capsules_list_kernel<<<grid, FT, 0, stream>>>(a, f, *list);
  else
    frame_capsules_kernel<true><<<grid, FT, 0, stream>>>(a, f);
  return cudaGetLastError();
}

}  // namespace rpl
