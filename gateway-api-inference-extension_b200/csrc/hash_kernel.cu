// hash_kernel.cu — hashPrompt for a batch (approximateprefix/hashing.go:34-98) on sm_90a.
#include "device_common.cuh"
#include "xxh64.cuh"

namespace eppscore {

// ---------------------------------------------------------------------------------------------
// hashPrompt for a batch, as two kernels:
//   hash_bodies_kernel  one lane per (request, block): the stripe state ("body") of a block depends on the
//                       block's own bytes only (the chain value is just the LAST 8 bytes of each link), so
//                       this is an embarrassingly parallel stream over the prompts — no barriers, high
//                       occupancy; it writes the 8-byte body states into the hashes buffer;
//   hash_chain_kernel   one warp per 32 requests: loads their body states (coalesced) into shared memory,
//                       runs the serial chain (one 8-byte tail round + avalanche per link, lane = request),
//                       and stores the hashes back in place (coalesced); also the trailing partial block
//                       (hashing.go:89-95), the generic path and n_hashes.
// A single fused kernel (r1_v2) stalled 3 of 4 warps at the barrier around the serial chain
// (profiles/r1_v4_ncu_hash_pick_prepare.txt: barrier + long-scoreboard stalls, IPC 1.9).
// Requests whose block size is not a multiple of 32 or whose start is not 16-byte aligned are hashed
// entirely by the chain kernel's generic serial path.
// ---------------------------------------------------------------------------------------------
constexpr int kHashWarps = 4;

template <int BC>  // BC = 64: the default 16-token block, fully unrolled; BC = 0: any multiple of 32
__device__ __forceinline__ uint64_t block_body_state(const uint8_t* p, int bc) {
  uint64_t v1 = XP1 + XP2, v2 = XP2, v3 = 0, v4 = 0 - XP1;
  if (BC == 64) {
    uint4 d[4];
#pragma unroll
    for (int k = 0; k < 4; k++) d[k] = ldg16(p + 16 * k);
#pragma unroll
    for (int st = 0; st < 2; st++) {
      const uint4 x = d[2 * st], y = d[2 * st + 1];
      v1 = xround(v1, ((uint64_t)x.y << 32) | x.x);
      v2 = xround(v2, ((uint64_t)x.w << 32) | x.z);
      v3 = xround(v3, ((uint64_t)y.y << 32) | y.x);
      v4 = xround(v4, ((uint64_t)y.w << 32) | y.z);
    }
    return xfinish_lanes(v1, v2, v3, v4) + (uint64_t)(64 + 8);
  }
  for (int s = 0; s < bc; s += 32) {
    const uint4 x = ldg16(p + s), y = ldg16(p + s + 16);
    v1 = xround(v1, ((uint64_t)x.y << 32) | x.x);
    v2 = xround(v2, ((uint64_t)x.w << 32) | x.z);
    v3 = xround(v3, ((uint64_t)y.y << 32) | y.x);
    v4 = xround(v4, ((uint64_t)y.w << 32) | y.z);
  }
  return xfinish_lanes(v1, v2, v3, v4) + (uint64_t)(bc + 8);
}


struct ReqDesc {
  const uint8_t* p;
  uint64_t seed;
  int nfull, rem;
  bool fast;
};
__device__ __forceinline__ ReqDesc load_desc(const HashArgs& a, int r, int bc) {
  ReqDesc d;
  const int64_t o = a.off[r];
  int64_t len = a.len ? (int64_t)a.len[r] : a.off[r + 1] - o;
  d.p = a.bytes + o;
  d.seed = a.seed ? a.seed[r] : 0ULL;
  d.nfull = 0;
  d.rem = 0;
  if (bc > 0 && len >= bc) {                             // hashing.go:51-60
    const int64_t cap = (int64_t)bc * (int64_t)a.max_blocks;
    if (len > cap) len = cap;                            // :62-65
    d.nfull = (int)(len / bc);
    d.rem = (int)(len - (int64_t)d.nfull * bc);
  }
  d.fast = bc > 0 && (bc & 31) == 0 && ((reinterpret_cast<uintptr_t>(d.p) & 15) == 0);
  return d;
}

constexpr int kBodyWarps = 8;

template <int BC>
__global__ void __launch_bounds__(kBodyWarps * 32) hash_bodies_kernel(HashArgs a) {
  pdl_launch_dependents();  // the chain kernel may be brought up while this grid drains
  const int lane = threadIdx.x & 31;
  const int bc = BC ? BC : a.block_chars;
  const int gw = blockIdx.x * kBodyWarps + (threadIdx.x >> 5), nw = gridDim.x * kBodyWarps;
  for (int r = gw; r < a.R; r += nw) {                   // one warp per request, 32 blocks per pass
    const ReqDesc d = load_desc(a, r, bc);               // same address in every lane: one broadcast load each
    if (!d.fast) continue;
    for (int b = lane; b < d.nfull; b += 32)
      a.hashes[(size_t)r * a.stride + b] = block_body_state<BC>(d.p + (size_t)b * bc, bc);
  }
}

// hash_bodies_pipe_kernel (EXPERIMENT, stage-mask bit 32; not the default): the same work as hash_bodies_kernel (lane = block
// of one request, a warp per request) as a PERSISTENT grid with the loads software-pipelined: while a warp digests request k,
// the 64 bytes per lane of its request k+1 are in flight and the descriptor of request k+2 is being fetched.  The idea was
// to hide the two dependent memory latencies (descriptor, then bytes) the one-shot form pays per warp; 64 registers per
// thread instead of 30 halve the resident warps (32 vs 64 per SM), against which the hardware's own overlap of many
// short-lived warps hides latency too.  Compare the two with tools/prof_step.py split.
template <int BC>
__global__ void __launch_bounds__(kBodyWarps * 32, 3) hash_bodies_pipe_kernel(HashArgs a) {
  pdl_launch_dependents();  // the chain kernel may be brought up while this grid drains
  const int lane = threadIdx.x & 31;
  const int bc = BC ? BC : a.block_chars;
  const int gw = blockIdx.x * kBodyWarps + (threadIdx.x >> 5), nw = gridDim.x * kBodyWarps;
  if (BC != 64) {  // other block sizes: not pipelined
    for (int r = gw; r < a.R; r += nw) {
      const ReqDesc d = load_desc(a, r, bc);
      if (!d.fast) continue;
      for (int b = lane; b < d.nfull; b += 32) a.hashes[(size_t)r * a.stride + b] = block_body_state<BC>(d.p + (size_t)b * bc, bc);
    }
    return;
  }
  // descriptors travel as RAW loaded values (start, end) and are only interpreted one iteration later, so that nothing
  // waits for them: {p, nfull, fast} of request k+1 are derived at the top of iteration k
  struct Raw {
    int64_t o, e;
  };
  auto load_raw = [&](int r) {
    Raw w;
    w.o = a.off[r];
    w.e = a.len ? w.o + (int64_t)a.len[r] : a.off[r + 1];
    return w;
  };
  auto derive = [&](const Raw& w, const uint8_t*& p, int& nfull) {  // load_desc without the seed; nfull = 0 unless fast
    int64_t len = w.e - w.o;
    p = a.bytes + w.o;
    nfull = 0;
    if (len >= 64) {
      const int64_t cap = 64LL * (int64_t)a.max_blocks;
      if (len > cap) len = cap;
      nfull = (int)(len >> 6);
    }
    if ((reinterpret_cast<uintptr_t>(p) & 15) != 0) nfull = 0;
  };
  int r = gw;
  if (r >= a.R) return;
  const uint8_t* p;
  int nfull;
  derive(load_raw(r), p, nfull);
  Raw raw_n = {0, 0};
  if (r + nw < a.R) raw_n = load_raw(r + nw);
  uint4 cur[4];
  bool on = lane < nfull;
#pragma unroll
  for (int k = 0; k < 4; k++) cur[k] = on ? ldg16(p + (size_t)lane * 64 + 16 * k) : make_uint4(0, 0, 0, 0);
  for (;;) {
    const int rn = r + nw, rnn = rn + nw;
    const bool have_n = rn < a.R;
    // the next request's bytes (its descriptor arrived during the previous digest), then the descriptor after that
    const uint8_t* pn = p;
    int nfull_n = 0;
    if (have_n) derive(raw_n, pn, nfull_n);
    uint4 nxt[4];
    const bool on_n = lane < nfull_n;
#pragma unroll
    for (int k = 0; k < 4; k++) nxt[k] = on_n ? ldg16(pn + (size_t)lane * 64 + 16 * k) : make_uint4(0, 0, 0, 0);
    if (rnn < a.R) raw_n = load_raw(rnn);
    if (on) {
      uint64_t v1 = XP1 + XP2, v2 = XP2, v3 = 0, v4 = 0 - XP1;
#pragma unroll
      for (int st = 0; st < 2; st++) {
        const uint4 x = cur[2 * st], y = cur[2 * st + 1];
        v1 = xround(v1, ((uint64_t)x.y << 32) | x.x);
        v2 = xround(v2, ((uint64_t)x.w << 32) | x.z);
        v3 = xround(v3, ((uint64_t)y.y << 32) | y.x);
        v4 = xround(v4, ((uint64_t)y.w << 32) | y.z);
      }
      a.hashes[(size_t)r * a.stride + lane] = xfinish_lanes(v1, v2, v3, v4) + (uint64_t)(64 + 8);
    }
    // more than 32 full blocks (max_blocks > 32): the rest of this request, not pipelined
    for (int b = lane + 32; b < nfull; b += 32) a.hashes[(size_t)r * a.stride + b] = block_body_state<64>(p + (size_t)b * 64, 64);
    if (!have_n) break;
    r = rn;
    p = pn;
    nfull = nfull_n;
    on = on_n;
#pragma unroll
    for (int k = 0; k < 4; k++) cur[k] = nxt[k];
  }
}

// One CTA (4 warps) per tile of 64 requests: all warps move the tile in and out (16 requests each, loads
// batched), warps 0 and 1 run the 64 serial chains (lane = request).  The kernel is latency bound (each
// link is ~35 dependent integer instructions), so the point is to keep many independent chains in flight
// per SM while keeping each tile's critical path short.
constexpr int kChainWarps = 2;                  // warps that run chains
constexpr int kTileReq = 32 * kChainWarps;      // requests per tile
constexpr int kMoveReq = kTileReq / kHashWarps; // requests each warp moves

__global__ void __launch_bounds__(kHashWarps * 32) hash_chain_kernel(HashArgs a) {
  pdl_wait();               // the body states come from the previous kernel of the stream
  pdl_launch_dependents();
  __shared__ uint64_t body[kTileReq][33];
  __shared__ int s_nfull[kTileReq], s_fast[kTileReq], s_maxfull[kChainWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bc = a.block_chars;
  const int ntiles = (a.R + kTileReq - 1) / kTileReq;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int base = tile * kTileReq;
    const int r = base + warp * 32 + lane;  // meaningful for the chain warps only
    ReqDesc d;
    d.p = nullptr;
    d.seed = 0;
    d.nfull = 0;
    d.rem = 0;
    d.fast = false;
    if (warp < kChainWarps) {
      if (r < a.R) d = load_desc(a, r, bc);
      int maxfull = d.nfull;
#pragma unroll
      for (int o = 16; o; o >>= 1) maxfull = max(maxfull, __shfl_xor_sync(0xffffffffu, maxfull, o));
      s_nfull[warp * 32 + lane] = d.nfull;
      s_fast[warp * 32 + lane] = d.fast ? 1 : 0;
      if (lane == 0) s_maxfull[warp] = maxfull;
    }
    __syncthreads();
    uint64_t prev = d.seed;
    int maxfull = 0;
#pragma unroll
    for (int w = 0; w < kChainWarps; w++) maxfull = max(maxfull, s_maxfull[w]);
    for (int c0 = 0; c0 < maxfull; c0 += 32) {
      // body states in (coalesced: lanes = blocks of one request); this warp's requests, 8 loads in flight
#pragma unroll
      for (int u0 = 0; u0 < kMoveReq; u0 += 8) {
        uint64_t v[8];
        bool on[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const int q = warp + (u0 + u) * kHashWarps, b = c0 + lane;
          on[u] = s_fast[q] && b < s_nfull[q];
          v[u] = on[u] ? a.hashes[(size_t)(base + q) * a.stride + b] : 0ULL;
        }
#pragma unroll
        for (int u = 0; u < 8; u++)
          if (on[u]) body[warp + (u0 + u) * kHashWarps][lane] = v[u];
      }
      __syncthreads();
      if (warp < kChainWarps) {  // the chain (lanes = requests)
        uint64_t(*mine)[33] = body + warp * 32;
        const int nb = min(32, d.nfull - c0);
        for (int i = 0; i < nb; i++) {
          if (d.fast)
            prev = xchain_aligned(mine[lane][i], prev);
          else
            prev = xxh64_link<false>(d.p + (size_t)(c0 + i) * bc, (uint32_t)bc, prev);  // hashing.go:80-87
          mine[lane][i] = prev;
        }
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < kMoveReq; u++) {  // hashes out (coalesced)
        const int q = warp + u * kHashWarps, b = c0 + lane;
        if (base + q < a.R && b < s_nfull[q]) a.hashes[(size_t)(base + q) * a.stride + b] = body[q][lane];
      }
      __syncthreads();
    }
    if (warp < kChainWarps && r < a.R) {
      if (d.rem > 0) {                                   // trailing partial block, hashing.go:89-95
        const uint8_t* t = d.p + (size_t)d.nfull * bc;
        const uint64_t h = ((reinterpret_cast<uintptr_t>(t) & 7) == 0) ? xxh64_link<true>(t, (uint32_t)d.rem, prev)
                                                                        : xxh64_link<false>(t, (uint32_t)d.rem, prev);
        a.hashes[(size_t)r * a.stride + d.nfull] = h;
      }
      a.n_hashes[r] = (uint16_t)(d.nfull + (d.rem > 0 ? 1 : 0));
    }
    __syncthreads();  // the tile descriptors are rewritten by the next tile
  }
}

// out-of-line slow paths (generic block sizes / unaligned prompts / the trailing partial block): keeping them out of the
// hot loops holds the fused kernel's register count down
// XXH64(data[0..n) || LE64(prev)) written for FEW REGISTERS (byte reads, no unrolling): the slow paths are rare, and a
// callee's register count is the kernel's register count.
static __device__ __noinline__ uint64_t link_slow(const uint8_t* d, uint32_t n, uint64_t prev) {
  const uint32_t len = n + 8;
  auto rd = [&](uint32_t off, uint32_t nbytes) {  // little-endian read of nbytes <= 8 bytes of the virtual message
    uint64_t v = 0;
#pragma unroll 1
    for (uint32_t k = 0; k < nbytes; k++) {
      const uint32_t i = off + k;
      const uint64_t b = i < n ? (uint64_t)d[i] : ((prev >> (8 * (i - n))) & 0xFFull);
      v |= b << (8 * k);
    }
    return v;
  };
  uint32_t p = 0;
  uint64_t h;
  if (len >= 32) {
    uint64_t v1 = XP1 + XP2, v2 = XP2, v3 = 0, v4 = 0 - XP1;
#pragma unroll 1
    do {
      v1 = xround(v1, rd(p, 8));
      v2 = xround(v2, rd(p + 8, 8));
      v3 = xround(v3, rd(p + 16, 8));
      v4 = xround(v4, rd(p + 24, 8));
      p += 32;
    } while (p + 32 <= len);
    h = xfinish_lanes(v1, v2, v3, v4);
  } else {
    h = XP5;
  }
  h += (uint64_t)len;
#pragma unroll 1
  while (p + 8 <= len) {
    h ^= xround(0, rd(p, 8));
    h = xrotl(h, 27) * XP1 + XP4;
    p += 8;
  }
  if (p + 4 <= len) {
    h ^= rd(p, 4) * XP1;
    h = xrotl(h, 23) * XP2 + XP3;
    p += 4;
  }
#pragma unroll 1
  while (p < len) {
    h ^= rd(p, 1) * XP5;
    h = xrotl(h, 11) * XP1;
    p++;
  }
  return xavalanche(h);
}
// the stripe state of one 64-byte block whose bytes are already in registers
__device__ __forceinline__ uint64_t body_state_64(const uint4 (&d)[4]) {
  uint64_t v1 = XP1 + XP2, v2 = XP2, v3 = 0, v4 = 0 - XP1;
#pragma unroll
  for (int st = 0; st < 2; st++) {
    const uint4 x = d[2 * st], y = d[2 * st + 1];
    v1 = xround(v1, ((uint64_t)x.y << 32) | x.x);
    v2 = xround(v2, ((uint64_t)x.w << 32) | x.z);
    v3 = xround(v3, ((uint64_t)y.y << 32) | y.x);
    v4 = xround(v4, ((uint64_t)y.w << 32) | y.z);
  }
  return xfinish_lanes(v1, v2, v3, v4) + (uint64_t)(64 + 8);
}

// ---------------------------------------------------------------------------------------------
// hash_fused_kernel: both stages in ONE kernel, warp-specialised.  A CTA owns tiles of 32 requests; seven BODY warps
// stream the prompts (lane = block, the stripe states go to a shared-memory buffer [request][block]), the CHAIN warp
// (lane = request) turns a buffer of body states into chained hashes in place, and the body warps write a finished
// buffer out (coalesced, 256 bytes per request row) when they get it back.  Two buffers ping-pong through named barriers
// (FULL: bodies -> chain, EMPTY: chain -> bodies), so the serial chain of chunk q overlaps the HBM stream of chunk q+1:
// the 8-byte body states never travel through HBM and the second launch is gone (r1: 28.9 us + 12.4 us as two kernels).
// ---------------------------------------------------------------------------------------------
constexpr int kFusedWarps = 8;                   // 7 body warps + 1 chain warp
constexpr int kFusedBody = kFusedWarps - 1;
constexpr int kFusedTile = 32;                   // requests per tile (one chain lane each)

__device__ __forceinline__ void nbar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void nbar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

template <int BC>
__global__ void __launch_bounds__(kFusedWarps * 32, 5) hash_fused_kernel(HashArgs a) {
  __shared__ uint64_t buf[2][kFusedTile][33];
  __shared__ int s_nfull[2][kFusedTile];
  __shared__ int s_base[2], s_c0[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bc = BC ? BC : a.block_chars;
  const int ntiles = (a.R + kFusedTile - 1) / kFusedTile;
  constexpr int FULL0 = 1, EMPTY0 = 3, NT = kFusedWarps * 32;
  int q = 0;  // chunk counter of this CTA: identical in every warp (same tile / chunk loop bounds)

  if (warp < kFusedBody) {
    // ---------------- body warps ----------------
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int base = tile * kFusedTile;
      // descriptors of this tile's requests: lane = request (every body warp computes the same 32 descriptors)
      ReqDesc d;
      d.p = nullptr;
      d.seed = 0;
      d.nfull = 0;
      d.rem = 0;
      d.fast = false;
      if (base + lane < a.R) d = load_desc(a, base + lane, bc);
      int maxfull = d.nfull;
#pragma unroll
      for (int o = 16; o; o >>= 1) maxfull = max(maxfull, __shfl_xor_sync(0xffffffffu, maxfull, o));
      int nchunks = (maxfull + 31) >> 5;
      if (nchunks < 1) nchunks = 1;  // the chain warp still runs once per tile (partial blocks, n_hashes)
      for (int ch = 0; ch < nchunks; ch++, q++) {
        const int b = q & 1, c0 = ch * 32;
        if (q >= 2) {
          nbar_sync(EMPTY0 + b, NT);  // the chain warp is done with the chunk that used this buffer
          // write that chunk's hashes out: 32 consecutive blocks of a request per warp store
          const int ob = s_base[b], oc = s_c0[b];
          for (int rq = warp; rq < kFusedTile; rq += kFusedBody) {
            const int blk = oc + lane;
            if (ob + rq < a.R && blk < s_nfull[b][rq]) a.hashes[(size_t)(ob + rq) * a.stride + blk] = buf[b][rq][lane];
          }
          nbar_sync(7, kFusedBody * 32);  // every body warp has read the old descriptors before they are replaced
        }
        if (warp == 0) {
          s_nfull[b][lane] = d.fast ? d.nfull : 0;  // (rows of the generic path are written by hash_slow_kernel)
          if (lane == 0) {
            s_base[b] = base;
            s_c0[b] = c0;
          }
        }
        // body states of blocks [c0, c0+32) of this warp's requests
        const int blk = c0 + lane;
        for (int rq = warp; rq < kFusedTile; rq += kFusedBody) {
          const int nf = __shfl_sync(0xffffffffu, d.nfull, rq);
          const int fs = __shfl_sync(0xffffffffu, d.fast ? 1 : 0, rq);
          const unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)reinterpret_cast<uintptr_t>(d.p), rq);
          if (fs && blk < nf)
            buf[b][rq][lane] = block_body_state<BC>(reinterpret_cast<const uint8_t*>((uintptr_t)pp) + (size_t)blk * bc, bc);
        }
        __threadfence_block();
        nbar_arrive(FULL0 + b, NT);
      }
    }
    // drain: the last (up to two) chunks still sit in the buffers
    for (int k = (q >= 2 ? q - 2 : 0); k < q; k++) {
      const int b = k & 1;
      nbar_sync(EMPTY0 + b, NT);
      const int ob = s_base[b], oc = s_c0[b];
      for (int rq = warp; rq < kFusedTile; rq += kFusedBody) {
        const int blk = oc + lane;
        if (ob + rq < a.R && blk < s_nfull[b][rq]) a.hashes[(size_t)(ob + rq) * a.stride + blk] = buf[b][rq][lane];
      }
    }
  } else {
    // ---------------- chain warp: lane = request ----------------
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int base = tile * kFusedTile;
      const int r = base + lane;
      ReqDesc d;
      d.p = nullptr;
      d.seed = 0;
      d.nfull = 0;
      d.rem = 0;
      d.fast = false;
      if (r < a.R) d = load_desc(a, r, bc);
      int maxfull = d.nfull;
#pragma unroll
      for (int o = 16; o; o >>= 1) maxfull = max(maxfull, __shfl_xor_sync(0xffffffffu, maxfull, o));
      int nchunks = (maxfull + 31) >> 5;
      if (nchunks < 1) nchunks = 1;
      uint64_t prev = d.seed;
      for (int ch = 0; ch < nchunks; ch++, q++) {
        const int b = q & 1, c0 = ch * 32;
        nbar_sync(FULL0 + b, NT);
        const int nb = min(32, d.nfull - c0);
        if (d.fast) {
          for (int i = 0; i < nb; i++) {
            prev = xchain_aligned(buf[b][lane][i], prev);
            buf[b][lane][i] = prev;
          }
        }
        // (requests of the generic path and trailing partial blocks are finished by hash_slow_kernel)
        if (ch == nchunks - 1 && r < a.R) a.n_hashes[r] = (uint16_t)(d.nfull + (d.rem > 0 ? 1 : 0));
        __threadfence_block();
        nbar_arrive(EMPTY0 + b, NT);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// hash_warp_kernel: both stages in one kernel WITHOUT any CTA-level synchronisation.  A WARP owns a tile of 32 requests:
//   A  lane = block: the stripe states of 32 blocks of one request after the other go to the warp's shared-memory tile
//      [request][block]; the next TWO requests' 64 bytes per lane are in flight while the current block is digested
//      (one ahead left the warps latency bound: 68 us for the plain form, 78 us with the probe, against 68 us now, H100);
//   B  lane = request: the serial chain over the tile's rows, in place (32 chains in flight per warp);
//   C  lane = block: the finished hashes leave the tile, 256 contiguous bytes per request.
// Only __syncwarp between the phases: no warp ever waits for another one, the chain phases of some warps overlap the HBM
// stream of the others, the 8-byte body states never travel through HBM and the second launch is gone.
// PROBE (schedule_device, when pick_sparse_kernel follows): between B and C each lane also runs indexer.Get over its request's
// new hashes while the tile holds them, exactly as pick_sparse_kernel would, and a request whose matched blocks all carry its
// first hit's inline set is RESOLVED: its ProbeRec holds the count and the set, and its row of hashes is not written (nothing
// reads it).  The index is not snapshot data, so this kernel still runs concurrently with a snapshot preparation.
// With PROBE, A, B and PROBE run per chunk of kProbeChunk blocks of every request, and A skips the requests whose walk ended
// at a miss while still resolvable: nothing reads their hashes past that miss, so their bytes are never loaded.  Every other
// request (one that meets a set change or a bitset row, a trailing partial block, the generic path) streams its whole row.
// ---------------------------------------------------------------------------------------------
constexpr int kWarpTileWarps = 8;
constexpr int kProbeU = 4;     // PROBE: hashes probed per lane at a time (both halves of each slot in flight: 128 registers)
constexpr int kProbeChunk = 4; // PROBE: blocks per request streamed, chained and probed before the next chunk

template <int BC, bool PROBE>
__global__ void __launch_bounds__(kWarpTileWarps * 32, 2) hash_warp_kernel(HashArgs a) {
  // phase A's lanes: K blocks of G requests per step, K steps per chunk (the plain form: one request of 32 blocks per step)
  constexpr int K = PROBE ? kProbeChunk : 32, G = 32 / K;
  static_assert(K * G == 32 && K % kProbeU == 0, "a chunk is a whole number of probe rounds and divides a warp");
  extern __shared__ __align__(16) unsigned char hw_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane / K, kb = lane % K;  // phase A: this lane's request within a step, and its block within the chunk
  uint64_t(*tile)[33] = reinterpret_cast<uint64_t(*)[33]>(hw_smem) + (size_t)warp * 32;
  const int bc = BC ? BC : a.block_chars;
  const int ntiles = (a.R + 31) / 32;
  const TSlot* slots = nullptr;
  uint64_t slot_mask = 0;
  if (PROBE) {
    slots = a.table->slots;
    slot_mask = a.table->mask;
  }
  for (int t = blockIdx.x * kWarpTileWarps + warp; t < ntiles; t += gridDim.x * kWarpTileWarps) {
    const int base = t * 32, r = base + lane;
    ReqDesc d;
    d.p = nullptr;
    d.seed = 0;
    d.nfull = 0;
    d.rem = 0;
    d.fast = false;
    if (r < a.R) d = load_desc(a, r, bc);
    const int nf_mine = d.fast ? d.nfull : 0;      // rows of the generic path belong to hash_slow_kernel
    int maxfull = nf_mine;
#pragma unroll
    for (int o = 16; o; o >>= 1) maxfull = max(maxfull, __shfl_xor_sync(0xffffffffu, maxfull, o));
    uint64_t prev = d.seed;
    // PROBE state of this lane's request (pick_sparse's matchLongestPrefix without the table): p_ok = resolvable so far
    // (the fast path without a trailing partial block: the others need hash_slow_kernel's hashes), p_open = still walking
    bool p_ok = PROBE && r < a.R && d.fast && d.rem == 0;
    bool p_open = p_ok && nf_mine > 0;
    uint32_t p_n = 0, ref_raw = 0, ref_w = 0;
    uint4 ref_hi = make_uint4(0u, 0u, 0u, 0u);
    for (int c0 = 0; c0 < maxfull; c0 += 32) {
      for (int s0 = 0; s0 < 32; s0 += K) {  // chunks of this 32-block window (one in the plain form)
        const int cb = c0 + s0, blk = cb + kb;
        // blocks of this lane's request still hashed: a resolved request stops at its first miss (nothing reads its row)
        const int nf_str = (PROBE && p_ok && !p_open) ? 0 : nf_mine;
        if (PROBE && !__any_sync(0xffffffffu, cb < nf_str)) break;
        // ---- A: body states ----
        if (BC == 64) {
          uint4 buf[3][4];  // a ring: step st digested while st+1 and st+2 are in flight (indices compile-time after unrolling)
          bool on[3];
          auto fetch = [&](int st, uint4 (&dst)[4], bool& o) {
            const int rq = st * G + sub;
            const int nf = __shfl_sync(0xffffffffu, nf_str, rq);
            const unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)reinterpret_cast<uintptr_t>(d.p), rq);
            o = blk < nf;
            if (o) {
              const uint8_t* q = reinterpret_cast<const uint8_t*>((uintptr_t)pp) + (size_t)blk * 64;
#pragma unroll
              for (int k = 0; k < 4; k++) dst[k] = ldg16(q + 16 * k);
            }
          };
          fetch(0, buf[0], on[0]);
          fetch(1, buf[1], on[1]);
#pragma unroll (PROBE ? K : 1)  // the probing form: every step unrolled (no spill at 128 registers)
          for (int st0 = 0; st0 < K; st0 += 3) {
#pragma unroll
            for (int j = 0; j < 3; j++) {
              const int st = st0 + j;
              if (st < K) {
                const int ns = (j + 2) % 3;
                on[ns] = false;
                if (st + 2 < K) fetch(st + 2, buf[ns], on[ns]);
                if (on[j]) tile[st * G + sub][s0 + kb] = body_state_64(buf[j]);
              }
            }
          }
        } else {
#pragma unroll 1
          for (int st = 0; st < K; st++) {
            const int rq = st * G + sub;
            const int nf = __shfl_sync(0xffffffffu, nf_str, rq);
            const unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)reinterpret_cast<uintptr_t>(d.p), rq);
            if (blk < nf)
              tile[rq][s0 + kb] = block_body_state<BC>(reinterpret_cast<const uint8_t*>((uintptr_t)pp) + (size_t)blk * bc, bc);
          }
        }
        __syncwarp();
        // ---- B: the chain, lane = request ----
        const int nb = min(K, nf_str - cb);
        for (int i = 0; i < nb; i++) {
          prev = xchain_aligned(tile[lane][s0 + i], prev);
          tile[lane][s0 + i] = prev;
        }
        // ---- PROBE: indexer.Get on the lane's own row, kProbeU blocks at a time, up to the first miss ----
        if (PROBE) {
          for (int i0 = 0; __any_sync(0xffffffffu, p_open && i0 < nb); i0 += kProbeU) {
            // the round's loads first: both 16-byte halves of each home slot (one 32-byte sector), so that the walk below does
            // not wait on a dependent load per hit for the members 2..9; hashes and home indices are read back from the tile
            uint4 lo[kProbeU], hi[kProbeU];
#pragma unroll
            for (int u = 0; u < kProbeU; u++) {
              lo[u] = make_uint4(0u, 0u, kCntFree, 0u);
              hi[u] = make_uint4(0u, 0u, 0u, 0u);
              if (p_open && i0 + u < nb) {
                const uint4* sp = reinterpret_cast<const uint4*>(&slots[tile[lane][s0 + i0 + u] & slot_mask]);
                lo[u] = ldg16(sp);
                hi[u] = ldg16(sp + 1);
              }
            }
#pragma unroll
            for (int u = 0; u < kProbeU; u++) {
              if (!p_open || i0 + u >= nb) continue;
              const uint64_t h = tile[lane][s0 + i0 + u], home = h & slot_mask;
              uint64_t idx = home;
              if (!table_find(slots, slot_mask, h, idx, lo[u])) {
                p_open = false;                                   // the first miss ends the matched prefix
                continue;
              }
              // members 2..9 (the slot's second half) count only for inline sets of more than two, as pick_sparse_kernel reads
              // them; a key found past its home slot (a probe chain) has its second half loaded here
              uint4 h2 = make_uint4(0u, 0u, 0u, 0u);
              if (!(lo[u].z & kCntRow) && (lo[u].z & kCntMask) > 2u)
                h2 = idx == home ? hi[u] : ldg16(reinterpret_cast<const uint4*>(&slots[idx]) + 1);
              if (cb + i0 + u == 0) {
                ref_raw = lo[u].z;                                // the first hit: the reference set
                ref_w = lo[u].w;
                ref_hi = h2;
                p_n = 1;
                if (ref_raw & kCntRow) p_ok = p_open = false;     // a bitset row: pick_sparse's exception table
              } else if (lo[u].z != ref_raw || !same_inline_set(ref_w, ref_hi, lo[u].w, h2)) {
                p_ok = p_open = false;                            // a different set: pick_sparse's exception table
              } else {
                p_n++;
              }
            }
          }
          if (cb + K >= nf_mine) p_open = false;                  // the whole row matched
        }
        __syncwarp();
      }
      // a resolved row whose walk is over is not written: nothing reads it
      const int nf_out = (PROBE && p_ok && !p_open) ? 0 : nf_mine;
      const int blk = c0 + lane;
      // ---- C: hashes out ----
#pragma unroll 4
      for (int rq = 0; rq < 32; rq++) {
        const int nf = __shfl_sync(0xffffffffu, nf_out, rq);
        if (blk < nf) a.hashes[(size_t)(base + rq) * a.stride + blk] = tile[rq][lane];
      }
      __syncwarp();
    }
    if (PROBE) {
      const uint32_t res = __ballot_sync(0xffffffffu, p_ok);
      if (lane == 0 && res) atomicAdd(a.resolved, (unsigned long long)__popc(res));
    }
    if (r < a.R) {
      a.n_hashes[r] = (uint16_t)(d.nfull + (d.rem > 0 ? 1 : 0));
      if (PROBE) {
        uint4* q = reinterpret_cast<uint4*>(a.probe + r);
        q[0] = make_uint4(ref_raw, ref_w, p_ok ? p_n : kProbeUnresolved, 0u);
        q[1] = ref_hi;
      }
    }
  }
}

// hash_chain_warp_kernel: the serial stage with one WARP per tile of 32 requests and no CTA-level synchronisation: the
// whole batch's chains are in flight at once (2048 warps for 64K requests, a fraction of the machine's 9472 warp slots), so
// the kernel takes about one chain's latency plus one tile load and store.  Also finishes the generic path (block sizes that
// are not a multiple of 32, unaligned prompts), trailing partial blocks (hashing.go:89-95) and n_hashes.
constexpr int kChainWarpsPerCta = 4;
__global__ void __launch_bounds__(kChainWarpsPerCta * 32) hash_chain_warp_kernel(HashArgs a) {
  __shared__ uint64_t tiles[kChainWarpsPerCta][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t(*tile)[33] = tiles[warp];
  const int bc = a.block_chars;
  const int ntiles = (a.R + 31) / 32;
  for (int t = blockIdx.x * kChainWarpsPerCta + warp; t < ntiles; t += gridDim.x * kChainWarpsPerCta) {
    const int base = t * 32, r = base + lane;
    ReqDesc d;
    d.p = nullptr;
    d.seed = 0;
    d.nfull = 0;
    d.rem = 0;
    d.fast = false;
    if (r < a.R) d = load_desc(a, r, bc);
    const int nf_fast = d.fast ? d.nfull : 0;
    int maxfast = nf_fast;
#pragma unroll
    for (int o = 16; o; o >>= 1) maxfast = max(maxfast, __shfl_xor_sync(0xffffffffu, maxfast, o));
    uint64_t prev = d.seed;
    for (int c0 = 0; c0 < maxfast; c0 += 32) {
      const int blk = c0 + lane;
#pragma unroll 8
      for (int rq = 0; rq < 32; rq++) {  // body states in: 256 contiguous bytes per request
        const int nf = __shfl_sync(0xffffffffu, nf_fast, rq);
        if (blk < nf) tile[rq][lane] = a.hashes[(size_t)(base + rq) * a.stride + blk];
      }
      __syncwarp();
      const int nb = min(32, nf_fast - c0);
      for (int i = 0; i < nb; i++) {      // the chain: lane = request
        prev = xchain_aligned(tile[lane][i], prev);
        tile[lane][i] = prev;
      }
      __syncwarp();
#pragma unroll 8
      for (int rq = 0; rq < 32; rq++) {  // hashes out
        const int nf = __shfl_sync(0xffffffffu, nf_fast, rq);
        if (blk < nf) a.hashes[(size_t)(base + rq) * a.stride + blk] = tile[rq][lane];
      }
      __syncwarp();
    }
    if (r < a.R) {
      uint64_t* out = a.hashes + (size_t)r * a.stride;
      if (!d.fast)
        for (int i = 0; i < d.nfull; i++) out[i] = prev = link_slow(d.p + (size_t)i * bc, (uint32_t)bc, prev);  // hashing.go:79-87
      if (d.rem > 0) out[d.nfull] = link_slow(d.p + (size_t)d.nfull * bc, (uint32_t)d.rem, prev);               // :89-95
      a.n_hashes[r] = (uint16_t)(d.nfull + (d.rem > 0 ? 1 : 0));
    }
  }
}

// What the fused kernels leave: requests whose block size is not a multiple of 32 or whose start is not 16-byte aligned
// (hashed here entirely, hashing.go:79-87) and trailing partial blocks (hashing.go:89-95).  One thread per request; a
// request that needs neither returns after reading its descriptor.  Kept out of the fused kernel because a slow path's
// registers are the whole kernel's registers (68 -> 48 per thread, 3 -> 5 CTAs per SM).
__global__ void __launch_bounds__(256) hash_slow_kernel(HashArgs a) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  const int bc = a.block_chars;
  const ReqDesc d = load_desc(a, r, bc);
  if (d.fast && d.rem == 0) return;
  uint64_t* out = a.hashes + (size_t)r * a.stride;
  uint64_t prev = d.seed;
  if (d.fast) {
    if (d.nfull > 0) prev = out[d.nfull - 1];
  } else {
    for (int i = 0; i < d.nfull; i++) out[i] = prev = link_slow(d.p + (size_t)i * bc, (uint32_t)bc, prev);
  }
  if (d.rem > 0) out[d.nfull] = link_slow(d.p + (size_t)d.nfull * bc, (uint32_t)d.rem, prev);
}

constexpr int kDefaultStages = 27;

// the probing form exists for the default form (the warp-tile kernel) only
bool hash_probe_applies(const HashArgs& a) {
  return a.block_chars > 0 && (a.block_chars & 31) == 0 && (a.stage_mask == 0 || a.stage_mask == kDefaultStages);
}

template <int BC, bool PROBE>
static void launch_warp_tile(const HashArgs& a, int blocks, size_t smem, cudaStream_t s) {
  cudaFuncSetAttribute(hash_warp_kernel<BC, PROBE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  hash_warp_kernel<BC, PROBE><<<blocks, kWarpTileWarps * 32, smem, s>>>(a);
}

int launch_hash_prompts(const HashArgs& a, cudaStream_t s, int sm_count) {
  if (a.R <= 0) return 0;
  // default 27: the warp-tile fused kernel where the block size allows it (on H100 the step is 7 % faster than with the
  // two-kernel form), otherwise bodies + the CTA-tile chain kernel
  const int stages0 = a.stage_mask ? a.stage_mask : kDefaultStages;
  if ((stages0 & 8) && a.block_chars > 0 && (a.block_chars & 31) == 0) {  // the warp-tile fused kernel
    const int ntiles = (a.R + 31) / 32;
    int blocks = sm_count * 2;  // (the register budget of two requests in flight per warp: 2 CTAs per SM)
    const int need = (ntiles + kWarpTileWarps - 1) / kWarpTileWarps;
    if (blocks > need) blocks = need;
    const size_t smem = (size_t)kWarpTileWarps * 32 * 33 * 8;
    const bool probe = a.probe != nullptr;  // (set only where hash_probe_applies)
    if (a.block_chars == 64)
      probe ? launch_warp_tile<64, true>(a, blocks, smem, s) : launch_warp_tile<64, false>(a, blocks, smem, s);
    else
      probe ? launch_warp_tile<0, true>(a, blocks, smem, s) : launch_warp_tile<0, false>(a, blocks, smem, s);
    hash_slow_kernel<<<(a.R + 255) / 256, 256, 0, s>>>(a);
    return 2;
  }
  if ((stages0 & 4) && a.block_chars > 0 && (a.block_chars & 31) == 0) {  // the warp-specialised fused kernel (CTA tiles)
    const int ntiles = (a.R + kFusedTile - 1) / kFusedTile;
    int blocks = sm_count * 5;
    if (blocks > ntiles) blocks = ntiles;
    if (a.block_chars == 64)
      hash_fused_kernel<64><<<blocks, kFusedWarps * 32, 0, s>>>(a);
    else
      hash_fused_kernel<0><<<blocks, kFusedWarps * 32, 0, s>>>(a);
    hash_slow_kernel<<<(a.R + 255) / 256, 256, 0, s>>>(a);
    return 2;
  }
  int launched = 0;
  const int stages = (stages0 & 3) ? (stages0 & 3) : 3;
  if ((stages & 1) && a.block_chars > 0 && (a.block_chars & 31) == 0) {
    long long blocks = ((long long)a.R + kBodyWarps - 1) / kBodyWarps;
    if (!(stages0 & 32)) {  // a warp per request, a few waves of CTAs
      const long long cap = (long long)sm_count * 64;
      if (blocks > cap) blocks = cap;
      if (a.block_chars == 64)
        hash_bodies_kernel<64><<<(unsigned)blocks, kBodyWarps * 32, 0, s>>>(a);
      else
        hash_bodies_kernel<0><<<(unsigned)blocks, kBodyWarps * 32, 0, s>>>(a);
    } else {             // experimental: persistent, software-pipelined
      static int occ64 = 0, occ0 = 0;
      if (!occ64) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ64, hash_bodies_pipe_kernel<64>, kBodyWarps * 32, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ0, hash_bodies_pipe_kernel<0>, kBodyWarps * 32, 0);
        if (occ64 < 1) occ64 = 1;
        if (occ0 < 1) occ0 = 1;
      }
      const long long cap = (long long)sm_count * (a.block_chars == 64 ? occ64 : occ0);
      if (blocks > cap) blocks = cap;
      if (a.block_chars == 64)
        hash_bodies_pipe_kernel<64><<<(unsigned)blocks, kBodyWarps * 32, 0, s>>>(a);
      else
        hash_bodies_pipe_kernel<0><<<(unsigned)blocks, kBodyWarps * 32, 0, s>>>(a);
    }
    launched++;
  }
  if (!(stages & 2)) return launched;
  if (stages0 & 16) {  // the CTA-tile chain kernel of round 1 (diagnostics)
    const int ntiles = (a.R + kTileReq - 1) / kTileReq;
    launch_maybe_pdl(a.pdl != 0 && launched > 0, hash_chain_kernel, dim3(ntiles), dim3(kHashWarps * 32), 0, s, a);
  } else {
    const int ntiles = (a.R + 31) / 32;
    hash_chain_warp_kernel<<<(ntiles + kChainWarpsPerCta - 1) / kChainWarpsPerCta, kChainWarpsPerCta * 32, 0, s>>>(a);
  }
  return launched + 1;
}

}  // namespace eppscore
