// vgicp_sort.cuh -- stable LSD radix sort of (key, 32-bit value) pairs on the device, written for this library's two uses:
//   * stage 1: the points of a cloud in Morton order of their finest k-NN grid cell (one spatial sort serves every level of the
//     grid: a coarser cell is a contiguous run of the sorted array);
//   * stage 2: the points of the target grouped by voxel id with the original index ascending inside a voxel (LSD passes are
//     stable), so that the per-voxel sums run in point order -- the order the CPU checker uses -- without atomics.
// Shape (one-sweep style): ONE histogram kernel counts the digits of all passes, then one scatter kernel per pass.  A scatter
// tile (256 threads x 8 keys, warp w owns a contiguous run of 256 keys) ranks its keys with warp match-any, publishes its digit
// counts and obtains the counts of all preceding tiles by decoupled look-back (tiles take tickets, so a tile only ever waits for
// tiles that started before it).  Digits are kSortRadixBits = 9 bits wide: 27-bit Morton codes (17 k points) sort in 3 passes,
// 33..36-bit ones (1 M points) in 4, voxel ids below 2^18 in 2.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vgicp {

constexpr int kNumSMs = 132;  // H100 SXM: the caps on grid-stride / persistent grids below are multiples of it

constexpr int kSortRadixBits = 9;
constexpr int kSortBins = 1 << kSortRadixBits;
constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortItems = 8;                              // keys per thread
constexpr int kSortTile = kSortThreads * kSortItems;       // 2048 keys per tile
constexpr int kSortMaxPasses = 8;
constexpr unsigned kSortFlagAgg = 1u << 30, kSortFlagIncl = 2u << 30, kSortFlagMask = 3u << 30, kSortValMask = ~kSortFlagMask;

__host__ __device__ inline int sort_num_passes(int key_bits) { return (key_bits + kSortRadixBits - 1) / kSortRadixBits; }
__host__ __device__ inline int sort_num_tiles(int n) { return (n + kSortTile - 1) / kSortTile; }
// zero-initialised scratch: digit histograms of all passes, one ticket per pass, look-back state of all passes
inline size_t sort_scratch_bytes(int n, int passes) {
  return sizeof(unsigned) * ((size_t)kSortMaxPasses * kSortBins + 64 + (size_t)passes * sort_num_tiles(n) * kSortBins);
}

// digit counts of every pass in one sweep over the keys; lanes with equal digits elect one to add for all (the inputs are
// spatially coherent: most lanes of a warp share their high digits)
template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads) k_sort_hist(const KeyT* __restrict__ keys, int n, int passes, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kSortMaxPasses * kSortBins];
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads) sh[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n_round = (n + 31) & ~31;
  for (int i = blockIdx.x * kSortThreads + threadIdx.x; i < n_round; i += gridDim.x * kSortThreads) {  // warp-uniform trip count
    const bool valid = i < n;
    const KeyT key = valid ? keys[i] : (KeyT)0;
    for (int p = 0; p < passes; p++) {
      const unsigned d = valid ? (unsigned)((key >> (p * kSortRadixBits)) & (KeyT)(kSortBins - 1)) : (unsigned)kSortBins + lane;
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      if (valid && lane == __ffs(peers) - 1) atomicAdd(&sh[p * kSortBins + d], (unsigned)__popc(peers));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < passes * kSortBins; i += kSortThreads)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// histogram accumulation for kernels that produce the keys themselves (stage 1 computes the Morton codes and their digit counts
// in one pass): call with all 32 lanes, then flush after a __syncthreads
__device__ __forceinline__ void sort_hist_add(unsigned* sh, int passes, bool valid, unsigned long long key) {
  const int lane = threadIdx.x & 31;
  for (int p = 0; p < passes; p++) {
    const unsigned d = valid ? (unsigned)((key >> (p * kSortRadixBits)) & (unsigned long long)(kSortBins - 1)) : (unsigned)kSortBins + lane;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (valid && lane == __ffs(peers) - 1) atomicAdd(&sh[p * kSortBins + d], (unsigned)__popc(peers));
  }
}

// shared memory of one scatter tile
struct SortTileSmem {
  unsigned warp_cnt[kSortWarps][kSortBins];  // per warp: digit counts, then (after the scan) offsets of the warp inside the tile
  unsigned digit_base[kSortBins];            // output position of the tile's first key of each digit
  unsigned scan_tmp[kSortWarps];
  unsigned tile;
};

// One tile of one pass: stable scatter of (key, value) by digit `pass` of the key.  vin == nullptr: the values are the positions
// 0..n-1.  hist: the kSortBins global digit counts of this pass; state: [num_tiles][kSortBins], zero before the pass.  Tiles may
// be processed in any order in which a tile never starts before all lower-numbered tiles have started or finished (tickets, or a
// persistent grid walking the tiles round-robin): a tile only ever waits for lower-numbered ones.
// On the last pass the caller may pass a float4 array to be permuted along (out4[pos] = {in4[value].xyz, value as bits}).
// Called by all kSortThreads threads of the block; ends with the tile's stores issued (no trailing barrier).
template <typename KeyT>
__device__ __forceinline__ void sort_pass_tile(SortTileSmem& sm, unsigned tile, const KeyT* __restrict__ kin, const unsigned* __restrict__ vin, KeyT* __restrict__ kout,
                                               unsigned* __restrict__ vout, int n, int pass, const unsigned* __restrict__ hist, unsigned* state, const float4* __restrict__ in4,
                                               float4* __restrict__ out4) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const unsigned lt = (1u << lane) - 1u;
  __syncthreads();  // (the previous tile's shared memory is no longer read)
  for (int i = tid; i < kSortWarps * kSortBins; i += kSortThreads) (&sm.warp_cnt[0][0])[i] = 0;
  __syncthreads();
  const int shift = pass * kSortRadixBits;
  const long long base = (long long)tile * kSortTile + (long long)w * (32 * kSortItems);
  KeyT key[kSortItems];
  unsigned val[kSortItems], rank[kSortItems];
#pragma unroll
  for (int r = 0; r < kSortItems; r++) {
    const long long idx = base + r * 32 + lane;
    const bool valid = idx < n;
    key[r] = valid ? kin[idx] : (KeyT)0;
    val[r] = valid ? (vin ? vin[idx] : (unsigned)idx) : 0u;
    const unsigned d = valid ? (unsigned)((key[r] >> shift) & (KeyT)(kSortBins - 1)) : (unsigned)kSortBins + lane;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int leader = __ffs(peers) - 1;
    unsigned prev = 0;
    if (valid && lane == leader) {
      prev = sm.warp_cnt[w][d];
      sm.warp_cnt[w][d] = prev + (unsigned)__popc(peers);
    }
    prev = __shfl_sync(0xffffffffu, prev, leader);
    rank[r] = prev + (unsigned)__popc(peers & lt);  // keys of this warp's run with the same digit that come before this one
    __syncwarp();
  }
  __syncthreads();
  // exclusive scan of the global digit counts (where each digit's output range starts)
  constexpr int J = kSortBins / kSortThreads;
  unsigned gstart[J];
  {
    unsigned c[J], sum = 0;
#pragma unroll
    for (int j = 0; j < J; j++) {  // thread t owns digits t*J .. t*J+J-1 (contiguous)
      c[j] = *reinterpret_cast<const volatile unsigned*>(&hist[tid * J + j]);
      sum += c[j];
    }
    unsigned incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) sm.scan_tmp[w] = incl;
    __syncthreads();
    unsigned wbase = 0;
    for (int ww = 0; ww < w; ww++) wbase += sm.scan_tmp[ww];
    unsigned run = wbase + incl - sum;
#pragma unroll
    for (int j = 0; j < J; j++) {
      gstart[j] = run;
      run += c[j];
    }
  }
  // per digit: offsets of the warps inside the tile, the tile's count, and the counts of all preceding tiles (look-back)
  volatile unsigned* st = state;
  unsigned run[J], excl[J];
#pragma unroll
  for (int j = 0; j < J; j++) {
    const int d = tid * J + j;
    run[j] = 0;
#pragma unroll
    for (int ww = 0; ww < kSortWarps; ww++) {
      const unsigned c = sm.warp_cnt[ww][d];
      sm.warp_cnt[ww][d] = run[j];
      run[j] += c;
    }
    excl[j] = 0;
    st[(size_t)tile * kSortBins + d] = (tile == 0 ? kSortFlagIncl : kSortFlagAgg) | run[j];
  }
  if (tile > 0) {
    // walk back over the preceding tiles, kLook of them per round with all loads in flight (a dependent chain of single loads
    // costs an L2 round trip per tile, which dominated a pass at 17 k points)
    constexpr int kLook = 8;
#pragma unroll
    for (int j = 0; j < J; j++) {
      const int d = tid * J + j;
      long long p = (long long)tile - 1;
      bool done = false;
      while (!done) {
        unsigned v[kLook];
#pragma unroll
        for (int u = 0; u < kLook; u++) v[u] = p - u >= 0 ? (unsigned)st[(size_t)(p - u) * kSortBins + d] : (2u << 30);
#pragma unroll
        for (int u = 0; u < kLook; u++) {
          if (done) break;
          if ((v[u] & kSortFlagMask) == 0u) break;  // not published yet (that tile started before this one: it will): re-read from here
          excl[j] += v[u] & kSortValMask;
          p--;
          if (v[u] & kSortFlagIncl) done = true;
        }
      }
      st[(size_t)tile * kSortBins + d] = kSortFlagIncl | (excl[j] + run[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < J; j++) sm.digit_base[tid * J + j] = gstart[j] + excl[j];
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kSortItems; r++) {
    const long long idx = base + r * 32 + lane;
    if (idx < n) {
      const unsigned d = (unsigned)((key[r] >> shift) & (KeyT)(kSortBins - 1));
      const unsigned pos = sm.digit_base[d] + sm.warp_cnt[w][d] + rank[r];
      kout[pos] = key[r];
      vout[pos] = val[r];
      if (out4) {
        float4 p = in4[val[r]];
        p.w = __uint_as_float(val[r]);
        out4[pos] = p;
      }
    }
  }
}

// stand-alone pass: one block per tile, tiles in ticket order
template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads) k_sort_pass(const KeyT* __restrict__ kin, const unsigned* __restrict__ vin, KeyT* __restrict__ kout, unsigned* __restrict__ vout, int n,
                                                            int pass, const unsigned* __restrict__ hist, unsigned* state, unsigned* ticket, const float4* __restrict__ in4,
                                                            float4* __restrict__ out4) {
  __shared__ SortTileSmem sm;
  if (threadIdx.x == 0) sm.tile = atomicAdd(ticket, 1u);
  __syncthreads();
  sort_pass_tile<KeyT>(sm, sm.tile, kin, vin, kout, vout, n, pass, hist, state, in4, out4);
}

// Sorts n pairs by the low `key_bits` bits of the keys.  (k0, v0) holds the input keys (the values are the positions 0..n-1, v0 is
// only written), (k1, v1) is the second buffer; the result ends up in buffer (passes & 1).  `scratch` = sort_scratch_bytes(n, passes)
// bytes that are zero on entry.  hist_done: the caller already filled the digit histograms (scratch's first kSortMaxPasses*kSortBins
// words).  in4 / out4: optional float4 array permuted along by the last pass.  *launches += kernels launched.
template <typename KeyT>
inline cudaError_t launch_sort_pairs(KeyT* k0, unsigned* v0, KeyT* k1, unsigned* v1, int n, int key_bits, unsigned char* scratch, bool hist_done, const float4* in4, float4* out4,
                                     int* launches, cudaStream_t stream) {
  const int passes = sort_num_passes(key_bits);
  if (passes < 1 || passes > kSortMaxPasses) return cudaErrorInvalidValue;
  unsigned* hist = reinterpret_cast<unsigned*>(scratch);
  unsigned* ticket = hist + (size_t)kSortMaxPasses * kSortBins;
  unsigned* state = ticket + 64;
  const int tiles = sort_num_tiles(n);
  if (!hist_done) {
    int hb = (n + kSortThreads * 8 - 1) / (kSortThreads * 8);
    k_sort_hist<KeyT><<<hb < 4 * kNumSMs ? (hb > 0 ? hb : 1) : 4 * kNumSMs, kSortThreads, 0, stream>>>(k0, n, passes, hist);
    if (launches) (*launches)++;
  }
  KeyT* kk[2] = {k0, k1};
  unsigned* vv[2] = {v0, v1};
  for (int p = 0; p < passes; p++) {
    const bool last = p == passes - 1;
    k_sort_pass<KeyT><<<tiles, kSortThreads, 0, stream>>>(kk[p & 1], p == 0 ? nullptr : vv[p & 1], kk[(p + 1) & 1], vv[(p + 1) & 1], n, p, hist + (size_t)p * kSortBins,
                                                         state + (size_t)p * tiles * kSortBins, ticket + p, last ? in4 : nullptr, last ? out4 : nullptr);
    if (launches) (*launches)++;
  }
  return cudaGetLastError();
}

}  // namespace vgicp
