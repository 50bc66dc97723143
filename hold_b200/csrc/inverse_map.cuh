// Inverse of a many-to-one map, for scatter-adds in a fixed order without atomics: the silhouette backward's vertex gather
// (items = the (face, corner) pairs, keys = vertex ids) and the K-NN backward (items = the (query, k) slots, keys = targets).
//
// inverse_map sorts the items by key with an LSD radix sort of 8-bit digits.  Every pass is stable: within a tile the rank of
// an item among the earlier items of its digit comes from __match_any_sync and per-warp counts in a fixed order, and the
// tiles' bases from an exclusive scan of the (digit, tile) counts.  So the items of a key come out in ascending item order,
// every position is a function of the keys alone, and no kernel uses an atomic.  The work is linear in the item count
// whatever the keys: a key chosen by every item costs what distinct keys cost.  The passes alone (radix_sort) also sort the
// BVH's Morton codes (mesh_bvh.cuh).
#pragma once
#include "common.cuh"

namespace hold {

constexpr int kImThreads = 256, kImRounds = 8, kImTile = kImThreads * kImRounds;
constexpr int kImBins = 256, kImWarps = kImThreads / 32;
static_assert(kImBins == kImThreads, "one bin per thread");

// One tile of items in item order, kImThreads at a time: visit(item, digit, rank) per item, rank = the number of earlier items
// of the tile with the same digit.  On return s_run holds the tile's count of each digit.  Synchronises the CTA.
template <typename Visit>
__device__ __forceinline__ void im_tile(const int* __restrict__ keys, int n, int shift, int* s_cnt, int* s_run, Visit&& visit) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  s_run[threadIdx.x] = 0;
  for (int r = 0; r < kImRounds; ++r) {
    const int i = blockIdx.x * kImTile + r * kImThreads + threadIdx.x;
    const bool live = i < n;
    const int d = live ? (keys[i] >> shift) & (kImBins - 1) : -1;
#pragma unroll
    for (int w = 0; w < kImWarps; ++w) s_cnt[w * kImBins + threadIdx.x] = 0;
    __syncthreads();
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int below = __popc(peers & ((1u << lane) - 1u));
    if (live && below == 0) s_cnt[warp * kImBins + d] = __popc(peers);
    __syncthreads();
    if (live) {
      int rank = s_run[d] + below;
      for (int w = 0; w < warp; ++w) rank += s_cnt[w * kImBins + d];
      visit(i, d, rank);
    }
    __syncthreads();
    int t = 0;
#pragma unroll
    for (int w = 0; w < kImWarps; ++w) t += s_cnt[w * kImBins + threadIdx.x];
    s_run[threadIdx.x] += t;
    __syncthreads();
  }
}

// hist[digit * tiles + tile] = the tile's count of the digit
__global__ void __launch_bounds__(kImThreads) k_im_hist(const int* __restrict__ keys, int n, int shift, int* __restrict__ hist) {
  __shared__ int s_cnt[kImWarps * kImBins], s_run[kImBins];
  im_tile(keys, n, shift, s_cnt, s_run, [](int, int, int) {});
  hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s_run[threadIdx.x];
}

// exclusive prefix sum of a[0, m) in place, one CTA
__global__ void __launch_bounds__(1024) k_im_scan(int* __restrict__ a, int m) {
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  for (int base = 0; base < m; base += 1024) {
    const int i = base + threadIdx.x;
    const int x = i < m ? a[i] : 0;
    int v = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int w = s_w[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_w[lane] = w;
    }
    __syncthreads();
    const int excl = s_carry + (warp ? s_w[warp - 1] : 0) + v - x;
    if (i < m) a[i] = excl;
    __syncthreads();   // s_carry and s_w are read
    if (threadIdx.x == 1023) s_carry = excl + x;
  }
}

// one stable pass: the items move to off[digit * tiles + tile] + their rank; vals NULL = the item indices
__global__ void __launch_bounds__(kImThreads) k_im_scatter(const int* __restrict__ keys, const int* __restrict__ vals, int n, int shift,
                                                           const int* __restrict__ off, int* __restrict__ keys_out, int* __restrict__ vals_out) {
  __shared__ int s_cnt[kImWarps * kImBins], s_run[kImBins], s_off[kImBins];
  s_off[threadIdx.x] = off[(size_t)threadIdx.x * gridDim.x + blockIdx.x];   // read after im_tile's first barrier
  im_tile(keys, n, shift, s_cnt, s_run, [&](int i, int d, int rank) {
    const int p = s_off[d] + rank;
    keys_out[p] = keys[i];
    vals_out[p] = vals ? vals[i] : i;
  });
}

// first[k], k in [0, nkeys]: the first position of the sorted keys that is >= k
__global__ void k_im_first(const int* __restrict__ sorted, int n, int nkeys, int* __restrict__ first) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > nkeys) return;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sorted[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  first[k] = lo;
}

struct InvMap {
  const int* order;   // [n]: the items sorted by key, ascending within a key
  const int* first;   // [nkeys + 1]: the items of key k are order[first[k] .. first[k + 1])
};

// ints of workspace inverse_map needs for n items and keys in [0, nkeys] (nkeys itself = no key: such items are left out)
inline size_t inverse_map_ints(int n, int nkeys) {
  return 4 * (size_t)n + (size_t)kImBins * ceil_div(max(n, 1), kImTile) + (size_t)nkeys + 1;
}

// ints of histogram radix_sort needs for n items
inline size_t radix_sort_hist_ints(int n) { return (size_t)kImBins * ceil_div(max(n, 1), kImTile); }

// Stable sort of the items [0, n) by the low `bits` bits of keys, ceil(bits / 8) passes ping-ponging through kb[] and vb[]
// (n ints each; pass p writes kb[p & 1], vb[p & 1]).  On return *kout, *vout = the sorted keys and the item indices.
inline int radix_sort(hold_ctx* ctx, const int* keys, int n, int bits, int* const kb[2], int* const vb[2], int* hist,
                      const int** kout, const int** vout, cudaStream_t s) {
  const int tiles = ceil_div(max(n, 1), kImTile);
  const int passes = ceil_div(bits, 8);
  const int* kin = keys;
  const int* vin = nullptr;
  for (int p = 0; p < passes; ++p) {
    int* ko = kb[p & 1];
    int* vo = vb[p & 1];
    if (n > 0) {
      k_im_hist<<<tiles, kImThreads, 0, s>>>(kin, n, 8 * p, hist);
      HOLD_LAUNCH_CHECK(ctx);
      k_im_scan<<<1, 1024, 0, s>>>(hist, kImBins * tiles);
      HOLD_LAUNCH_CHECK(ctx);
      k_im_scatter<<<tiles, kImThreads, 0, s>>>(kin, vin, n, 8 * p, hist, ko, vo);
      HOLD_LAUNCH_CHECK(ctx);
    }
    kin = ko, vin = vo;
  }
  *kout = kin, *vout = vin;
  return HOLD_OK;
}

// keys [n] in [0, nkeys] -> *out, all of it inside ws (inverse_map_ints(n, nkeys) ints).  Launches only; sized from n and nkeys.
inline int inverse_map(hold_ctx* ctx, const int* keys, int n, int nkeys, int* ws, InvMap* out, cudaStream_t s) {
  int* const kb[2] = {ws, ws + n};
  int* const vb[2] = {ws + 2 * (size_t)n, ws + 3 * (size_t)n};
  int* hist = ws + 4 * (size_t)n;
  int* first = hist + radix_sort_hist_ints(n);
  int bits = 1;
  while (bits < 31 && (nkeys >> bits) != 0) ++bits;
  const int *kin, *vin;
  int rc = radix_sort(ctx, keys, n, bits, kb, vb, hist, &kin, &vin, s);
  if (rc) return rc;
  k_im_first<<<ceil_div(nkeys + 1, 256), 256, 0, s>>>(kin, n, nkeys, first);
  HOLD_LAUNCH_CHECK(ctx);
  out->order = vin, out->first = first;
  return HOLD_OK;
}

}  // namespace hold
