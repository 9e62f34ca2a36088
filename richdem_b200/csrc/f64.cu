// float64 rasters through order-preserving float keys (DESIGN §0 "float64 elevations").
//
// FillDepressions<D8/D4>, pit_mask, HasDepressions, ResolveFlatsEpsilon, d8_flow_directions, FA_D8 and FA_D4 use an
// elevation in only three ways: they compare it with other elevations, with the raster's NoData value and with
// numeric_limits<T>::max(); the fill copies one cell's value into another; and the flats' last step applies
// nextafter(z, +inf) k times.  So for a map kappa from doubles to floats that is strictly increasing on the raster's
// values, sends DBL_MAX, -DBL_MAX, +-inf and NaN to FLT_MAX, -FLT_MAX, +-inf and NaN, and gives -0.0 and +0.0 keys that
// compare equal, the float engine on kappa(Z) takes the control flow the double template takes on Z, and every value it
// copies is kappa of the value the double run copies.  This file builds kappa(Z) (the only new hot path), maps a filled
// key raster back to doubles, and applies the flats' increment mask as double ulps.  The float engines run unchanged.
// Over row bands the same engines run on kappa_G, one map shared by every band (the second half of this file).
//
// kappa, chosen by looking at the input:
//   case 1  every value is NaN, +-inf or a float-exact double with |z| < FLT_MAX (a widened float raster):
//           kappa(z) = (float)z, one pass.  A cell at +-FLT_MAX goes to case 2: its image would collide with DBL_MAX's.
//   case 2  dense ranks: sort (order key, cell) pairs by an LSD radix sort over the 8-bit digits that are not the same
//           for every key, rank the runs of equal values (+-0 together, every NaN apart), and give rank r the key
//           __uint_as_float(0x00800000 + r): positive normals, strictly inside (-FLT_MAX, FLT_MAX) because a raster
//           holds fewer than 2^31 - 2^25 cells.  The sorted distinct doubles are the inverse table.
// kappa(nodata) is the key of a cell equal to nodata; without one, the constant's image when nodata is one, else NaN
// (which equals nothing, as nodata then does).
//
// Everything here uses plain loads, shared-memory atomics, barriers and full-mask warp collectives (no TMA, no PTX), so
// the test suite's CPU model of the kernels runs it as it runs the float engines.
#include "common.cuh"

#include <cfloat>

namespace rdb {

namespace {

constexpr int SORT_THREADS = 256;  // every kernel below assumes 256 threads (8 warps) per block
constexpr int SORT_ITEMS = 16;
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;  // cells per tile of a sort pass, entries per chunk of a scan
constexpr uint32_t RANK_BASE = 0x00800000u;           // FLT_MIN: the key of rank 0
constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t NO_KEY = 0xffffffffu;  // "no cell equals nodata" (a NaN pattern: never the key of a cell equal to it)

// monotone uint64 image of a double (negative values reversed below the positive ones); -0.0 sits just below +0.0
__device__ __forceinline__ uint64_t order_key(double v) {
  const uint64_t b = (uint64_t)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double order_value(uint64_t k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ float rank_key(double v, uint32_t r) {
  if (v != v) return __uint_as_float(0x7fc00000u);
  if (v == (double)INFINITY) return INFINITY;
  if (v == -(double)INFINITY) return -INFINITY;
  if (v == DBL_MAX) return FLT_MAX;
  if (v == -DBL_MAX) return -FLT_MAX;
  return __uint_as_float(RANK_BASE + r);
}

// kappa^-1 of a key the float engine produced (table: case 2's sorted distinct doubles, null in case 1)
__device__ __forceinline__ double key_value(float k, const double *__restrict__ table) {
  if (k != k) return __longlong_as_double(0x7ff8000000000000ll);
  if (k == INFINITY) return (double)INFINITY;
  if (k == -INFINITY) return -(double)INFINITY;
  if (!table) return (double)k;
  if (k == FLT_MAX) return DBL_MAX;
  if (k == -FLT_MAX) return -DBL_MAX;
  return table[__float_as_uint(k) - RANK_BASE];
}

// case 1, speculatively: key = (float)z; *inexact = 1 if some value is none of NaN, +-inf, a float-exact |z| < FLT_MAX.
// *nd_key receives the key of some cell equal to nodata.
__global__ void __launch_bounds__(256) f64_cast_kernel(const double *__restrict__ z, float *__restrict__ key, size_t n,
                                                       double nodata, int *inexact, uint32_t *nd_key) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  int bad = 0, found = 0;
  uint32_t nd_bits = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double v = z[i];
    const float f = (float)v;
    const bool special = v != v || v == (double)INFINITY || v == -(double)INFINITY;
    if (!special && !((double)f == v && fabs(v) < (double)FLT_MAX)) bad = 1;
    if (v == nodata) {
      found = 1;
      nd_bits = __float_as_uint(f);
    }
    key[i] = f;
  }
  if (found) *nd_key = nd_bits;  // cells equal to nodata share a key (up to the sign of a zero): any writer will do
  if (__syncthreads_or(bad) && threadIdx.x == 0) *inexact = 1;
}

// the (order key, cell) pair at position i: from the previous pass's output, or straight from Z before the first pass
__device__ __forceinline__ void load_pair(size_t i, const uint64_t *__restrict__ ks, const uint32_t *__restrict__ is,
                                          const double *__restrict__ z, uint64_t &k, uint32_t &idx) {
  if (z) {
    k = order_key(z[i]);
    idx = (uint32_t)i;
  } else {
    k = ks[i];
    idx = is[i];
  }
}

// all eight digit histograms in one pass: hist[d * 256 + b] counts the keys whose digit d (bits 8d..8d+7) is b
__global__ void __launch_bounds__(256) digit_hist_kernel(const double *__restrict__ z, size_t n, uint32_t *hist) {
  __shared__ uint32_t s[8 * 256];
  for (int k = threadIdx.x; k < 8 * 256; k += blockDim.x) s[k] = 0;
  __syncthreads();
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t k = order_key(z[i]);
#pragma unroll
    for (int d = 0; d < 8; d++) atomicAdd(&s[d * 256 + (int)((k >> (8 * d)) & 255u)], 1u);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < 8 * 256; k += blockDim.x)
    if (s[k]) atomicAdd(&hist[k], s[k]);
}

// exclusive scan of one value per thread over the block (256 threads); total = the block's sum.  ws: 8 shared words.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *ws, uint32_t &total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(FULL, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  uint32_t before = 0;
  total = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t s = ws[k];
    if (k < wid) before += s;
    total += s;
  }
  __syncthreads();  // ws is reused by the next call
  return before + x - v;
}

// per-tile digit counts of one sort pass, digit-major: counts[b * tiles + tile]
__global__ void __launch_bounds__(256) tile_count_kernel(const uint64_t *__restrict__ ks, const double *__restrict__ z, size_t n,
                                                         int shift, uint32_t *__restrict__ counts, uint32_t tiles) {
  __shared__ uint32_t s[256];
  s[threadIdx.x] = 0;
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * SORT_TILE;
  for (int r = 0; r < SORT_ITEMS; r++) {
    const size_t i = base + (size_t)r * SORT_THREADS + threadIdx.x;
    if (i < n) {
      const uint64_t k = z ? order_key(z[i]) : ks[i];
      atomicAdd(&s[(int)((k >> shift) & 255u)], 1u);
    }
  }
  __syncthreads();
  counts[(size_t)threadIdx.x * tiles + blockIdx.x] = s[threadIdx.x];
}

// stable scatter of one sort pass.  offsets[b * tiles + tile] is where the tile's first digit-b key goes.  The tile is
// read in rounds of 256 consecutive cells; inside a round a key's place is the count of earlier same-digit keys of its
// tile: earlier rounds (s_base), earlier warps (prefix of s_wcnt) and lower lanes (a peer mask from 8 ballots).
__global__ void __launch_bounds__(256) tile_scatter_kernel(const uint64_t *__restrict__ ks, const uint32_t *__restrict__ is,
                                                           const double *__restrict__ z, uint64_t *__restrict__ ko,
                                                           uint32_t *__restrict__ io, size_t n, int shift,
                                                           const uint32_t *__restrict__ offsets, uint32_t tiles) {
  __shared__ uint32_t s_base[256];
  __shared__ uint32_t s_wcnt[8][256];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  s_base[threadIdx.x] = offsets[(size_t)threadIdx.x * tiles + blockIdx.x];
  const size_t base = (size_t)blockIdx.x * SORT_TILE;
  for (int r = 0; r < SORT_ITEMS; r++) {
#pragma unroll
    for (int w = 0; w < 8; w++) s_wcnt[w][threadIdx.x] = 0;
    __syncthreads();
    const size_t i = base + (size_t)r * SORT_THREADS + threadIdx.x;
    const bool valid = i < n;
    uint64_t k = 0;
    uint32_t idx = 0;
    if (valid) load_pair(i, ks, is, z, k, idx);
    const uint32_t d = (uint32_t)(k >> shift) & 255u;
    uint32_t peers = __ballot_sync(FULL, valid);
#pragma unroll
    for (int b = 0; b < 8; b++) {
      const uint32_t bit = (d >> b) & 1u;
      const uint32_t bal = __ballot_sync(FULL, (int)bit);
      peers &= bit ? bal : ~bal;
    }
    const int below = __popc(peers & ((1u << lane) - 1u));
    if (valid && below == 0) s_wcnt[wid][d] = (uint32_t)__popc(peers);
    __syncthreads();
    {  // thread b: prefix of digit b over the warps, starting at the tile's running position
      uint32_t run = s_base[threadIdx.x];
#pragma unroll
      for (int w = 0; w < 8; w++) {
        const uint32_t c = s_wcnt[w][threadIdx.x];
        s_wcnt[w][threadIdx.x] = run;
        run += c;
      }
      s_base[threadIdx.x] = run;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = s_wcnt[wid][d] + (uint32_t)below;
      ko[pos] = k;
      io[pos] = idx;
    }
    __syncthreads();  // s_wcnt is cleared for the next round
  }
}

// entry sources of the chunk scans: a uint32 array, or the run heads of the sorted keys
struct ArraySrc {
  const uint32_t *a;
  __device__ __forceinline__ uint32_t operator()(size_t i) const { return a[i]; }
};
struct HeadSrc {  // 1 where a run of equal values starts (compared as doubles: +-0 share a run, each NaN is its own)
  const uint64_t *ks;
  const double *z;
  __device__ __forceinline__ uint32_t operator()(size_t i) const {
    if (i == 0) return 1;
    const double a = z ? z[i - 1] : order_value(ks[i - 1]);
    const double b = z ? z[i] : order_value(ks[i]);
    return !(a == b);
  }
};

template <class Src>
__global__ void __launch_bounds__(256) chunk_sum_kernel(Src src, size_t m, uint32_t *__restrict__ sums) {
  __shared__ uint32_t ws[8];
  const size_t base = (size_t)blockIdx.x * SORT_TILE;
  uint32_t acc = 0;
  for (int r = 0; r < SORT_ITEMS; r++) {
    const size_t i = base + (size_t)r * SORT_THREADS + threadIdx.x;
    if (i < m) acc += src(i);
  }
  uint32_t total;
  block_exclusive_scan(acc, ws, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// exclusive scan of the chunk sums, one block: 16 consecutive entries per thread and a carry across 4096-entry steps
__global__ void __launch_bounds__(256) sums_scan_kernel(uint32_t *sums, size_t nb) {
  __shared__ uint32_t ws[8];
  uint32_t carry = 0;
  for (size_t c = 0; c < nb; c += SORT_TILE) {
    const size_t b0 = c + (size_t)threadIdx.x * SORT_ITEMS;
    uint32_t v[SORT_ITEMS], acc = 0;
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; j++) {
      v[j] = b0 + j < nb ? sums[b0 + j] : 0u;
      acc += v[j];
    }
    uint32_t total;
    uint32_t run = carry + block_exclusive_scan(acc, ws, total);
#pragma unroll
    for (int j = 0; j < SORT_ITEMS; j++) {
      if (b0 + j < nb) sums[b0 + j] = run;
      run += v[j];
    }
    carry += total;
  }
}

// a[i] = exclusive prefix sum (chunk offsets from sums_scan_kernel)
__global__ void __launch_bounds__(256) scan_apply_kernel(uint32_t *a, size_t m, const uint32_t *__restrict__ sums) {
  __shared__ uint32_t ws[8];
  const size_t base = (size_t)blockIdx.x * SORT_TILE;
  uint32_t carry = sums[blockIdx.x];
  for (int r = 0; r < SORT_ITEMS; r++) {
    const size_t i = base + (size_t)r * SORT_THREADS + threadIdx.x;
    const uint32_t v = i < m ? a[i] : 0u;
    uint32_t total;
    const uint32_t ex = block_exclusive_scan(v, ws, total);
    if (i < m) a[i] = carry + ex;
    carry += total;
  }
}

// ranks of the sorted pairs -> key of every cell, the inverse table (may be null) and the key of a cell equal to nodata
__global__ void __launch_bounds__(256) rank_scatter_kernel(const uint64_t *__restrict__ ks, const uint32_t *__restrict__ is,
                                                           const double *__restrict__ z, size_t n,
                                                           const uint32_t *__restrict__ sums, float *__restrict__ key,
                                                           double *__restrict__ table, double nodata, uint32_t *nd_key,
                                                           uint32_t *distinct) {
  __shared__ uint32_t ws[8];
  const HeadSrc head{ks, z};
  const size_t base = (size_t)blockIdx.x * SORT_TILE;
  uint32_t carry = sums[blockIdx.x];
  int found = 0;
  uint32_t nd_bits = 0;
  for (int r = 0; r < SORT_ITEMS; r++) {
    const size_t i = base + (size_t)r * SORT_THREADS + threadIdx.x;
    const bool valid = i < n;
    const uint32_t h = valid ? head(i) : 0u;
    uint32_t total;
    const uint32_t rank = carry + block_exclusive_scan(h, ws, total) + h - 1u;
    carry += total;
    if (valid) {
      uint64_t k;
      uint32_t idx;
      load_pair(i, ks, is, z, k, idx);
      const double v = order_value(k);
      const float f = rank_key(v, rank);
      key[idx] = f;
      if (h && table) table[rank] = v;
      if (distinct && i == n - 1) *distinct = rank + 1u;
      if (v == nodata) {
        found = 1;
        nd_bits = __float_as_uint(f);
      }
    }
  }
  if (found) *nd_key = nd_bits;
}

// the fill's write-back: cells whose key the fill raised take kappa^-1 of it; the others keep their own bits
__global__ void __launch_bounds__(256) f64_writeback_kernel(double *__restrict__ z, const float *__restrict__ key0,
                                                            const float *__restrict__ keyf, size_t n,
                                                            const double *__restrict__ table) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float b = keyf[i];
    if (__float_as_uint(b) != __float_as_uint(key0[i])) z[i] = key_value(b, table);
  }
}

// k successive nextafter(z, +inf) on a double (flats/Barnes2014.hpp:527-528), the double twin of flats.cu's
// advance_ulps: saturates at +inf, and a negative value that reaches zero lands on -0.0
__device__ __forceinline__ double advance_ulps_f64(double z, int k) {
  if (k <= 0 || z != z) return z;
  const uint64_t b = (uint64_t)__double_as_longlong(z);
  const bool neg = (b >> 63) != 0;
  const long long mag = (long long)(b & 0x7fffffffffffffffull);
  long long key = neg ? -mag : mag;  // -0.0 and +0.0 share key 0
  key += k;
  if (key >= 0x7ff0000000000000ll) return (double)INFINITY;
  if (key > 0) return __longlong_as_double(key);
  if (key == 0) return neg ? __longlong_as_double((long long)0x8000000000000000ull) : 0.0;
  return __longlong_as_double((long long)(0x8000000000000000ull | (uint64_t)(-key)));
}

// ResolveFlatsEpsilon's apply (flats/Barnes2014.hpp:496-550) with the increment mask of the key raster: interior cells only
__global__ void __launch_bounds__(256) f64_apply_ulps_kernel(double *__restrict__ z, const int32_t *__restrict__ mask, int W,
                                                             int H) {
  const size_t n = (size_t)W * H, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int m = mask[i];
    if (m <= 0) continue;
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    if (x > 0 && y > 0 && x < W - 1 && y < H - 1) z[i] = advance_ulps_f64(z[i], m);
  }
}

// d8_flats_alter_dem's step on a double (flats/flat_resolution.hpp:565-568).  The reference calls nextafterf even for
// U = double, so the double is rounded to the nearest float (ties to even, overflow to +-inf), takes k float-ulp steps
// towards +inf that saturate at +inf, and the float is widened back.  Both conversions are integer arithmetic on the
// bits, so subnormal doubles and floats take the IEEE path whatever flush-to-zero setting the build uses.  A NaN cell
// never carries a flat label (it equals no neighbour); it is returned unchanged.
__device__ __forceinline__ uint32_t f32_bits_rn(double z) {
  const uint64_t b = (uint64_t)__double_as_longlong(z);
  const uint32_t sign = (uint32_t)(b >> 32) & 0x80000000u;
  const uint64_t mag = b & 0x7fffffffffffffffull;
  const int fe = (int)(mag >> 52) - 1023 + 127;  // biased float exponent of a normal result
  if (fe >= 255) return sign | 0x7f800000u;       // +-inf and every double from 2^128 up
  uint32_t r;
  uint64_t rem, half;
  if (fe >= 1) {
    r = ((uint32_t)fe << 23) | (uint32_t)((mag & 0x000fffffffffffffull) >> 29);
    rem = mag & 0x1fffffffull;
    half = 0x10000000ull;
  } else {  // a float subnormal, in units of 2^-149; a carry out of the fraction gives FLT_MIN's encoding
    const int shift = 30 - fe;
    if (shift > 54) return sign;  // below half of the least subnormal (double subnormals included)
    const uint64_t sig = (mag & 0x000fffffffffffffull) | 0x0010000000000000ull;
    r = (uint32_t)(sig >> shift);
    rem = sig & ((1ull << shift) - 1);
    half = 1ull << (shift - 1);
  }
  if (rem > half || (rem == half && (r & 1u))) r++;  // a carry into the exponent is the right rounding, up to +inf
  return sign | r;
}

__device__ __forceinline__ double f64_of_f32_bits(uint32_t f) {
  const uint64_t sign = (uint64_t)(f & 0x80000000u) << 32;
  const uint32_t mag = f & 0x7fffffffu;
  if (mag >= 0x7f800000u) return __longlong_as_double((long long)(sign | 0x7ff0000000000000ull | ((uint64_t)(mag & 0x7fffffu) << 29)));
  if (mag == 0) return __longlong_as_double((long long)sign);
  int e = (int)(mag >> 23);
  uint32_t m = mag & 0x7fffffu;
  if (e == 0) {  // subnormal: normalise
    e = 1;
    while (!(m & 0x800000u)) {
      m <<= 1;
      e--;
    }
    m &= 0x7fffffu;
  }
  return __longlong_as_double((long long)(sign | ((uint64_t)(e - 127 + 1023) << 52) | ((uint64_t)m << 29)));
}

__device__ __forceinline__ double float_steps_f64(double z, int k) {
  if (k <= 0 || z != z) return z;
  const uint32_t f = f32_bits_rn(z);
  const bool neg = (f >> 31) != 0;
  const long long mag = (long long)(f & 0x7fffffffu);
  long long key = (neg ? -mag : mag) + k;  // as flats.cu's advance_ulps: -0.0 and +0.0 share key 0
  uint32_t r;
  if (key >= 0x7f800000ll) r = 0x7f800000u;
  else if (key > 0) r = (uint32_t)key;
  else if (key == 0) r = neg ? 0x80000000u : 0u;
  else r = 0x80000000u | (uint32_t)(-key);
  return f64_of_f32_bits(r);
}

// d8_flats_alter_dem (flat_resolution.hpp:546-580) with the increment mask of the key raster: interior cells only
__global__ void __launch_bounds__(256) f64_float_steps_kernel(double *__restrict__ z, const int32_t *__restrict__ mask, int W,
                                                              int H) {
  const size_t n = (size_t)W * H, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int m = mask[i];
    if (m <= 0) continue;
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    if (x > 0 && y > 0 && x < W - 1 && y < H - 1) z[i] = float_steps_f64(z[i], m);
  }
}

unsigned stream_blocks(size_t n) {
  const size_t want = (n + 255) / 256, cap = (size_t)ctx().num_sms * 8;
  return (unsigned)(want < cap ? want : cap);
}

// d_sums[b] = the sum of src over the chunks before chunk b (nb chunks of 4096 entries of m)
template <class Src>
void chunk_sums_dev(Src src, size_t m, uint32_t *d_sums, size_t nb) {
  Ctx &c = ctx();
  chunk_sum_kernel<Src><<<(unsigned)nb, 256, 0, c.stream>>>(src, m, d_sums);
  sums_scan_kernel<<<1, 256, 0, c.stream>>>(d_sums, nb);
  RDB_CK(cudaGetLastError());
  count_launch(2);
}

float host_bits_float(uint32_t b) {
  float f;
  memcpy(&f, &b, sizeof f);
  return f;
}

// kappa(nodata) when no cell equals nodata
float nodata_image(double nodata) {
  if (nodata == (double)INFINITY) return INFINITY;
  if (nodata == -(double)INFINITY) return -INFINITY;
  if (nodata == DBL_MAX) return FLT_MAX;
  if (nodata == -DBL_MAX) return -FLT_MAX;
  return host_bits_float(0x7fc00000u);
}

// case 2 of kappa: d_key = the dense-rank keys, *d_nd = the key of a cell equal to nodata (left alone without one),
// *table (may be null) = the sorted distinct values, *d_distinct (may be null) = their number.  hist: 2048 device words.
void rank_route(const double *d_z, float *d_key, size_t n, double nodata, DevBuf<double> *table, uint32_t *d_nd,
                uint32_t *d_distinct, uint32_t *d_hist) {
  Ctx &c = ctx();
  uint32_t *hb = (uint32_t *)c.pinned;  // 2048 words fit the 64 KiB pinned scratch
  // which digits differ between keys
  RDB_CK(cudaMemsetAsync(d_hist, 0, 8 * 256 * sizeof(uint32_t), c.stream));
  digit_hist_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, n, d_hist);
  RDB_CK(cudaGetLastError());
  count_launch();
  RDB_CK(cudaMemcpyAsync(hb, d_hist, 8 * 256 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  int shifts[8], passes = 0;
  for (int d = 0; d < 8; d++) {
    uint32_t top = 0;
    for (int b = 0; b < 256; b++) top = hb[d * 256 + b] > top ? hb[d * 256 + b] : top;
    if (top != (uint32_t)n) shifts[passes++] = 8 * d;
  }

  const size_t tiles = (n + SORT_TILE - 1) / SORT_TILE;
  DevBuf<uint64_t> ka, kb;
  DevBuf<uint32_t> ia, ib, counts, sums;
  sums.alloc(tiles);  // chunk sums: n / 4096 chunks of run heads, 256 * tiles / 4096 of tile counts
  if (passes) {
    ka.alloc(n), kb.alloc(n), ia.alloc(n), ib.alloc(n), counts.alloc(256 * tiles);
  }
  const uint64_t *ks = nullptr;
  const uint32_t *is = nullptr;
  const double *zsrc = d_z;  // the first pass reads Z itself
  for (int p = 0; p < passes; p++) {
    uint64_t *ko = (p & 1) ? kb.p : ka.p;
    uint32_t *io = (p & 1) ? ib.p : ia.p;
    const size_t m = 256 * tiles, nb = (m + SORT_TILE - 1) / SORT_TILE;
    tile_count_kernel<<<(unsigned)tiles, 256, 0, c.stream>>>(ks, zsrc, n, shifts[p], counts.p, (uint32_t)tiles);
    chunk_sums_dev(ArraySrc{counts.p}, m, sums.p, nb);
    scan_apply_kernel<<<(unsigned)nb, 256, 0, c.stream>>>(counts.p, m, sums.p);
    tile_scatter_kernel<<<(unsigned)tiles, 256, 0, c.stream>>>(ks, is, zsrc, ko, io, n, shifts[p], counts.p, (uint32_t)tiles);
    RDB_CK(cudaGetLastError());
    count_launch(3);
    ks = ko, is = io, zsrc = nullptr;
  }
  counts.reset();
  if (table) table->alloc(n);
  chunk_sums_dev(HeadSrc{ks, zsrc}, n, sums.p, tiles);
  rank_scatter_kernel<<<(unsigned)tiles, 256, 0, c.stream>>>(ks, is, zsrc, n, sums.p, d_key, table ? table->p : nullptr, nodata,
                                                             d_nd, d_distinct);
  RDB_CK(cudaGetLastError());
  count_launch();
}

}  // namespace

float f64_keys_dev(const double *d_z, float *d_key, size_t n, double nodata, DevBuf<double> *table, int *ranked) {
  Ctx &c = ctx();
  DevBuf<uint32_t> flags(2 + 8 * 256);  // [0] inexact, [1] nodata key, [2..] digit histograms
  uint32_t *d_inexact = flags.p, *d_nd = flags.p + 1, *d_hist = flags.p + 2;
  RDB_CK(cudaMemsetAsync(d_inexact, 0, sizeof(uint32_t), c.stream));
  RDB_CK(cudaMemsetAsync(d_nd, 0xff, sizeof(uint32_t), c.stream));
  f64_cast_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, d_key, n, nodata, (int *)d_inexact, d_nd);
  RDB_CK(cudaGetLastError());
  count_launch();
  uint32_t *hb = (uint32_t *)c.pinned;
  RDB_CK(cudaMemcpyAsync(hb, flags.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (ranked) *ranked = hb[0] != 0;
  if (hb[0] == 0) return hb[1] != NO_KEY ? host_bits_float(hb[1]) : nodata_image(nodata);
  RDB_CK(cudaMemsetAsync(d_nd, 0xff, sizeof(uint32_t), c.stream));
  rank_route(d_z, d_key, n, nodata, table, d_nd, nullptr, d_hist);
  RDB_CK(cudaMemcpyAsync(hb, d_nd, sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  return hb[0] != NO_KEY ? host_bits_float(hb[0]) : nodata_image(nodata);
}

// FillDepressions<D8 / D4> of a double raster: fill the key raster, then write kappa^-1 of every raised key
void fill_depressions_dev(double *d_z, int w, int h, bool topo4) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  DevBuf<float> k0(n), kf(n);
  DevBuf<double> table;
  f64_keys_dev(d_z, k0.p, n, 0.0, &table, nullptr);
  RDB_CK(cudaMemcpyAsync(kf.p, k0.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  fill_depressions_dev(kf.p, w, h, topo4);
  f64_writeback_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, k0.p, kf.p, n, table.p);
  RDB_CK(cudaGetLastError());
  count_launch();
  c.stats.cells = (int64_t)n;
}

// ResolveFlatsEpsilon: the increment mask of the key raster (GetFlatMask), applied as double ulps to the original values
void resolve_flats_epsilon_dev(double *d_z, int w, int h, double nodata) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  DevBuf<float> key(n);
  const float nd = f64_keys_dev(d_z, key.p, n, nodata, nullptr, nullptr);
  DevBuf<int32_t> mask(n);
  resolve_flats_dev(key.p, w, h, nd, mask.p, nullptr, false);
  f64_apply_ulps_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, mask.p, w, h);
  RDB_CK(cudaGetLastError());
  count_launch();
}

// GetFlatMask<double>: the increment mask and labels of the key raster (the flats compare elevations only)
void get_flat_mask_dev(const double *d_z, int32_t *d_mask, int32_t *d_labels, int w, int h, double nodata) {
  const size_t n = (size_t)w * h;
  DevBuf<float> key(n);
  const float nd = f64_keys_dev(d_z, key.p, n, nodata, nullptr, nullptr);
  get_flat_mask_dev(key.p, d_mask, d_labels, w, h, nd);
}

// barnes_flat_resolution_d8<double, uint8_t> (flats/flat_resolution.hpp:588-607): D8 directions of the doubles, then the
// increment mask and labels of the flats the direction grid shows, on the keys (flats_from_dirs_kernel compares with ==
// and < only), then either d8_flow_flats or d8_flats_alter_dem's float steps on the doubles and their directions again
void d8_flow_directions_flats_dev(double *d_z, uint8_t *d_dirs, int w, int h, double nodata, bool alter) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  d8_flow_directions_dev(d_z, d_dirs, w, h, nodata);
  DevBuf<float> key(n);
  const float nd = f64_keys_dev(d_z, key.p, n, nodata, nullptr, nullptr);
  DevBuf<int32_t> mask(n), labels(alter ? 0 : n);
  resolve_flats_dev(key.p, w, h, nd, mask.p, alter ? nullptr : labels.p, false, d_dirs);
  key.reset();
  if (alter) {
    f64_float_steps_dev(d_z, mask.p, w, h);
    d8_flow_directions_dev(d_z, d_dirs, w, h, nodata);
  } else {
    d8_flow_flats_dev(mask.p, labels.p, d_dirs, w, h);
  }
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// ---- kappa_G: one key map for a raster cut into row bands (DESIGN §0.1 "kappa over row bands") ---------------------
// Cast route when every band is float-exact.  Otherwise band b sorts its owned values into D_b (its sorted distinct
// values other than NaN, +-inf and +-DBL_MAX) and every value v gets the key r(v) = sum over the bands c of
// |{u in D_c : u < v}|: strictly increasing on the raster's values (v < v' and v in D_a give |{u in D_a : u < v'}| >
// |{u in D_a : u < v}|), equal for equal values, and the same in every band that holds v.  The own band's term is the
// local dense rank; the other bands' terms come from passing every D_c along the rank chain, G - 1 steps in each
// direction, and counting with a merge-path kernel how many received values lie below each element of D_b.

namespace {

constexpr int MERGE_ITEMS = 8;
constexpr int MERGE_TILE = 256 * MERGE_ITEMS;  // merged entries per block of the count kernel

__device__ __forceinline__ bool rank_form(float k) { return k == k && fabsf(k) < FLT_MAX; }  // not a sentinel image

// a message of the chain: [0] the entry count (int64 bits), then the values (and, for kappa_G^-1, the keys after them)
__device__ __forceinline__ size_t msg_count(const double *msg) { return (size_t)__double_as_longlong(msg[0]); }

// merge path of sorted a (na) and b (nb), a first on ties: how many of the first d merged entries come from a
__device__ __forceinline__ size_t merge_split(const double *a, size_t na, const double *b, size_t nb, size_t d) {
  size_t lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (a[mid] <= b[d - mid - 1]) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// cnt[i] += |{u in msg : u < a[i]}| for the sorted a (m values, no NaN) and the sorted values of a chain message.  Block
// k takes merged entries [k T, (k+1) T): it finds its ranges of a and of the message by two merge-path searches, stages
// them in shared memory (coalesced), and every thread merges 8 consecutive entries.  When an element of a is emitted,
// the message entries merged before it are exactly those below it.
__global__ void __launch_bounds__(256) merge_count_kernel(const double *__restrict__ a, size_t m, const double *__restrict__ msg,
                                                          uint32_t *__restrict__ cnt) {
  __shared__ double s[MERGE_TILE];
  __shared__ size_t s_split[2];
  const size_t mb = msg_count(msg);
  const double *b = msg + 1;
  const size_t total = m + mb, d0 = (size_t)blockIdx.x * MERGE_TILE;
  if (d0 >= total) return;  // the whole block
  const size_t d1 = d0 + MERGE_TILE < total ? d0 + MERGE_TILE : total;
  if (threadIdx.x < 2) s_split[threadIdx.x] = merge_split(a, m, b, mb, threadIdx.x ? d1 : d0);
  __syncthreads();
  const size_t i0 = s_split[0], j0 = d0 - i0, i1 = s_split[1], j1 = d1 - i1;
  const int na = (int)(i1 - i0), nb = (int)(j1 - j0);
  for (int k = threadIdx.x; k < na + nb; k += blockDim.x) s[k] = k < na ? a[i0 + k] : b[j0 + (k - na)];
  __syncthreads();
  const int dt = (int)threadIdx.x * MERGE_ITEMS < na + nb ? (int)threadIdx.x * MERGE_ITEMS : na + nb;
  int lo = dt > nb ? dt - nb : 0, hi = dt < na ? dt : na;
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (s[mid] <= s[na + dt - mid - 1]) lo = mid + 1;
    else hi = mid;
  }
  int i = lo, j = dt - lo;
  for (int k = 0; k < MERGE_ITEMS && i + j < na + nb; k++) {
    if (j >= nb || (i < na && s[i] <= s[na + j])) {
      cnt[i0 + i] += (uint32_t)(j0 + j);
      i++;
    } else {
      j++;
    }
  }
}

// the band's table: [0] first entry of D_b in the sorted distinct values (past -DBL_MAX and below), [1] |D_b|,
// [2] |{u in D_b : u < nodata}|.  One thread.
__global__ void band_table_bounds_kernel(const double *__restrict__ table, const uint32_t *__restrict__ distinct, double nodata,
                                         long long *info) {
  const size_t m = *distinct;
  size_t lo = 0, hi = m;
  const uint64_t klo = order_key(-DBL_MAX) + 1, khi = order_key(DBL_MAX);
  while (lo < hi) {  // first entry above -DBL_MAX
    const size_t mid = (lo + hi) / 2;
    if (order_key(table[mid]) < klo) lo = mid + 1;
    else hi = mid;
  }
  const size_t first = lo;
  hi = m;
  while (lo < hi) {  // first entry at DBL_MAX or above
    const size_t mid = (lo + hi) / 2;
    if (order_key(table[mid]) < khi) lo = mid + 1;
    else hi = mid;
  }
  const size_t end = lo;
  lo = first, hi = end;
  while (lo < hi) {  // a NaN nodata counts nothing
    const size_t mid = (lo + hi) / 2;
    if (table[mid] < nodata) lo = mid + 1;
    else hi = mid;
  }
  info[0] = (long long)first;
  info[1] = (long long)(end - first);
  info[2] = (long long)(lo - first);
}

__global__ void __launch_bounds__(256) iota_kernel(uint32_t *__restrict__ a, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a[i] = (uint32_t)i;
}

// local dense-rank keys -> global keys (lo: the table index of D_b[0]); sentinel images stay
__global__ void __launch_bounds__(256) band_gather_kernel(float *__restrict__ key, size_t n, const uint32_t *__restrict__ r,
                                                          uint32_t lo) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float k = key[i];
    if (rank_form(k)) key[i] = __uint_as_float(RANK_BASE + r[__float_as_uint(k) - RANK_BASE - lo]);
  }
}

// index of key rr in the strictly increasing keys[0, m), or m
__device__ __forceinline__ size_t find_key(const uint32_t *__restrict__ keys, size_t m, uint32_t rr) {
  size_t lo = 0, hi = m;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (keys[mid] < rr) lo = mid + 1;
    else hi = mid;
  }
  return lo < m && keys[lo] == rr ? lo : m;
}

// kappa_G^-1 from the band's own table (r(D_b), D_b): cells the fill did not raise keep their bits; a raised cell whose
// level is not in D_b is left pending for the chain pass
__global__ void __launch_bounds__(256) band_writeback_kernel(double *__restrict__ z, const float *__restrict__ key0,
                                                             const float *__restrict__ keyf, size_t n, const uint32_t *__restrict__ r,
                                                             const double *__restrict__ vals, size_t m, uint8_t *__restrict__ pending,
                                                             int *miss) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  int missed = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float b = keyf[i];
    uint8_t p = 0;
    if (__float_as_uint(b) != __float_as_uint(key0[i])) {
      if (!rank_form(b)) {
        z[i] = key_value(b, vals);
      } else {
        const size_t at = find_key(r, m, __float_as_uint(b) - RANK_BASE);
        if (at < m) z[i] = vals[at];
        else p = 1, missed = 1;
      }
    }
    pending[i] = p;
  }
  if (__syncthreads_or(missed) && threadIdx.x == 0) *miss = 1;
}

// the pending cells whose level a received table (values, then keys after cap values) holds
__global__ void __launch_bounds__(256) band_lookup_kernel(double *__restrict__ z, const float *__restrict__ keyf, size_t n,
                                                          uint8_t *__restrict__ pending, const double *__restrict__ msg, size_t cap,
                                                          int *left) {
  const size_t mb = msg_count(msg);
  const double *vals = msg + 1;
  const uint32_t *keys = reinterpret_cast<const uint32_t *>(msg + 1 + cap);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  int still = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!pending[i]) continue;
    const size_t at = find_key(keys, mb, __float_as_uint(keyf[i]) - RANK_BASE);
    if (at < mb) {
      z[i] = vals[at];
      pending[i] = 0;
    } else {
      still = 1;
    }
  }
  if (left && __syncthreads_or(still) && threadIdx.x == 0) *left = 1;
}

// a kappa(nodata) that is a sentinel image, else 0
float sentinel_image(double v) {
  if (v != v) return host_bits_float(0x7fc00000u);
  if (v == (double)INFINITY || v == -(double)INFINITY || v == DBL_MAX || v == -DBL_MAX) return nodata_image(v);
  return 0.f;
}

// a chain message's header on the device
void set_msg_count(double *d_msg, size_t count) {
  Ctx &c = ctx();
  int64_t *h = (int64_t *)c.pinned;
  *h = (int64_t)count;
  RDB_CK(cudaMemcpyAsync(d_msg, h, sizeof(int64_t), cudaMemcpyHostToDevice, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// Pass every band's message (slots doubles after the header) along the chain: G - 1 steps, each sending up what came
// from below and down what came from above (the own message first); visit(msg) runs on each message received.  A side
// without a neighbour receives nothing, so what it forwards has count 0.
template <class Visit>
void chain_pass(const rdb200_comm *comm, const double *d_own, size_t slots, Visit &&visit) {
  Ctx &c = ctx();
  const int rank = comm_rank(comm), world = comm_world(comm);
  if (world == 1) return;
  const size_t words = slots + 1;
  DevBuf<double> bufs(4 * words);  // receive from above / below, two of each (the one received last is sent next)
  RDB_CK(cudaMemsetAsync(bufs.p, 0, 4 * words * sizeof(double), c.stream));
  double *from_up[2] = {bufs.p, bufs.p + words}, *from_dn[2] = {bufs.p + 2 * words, bufs.p + 3 * words};
  const double *send_up = d_own, *send_dn = d_own;
  for (int s = 0; s < world - 1; s++) {
    double *ru = from_up[s & 1], *rd = from_dn[s & 1];
    comm_exchange(comm, send_up, ru, send_dn, rd, words * sizeof(double));
    if (rank > 0) visit(ru);
    if (rank < world - 1) visit(rd);
    send_dn = ru;  // what came from above goes on down, what came from below goes on up
    send_up = rd;
  }
}

}  // namespace

int32_t read_i32(const int32_t *d) {
  Ctx &c = ctx();
  int32_t *h = (int32_t *)c.pinned;
  RDB_CK(cudaMemcpyAsync(h, d, sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  return *h;
}

float mgpu_f64_keys_dev(const rdb200_comm *comm, const double *d_band, float *d_band_keys, int w, int hloc, int gt, int gb,
                        double nodata, BandKeys *inv, int *ranked) {
  Ctx &c = ctx();
  const int rank = comm_rank(comm), world = comm_world(comm);
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * (hloc - gt - gb), off = (size_t)w * gt;
  const double *d_z = d_band + off;
  float *d_key = d_band_keys + off;
  DevBuf<uint32_t> flags(4 + 8 * 256);  // [0] inexact, [1] nodata key, [2] distinct values, [3] spare, [4..] histograms
  uint32_t *d_inexact = flags.p, *d_nd = flags.p + 1, *d_distinct = flags.p + 2, *d_hist = flags.p + 4;
  RDB_CK(cudaMemsetAsync(d_inexact, 0, sizeof(uint32_t), c.stream));
  RDB_CK(cudaMemsetAsync(d_nd, 0xff, sizeof(uint32_t), c.stream));
  f64_cast_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, d_key, n, nodata, (int *)d_inexact, d_nd);
  RDB_CK(cudaGetLastError());
  count_launch();
  uint32_t *hb = (uint32_t *)c.pinned;
  RDB_CK(cudaMemcpyAsync(hb, flags.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  const uint32_t nd_local = hb[1];
  // the route and whether nodata occurs anywhere: one MAX all-reduce of {inexact, nodata occurs here}
  DevBuf<int32_t> vote(2);
  hb[0] = hb[0] != 0;
  hb[1] = nd_local != NO_KEY;
  RDB_CK(cudaMemcpyAsync(vote.p, hb, 2 * sizeof(int32_t), cudaMemcpyHostToDevice, c.stream));
  comm_allreduce(comm, vote.p, 2, RDB200_MAX_I32);
  RDB_CK(cudaMemcpyAsync(hb, vote.p, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  const bool rank_keys = hb[0] != 0, nd_found = hb[1] != 0;
  if (ranked) *ranked = rank_keys;
  if (inv) inv->ranked = rank_keys;
  float nd;
  if (!rank_keys) {  // cast route: (float)z in every band, no cap
    nd = !nd_found ? nodata_image(nodata) : nd_local != NO_KEY ? host_bits_float(nd_local) : (float)nodata;
    exchange_band_rows(comm, d_band_keys, sizeof(float), w, hloc, gt, gb);
    return nd;
  }

  // rank route: local dense ranks and the band's sorted distinct values
  RDB_CK(cudaMemsetAsync(d_distinct, 0, sizeof(uint32_t), c.stream));
  DevBuf<double> table;
  rank_route(d_z, d_key, n, nodata, &table, d_nd, d_distinct, d_hist);
  DevBuf<long long> info(3);
  band_table_bounds_kernel<<<1, 1, 0, c.stream>>>(table.p, d_distinct, nodata, info.p);
  RDB_CK(cudaGetLastError());
  count_launch();
  long long hi[3];
  RDB_CK(cudaMemcpyAsync(c.pinned, info.p, sizeof hi, cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  memcpy(hi, c.pinned, sizeof hi);
  const uint32_t lo = (uint32_t)hi[0];
  const size_t m = (size_t)hi[1];

  // every band's |D_b| (slot b) and sum_b |{u in D_b : u < nodata}| = r(nodata) (slot G): one SUM all-reduce, so every
  // rank sees the same counts and takes the same decision on the cap
  std::vector<int32_t> counts(world + 1, 0);
  counts[rank] = (int32_t)m;
  counts[world] = (int32_t)hi[2];
  DevBuf<int32_t> d_counts(world + 1);
  RDB_CK(cudaMemcpyAsync(d_counts.p, counts.data(), counts.size() * sizeof(int32_t), cudaMemcpyHostToDevice, c.stream));
  comm_allreduce(comm, d_counts.p, counts.size(), RDB200_SUM_I32);
  RDB_CK(cudaMemcpyAsync(counts.data(), d_counts.p, counts.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  int64_t total = 0;
  size_t maxm = 0;
  for (int b = 0; b < world; b++) {
    total += counts[b];
    maxm = (size_t)counts[b] > maxm ? (size_t)counts[b] : maxm;
  }
  const int64_t cap = c.params.f64_band_rank_cap > 0 ? c.params.f64_band_rank_cap : ((int64_t)1 << 31) - ((int64_t)1 << 25);
  if (total >= cap)
    fail("float64 row bands: the bands hold %lld distinct values in all; order keys take fewer than %lld", (long long)total,
         (long long)cap);

  // the own message: [count | D_b], and r = the own term (the local dense rank) to which the chain adds the others
  DevBuf<double> own(maxm + 1);
  RDB_CK(cudaMemcpyAsync(own.p + 1, table.p + lo, m * sizeof(double), cudaMemcpyDeviceToDevice, c.stream));
  table.reset();
  set_msg_count(own.p, m);
  DevBuf<uint32_t> r(m);
  if (m) {  // (a band of NaN, +-inf and +-DBL_MAX only has no D_b)
    iota_kernel<<<stream_blocks(m), 256, 0, c.stream>>>(r.p, m);
    RDB_CK(cudaGetLastError());
    count_launch();
  }
  const unsigned blocks = (unsigned)((m + maxm + MERGE_TILE - 1) / MERGE_TILE);
  chain_pass(comm, own.p, maxm, [&](const double *msg) {
    if (m == 0) return;
    merge_count_kernel<<<blocks, 256, 0, c.stream>>>(own.p + 1, m, msg, r.p);
    RDB_CK(cudaGetLastError());
    count_launch();
  });
  band_gather_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_key, n, r.p, lo);
  RDB_CK(cudaGetLastError());
  count_launch();
  const float img = sentinel_image(nodata);
  nd = !nd_found ? nodata_image(nodata) : img != 0.f ? img : host_bits_float(RANK_BASE + (uint32_t)counts[world]);
  exchange_band_rows(comm, d_band_keys, sizeof(float), w, hloc, gt, gb);
  if (inv) {
    inv->m = m;
    inv->cap = maxm;
    inv->vals.alloc(maxm + 1);
    RDB_CK(cudaMemcpyAsync(inv->vals.p, own.p, (m + 1) * sizeof(double), cudaMemcpyDeviceToDevice, c.stream));
    inv->keys.alloc(m);
    RDB_CK(cudaMemcpyAsync(inv->keys.p, r.p, m * sizeof(uint32_t), cudaMemcpyDeviceToDevice, c.stream));
  }
  return nd;
}

// kappa_G^-1 of a filled key band into the owned rows of the double band: unraised cells keep their bits, raised cells
// take the value of their key -- from the band's own table, else from the tables of the other bands.  The second chain
// pass forwards (value, key) tables rather than the missing keys: a query pass would carry 12 B per distinct missing
// level as a table carries 12 B per distinct value, and a band can miss as many levels as it owns cells, but the queries
// would first have to be made distinct (a sort with its scratch).  The pass runs only when some band missed a level.
void mgpu_f64_writeback_dev(const rdb200_comm *comm, const BandKeys &inv, double *d_band, const float *k0, const float *kf, int w,
                            int hloc, int gt, int gb) {
  Ctx &c = ctx();
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  const size_t n = (size_t)w * (hloc - gt - gb), off = (size_t)w * gt;
  double *d_z = d_band + off;
  k0 += off;
  kf += off;
  if (!inv.ranked) {
    f64_writeback_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, k0, kf, n, nullptr);
    RDB_CK(cudaGetLastError());
    count_launch();
    return;
  }
  DevBuf<uint8_t> pending(n);
  DevBuf<int32_t> flag(2);  // [0] some level missed (MAX over the ranks), [1] some level still missing after the pass
  RDB_CK(cudaMemsetAsync(flag.p, 0, 2 * sizeof(int32_t), c.stream));
  band_writeback_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, k0, kf, n, inv.keys.p, inv.vals.p + 1, inv.m, pending.p,
                                                                flag.p);
  RDB_CK(cudaGetLastError());
  count_launch();
  comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
  if (read_i32(flag.p) == 0) return;
  // the own table: [count | values (cap slots) | keys (cap uint32, in cap / 2 + 1 slots)]
  const size_t cap = inv.cap, slots = cap + cap / 2 + 1;
  DevBuf<double> own(slots + 1);
  RDB_CK(cudaMemcpyAsync(own.p, inv.vals.p, (inv.m + 1) * sizeof(double), cudaMemcpyDeviceToDevice, c.stream));
  RDB_CK(cudaMemcpyAsync(own.p + 1 + cap, inv.keys.p, inv.m * sizeof(uint32_t), cudaMemcpyDeviceToDevice, c.stream));
  chain_pass(comm, own.p, slots, [&](const double *msg) {
    band_lookup_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, kf, n, pending.p, msg, cap, nullptr);
    RDB_CK(cudaGetLastError());
    count_launch();
  });
  // every raised key is the key of some cell of the raster: a level found nowhere is a broken invariant
  band_lookup_kernel<<<stream_blocks(n), 256, 0, c.stream>>>(d_z, kf, n, pending.p, own.p, cap, flag.p + 1);
  RDB_CK(cudaGetLastError());
  count_launch();
  if (read_i32(flag.p + 1)) fail("float64 row bands: a filled level has no value in any band");
}

// ResolveFlatsEpsilon's increment mask applied as double ulps (interior cells of the w x h raster only)
void f64_apply_ulps_dev(double *d_z, const int32_t *d_mask, int w, int h) {
  f64_apply_ulps_kernel<<<stream_blocks((size_t)w * h), 256, 0, ctx().stream>>>(d_z, d_mask, w, h);
  RDB_CK(cudaGetLastError());
  count_launch();
}

// d8_flats_alter_dem's float steps of the increment mask (interior cells of the w x h raster only)
void f64_float_steps_dev(double *d_z, const int32_t *d_mask, int w, int h) {
  f64_float_steps_kernel<<<stream_blocks((size_t)w * h), 256, 0, ctx().stream>>>(d_z, d_mask, w, h);
  RDB_CK(cudaGetLastError());
  count_launch();
}

}  // namespace rdb
