// Barnes-2014 flat resolution on H100 (reference flats/flats.hpp:21-28, flats/Barnes2014.hpp).
//
// The reference builds the increment mask with serial FIFO floods; its outputs only depend on
// order-independent quantities, which is what the kernels below compute:
//   flats     (find_flats.hpp:28-69)     3x3 stencil classification
//   edges     (Barnes2014.hpp:309-369)   low edge  = NOT_A_FLAT data cell with an equal-elevation
//                                                     IS_A_FLAT neighbour;
//                                        high edge = IS_A_FLAT cell with a higher neighbour
//   labels    (:244-280, :437-441)       8-connected components of exactly-equal elevation that
//                                        contain a low edge  -> lock-free union-find (atomicCAS hooks
//                                        onto the smaller root) + path flattening
//   away      (:62-110)                  1 + multi-source BFS distance from the high edges through
//                                        same-label IS_A_FLAT cells;  H[label] = max away
//   towards   (:152-211)                 1 + BFS distance from the low edges (same stepping rule)
//   mask      (:191-194)                 2*towards + (away>0 ? H[label]-away : 0)
//   apply     (:496-550)                 interior cells with label!=0: `mask` x nextafter(z,+inf),
//                                        done as one integer add on the ordered float key
// BFS levels are level-synchronous launches over compacted frontier arrays; a launch reads its
// frontier length from device memory, so the host only synchronises every few levels.
#include "common.cuh"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <memory>

#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace rdb {

namespace {

constexpr uint8_t FT_FLAT = 1, FT_LOW = 2, FT_HIGH = 4, FT_NODATA = 8;

struct LevelCtl {
  int count;
  int pad;
};
struct FlatDev {
  LevelCtl ctl[3];
  int n_low, n_high, n_flat, n_raised;
  int rounds_done;
  int dist_overflow;  // a geodesic distance reached 2^24, where float steps of 1 stop being exact
};

// a3: FindFlats
__global__ void __launch_bounds__(256) flats_classify_kernel(const float *__restrict__ dem, uint8_t *__restrict__ ft,
                                                              int W, int H, float nodata, FlatDev *dev) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int isflat = 0;
  if (i < n) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const float e = __ldg(dem + i);
    uint8_t f = 0;
    if (e == nodata) {
      f = FT_NODATA;
    } else if (!(x == 0 || y == 0 || x == W - 1 || y == H - 1)) {
      f = FT_FLAT;
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        const float ne = __ldg(dem + (size_t)(y + d8dy(k)) * W + (x + d8dx(k)));
        if (ne < e || ne == nodata) f = 0;  // find_flats.hpp:58-61
      }
    }
    ft[i] = f;
    isflat = f == FT_FLAT;
  }
  const int cnt = __syncthreads_count(isflat);
  if (threadIdx.x == 0 && cnt) atomicAdd(&dev->n_flat, cnt);
}

// a4: FindFlatEdges
__global__ void __launch_bounds__(256) flats_edges_kernel(const float *__restrict__ dem, uint8_t *ft, int W, int H,
                                                           FlatDev *dev) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int low = 0, high = 0;
  if (i < n) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const uint8_t f = ft[i] & (FT_FLAT | FT_NODATA);
    if (!(f & FT_NODATA)) {
      const float e = __ldg(dem + i);
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        const int nx = x + d8dx(k), ny = y + d8dy(k);
        if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
        const size_t ni = (size_t)ny * W + nx;
        const float ne = __ldg(dem + ni);
        if (f == 0) {
          if ((ft[ni] & FT_FLAT) && ne == e) low = 1;  // Barnes2014.hpp:343-350
        } else {
          if (e < ne) high = 1;  // :354-360
        }
      }
    }
  }
  // NOTE: neighbours' FT_FLAT/FT_NODATA bits are final (written by the previous kernel); this
  // kernel only ORs the edge bits into its own cell, so concurrent reads of bit 0 are safe.
  if (low | high) ft[i] = (uint8_t)(ft[i] | (low ? FT_LOW : 0) | (high ? FT_HIGH : 0));
  const int nl = __syncthreads_count(low), nh = __syncthreads_count(high);
  if (threadIdx.x == 0) {
    if (nl) atomicAdd(&dev->n_low, nl);
    if (nh) atomicAdd(&dev->n_high, nh);
  }
}

// a3 + a4 in one pass (single-GPU path): a block owns a 128 x 32 window, stages the elevations with a two-cell rim in
// shared memory (every DEM row is fetched once per block instead of ~18 scalar loads per cell through L1/L2), classifies
// the window plus a one-cell rim (the edge rules look at the neighbours' IS_A_FLAT bit), then derives the edge bits and
// stores four flag bytes per thread.  Cells outside the raster are staged as NaN / class 0, which every comparison of the
// two rules treats like "skip" (the reference bounds-checks instead, Barnes2014.hpp:337-341).
constexpr int CE_TX = 128, CE_TY = 32;
__global__ void __launch_bounds__(256) flats_classify_edges_kernel(const float *__restrict__ dem, uint8_t *__restrict__ ft,
                                                                    int W, int H, float nodata, FlatDev *dev) {
  constexpr int DW = CE_TX + 4, DH = CE_TY + 4;  // staged elevations
  constexpr int CW = CE_TX + 2, CH = CE_TY + 2;  // classified region
  __shared__ float sD[DH][DW];
  __shared__ uint8_t sC[CH][CW + 2];
  const int x0 = blockIdx.x * CE_TX, y0 = blockIdx.y * CE_TY;
  const float qnan = __int_as_float(0x7fc00000);
  for (int k = threadIdx.x; k < DW * DH; k += 256) {
    const int r = k / DW, cidx = k - r * DW;
    const int x = x0 - 2 + cidx, y = y0 - 2 + r;
    sD[r][cidx] = (x >= 0 && y >= 0 && x < W && y < H) ? __ldg(dem + (size_t)y * W + x) : qnan;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < CW * CH; k += 256) {
    const int r = k / CW, cidx = k - r * CW;
    const int x = x0 - 1 + cidx, y = y0 - 1 + r;
    uint8_t f = 0;
    if (x >= 0 && y >= 0 && x < W && y < H) {
      const float e = sD[r + 1][cidx + 1];
      if (e == nodata) {
        f = FT_NODATA;
      } else if (!(x == 0 || y == 0 || x == W - 1 || y == H - 1)) {
        f = FT_FLAT;
#pragma unroll
        for (int n = 1; n <= 8; n++) {
          const float ne = sD[r + 1 + d8dy(n)][cidx + 1 + d8dx(n)];
          if (ne < e || ne == nodata) {  // find_flats.hpp:58-61 (most cells leave at their first lower neighbour)
            f = 0;
            break;
          }
        }
      }
    }
    sC[r][cidx] = f;
  }
  __syncthreads();
  int nflat = 0, nlow = 0, nhigh = 0;
  for (int g = threadIdx.x; g < CE_TX * CE_TY / 4; g += 256) {
    const int r = g / (CE_TX / 4), c4 = (g - r * (CE_TX / 4)) * 4;
    const int y = y0 + r;
    if (y >= H) continue;
    uint8_t out[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int cidx = c4 + j, x = x0 + cidx;
      uint8_t f = sC[r + 1][cidx + 1];
      if (x < W && !(f & FT_NODATA)) {
        const float e = sD[r + 2][cidx + 2];
        int low = 0, high = 0;
        if (f == 0) {
#pragma unroll
          for (int n = 1; n <= 8; n++) {
            if ((sC[r + 1 + d8dy(n)][cidx + 1 + d8dx(n)] & FT_FLAT) && sD[r + 2 + d8dy(n)][cidx + 2 + d8dx(n)] == e) {
              low = 1;  // Barnes2014.hpp:343-350
              break;
            }
          }
        } else {
#pragma unroll
          for (int n = 1; n <= 8; n++) {
            if (e < sD[r + 2 + d8dy(n)][cidx + 2 + d8dx(n)]) {
              high = 1;  // :354-360
              break;
            }
          }
        }
        nflat += f == FT_FLAT;
        f = (uint8_t)(f | (low ? FT_LOW : 0) | (high ? FT_HIGH : 0));
        nlow += low;
        nhigh += high;
      }
      out[j] = f;
    }
    const int x = x0 + c4;
    uint8_t *o = ft + (size_t)y * W + x;
    if (x + 3 < W && ((W & 3) == 0)) {
      *reinterpret_cast<uchar4 *>(o) = make_uchar4(out[0], out[1], out[2], out[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; j++)
        if (x + j < W) o[j] = out[j];
    }
  }
  // one atomic per counter and block (a per-warp atomic on three fixed addresses serialises at L2: at 32768^2 that
  // was most of this kernel's time)
  for (int o = 16; o > 0; o >>= 1) {
    nflat += __shfl_xor_sync(0xffffffffu, nflat, o);
    nlow += __shfl_xor_sync(0xffffffffu, nlow, o);
    nhigh += __shfl_xor_sync(0xffffffffu, nhigh, o);
  }
  __shared__ int sCnt[3][8];
  if ((threadIdx.x & 31) == 0) {
    sCnt[0][threadIdx.x >> 5] = nflat;
    sCnt[1][threadIdx.x >> 5] = nlow;
    sCnt[2][threadIdx.x >> 5] = nhigh;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    int tot = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) tot += sCnt[threadIdx.x][k];
    if (tot) atomicAdd(threadIdx.x == 0 ? &dev->n_flat : (threadIdx.x == 1 ? &dev->n_low : &dev->n_high), tot);
  }
}

// Flat / edge flags from a D8 DIRECTION grid instead of from the elevations (flats/flat_resolution.hpp:382-413,
// find_flat_edges of the direction-grid flat resolution): a flat cell is a cell marked NO_FLOW (0), NoData is the
// grid's 255; low edge = cell with flow that has an equal-elevation NO_FLOW neighbour, high edge = NO_FLOW cell with a
// higher neighbour; neighbours outside the grid or NoData in the direction grid are skipped.
__global__ void __launch_bounds__(256) flats_from_dirs_kernel(const float *__restrict__ dem, const uint8_t *__restrict__ dirs,
                                                               uint8_t *__restrict__ ft, int W, int H, FlatDev *dev) {
  const size_t n = (size_t)W * H;
  int nflat = 0, nlow = 0, nhigh = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const uint8_t d = dirs[i];
    uint8_t f = d == 255 ? FT_NODATA : (d == 0 ? FT_FLAT : 0);
    if (d != 255) {
      const float e = __ldg(dem + i);
      for (int k = 1; k <= 8; k++) {
        const int nx = x + d8dx(k), ny = y + d8dy(k);
        if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
        const size_t ni = (size_t)ny * W + nx;
        const uint8_t dn = dirs[ni];
        if (dn == 255) continue;
        const float ne = __ldg(dem + ni);
        if (d != 0 && dn == 0 && ne == e) {
          f |= FT_LOW;
          break;
        } else if (d == 0 && e < ne) {
          f |= FT_HIGH;
          break;
        }
      }
    }
    ft[i] = f;
    nflat += (f & FT_FLAT) != 0;
    nlow += (f & FT_LOW) != 0;
    nhigh += (f & FT_HIGH) != 0;
  }
  for (int o = 16; o > 0; o >>= 1) {
    nflat += __shfl_xor_sync(0xffffffffu, nflat, o);
    nlow += __shfl_xor_sync(0xffffffffu, nlow, o);
    nhigh += __shfl_xor_sync(0xffffffffu, nhigh, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (nflat) atomicAdd(&dev->n_flat, nflat);
    if (nlow) atomicAdd(&dev->n_low, nlow);
    if (nhigh) atomicAdd(&dev->n_high, nhigh);
  }
}

// d8_flow_flats (flats/flat_resolution.hpp:97-116) with d8_masked_FlowDir (:37-63): interior cells still marked NO_FLOW
// take the direction of their lowest same-label neighbour in the increment mask (cardinal neighbours win ties)
__global__ void __launch_bounds__(256) d8_flow_flats_kernel(const int32_t *__restrict__ mask, const int32_t *__restrict__ labels,
                                                             uint8_t *dirs, int W, int H) {
  const size_t n = (size_t)W * H;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    if (x < 1 || y < 1 || x >= W - 1 || y >= H - 1) continue;
    if (dirs[i] != 0) continue;
    const int lab = labels[i];
    int minimum = mask[i], flowdir = 0;
    for (int k = 1; k <= 8; k++) {
      const size_t ni = (size_t)(y + d8dy(k)) * W + (x + d8dx(k));
      if (labels[ni] != lab) continue;
      const int m = mask[ni];
      if (m < minimum || (m == minimum && flowdir > 0 && (flowdir & 1) == 0 && (k & 1) == 1)) {
        minimum = m;
        flowdir = k;
      }
    }
    dirs[i] = (uint8_t)flowdir;
  }
}

// ---- union-find over exactly-equal elevations --------------------------------------------------
__device__ __forceinline__ int uf_find(int *parent, int i) {
  int p = parent[i];
  while (p != i) {
    const int gp = parent[p];
    if (gp != p) parent[i] = gp;  // path halving (benign race: always points to an ancestor)
    i = p;
    p = gp;
  }
  return i;
}

__device__ __forceinline__ void uf_union(int *parent, int a, int b) {
  for (;;) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    // hook the larger root under the smaller one
    const int old = atomicCAS(&parent[b], b, a);
    if (old == b) return;
  }
}

__global__ void __launch_bounds__(256) uf_init_kernel(int *parent, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) parent[i] = (int)i;
}

__global__ void __launch_bounds__(256) uf_union_kernel(const float *__restrict__ dem, const uint8_t *__restrict__ ft,
                                                        int *parent, int W, int H) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (ft[i] & FT_NODATA) return;  // a flat's target elevation is a data value (Barnes2014.hpp:257)
  const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
  const float e = __ldg(dem + i);
  // forward half of the 8-neighbourhood: E(5), SE(6), S(7), SW(8)
#pragma unroll
  for (int k = 5; k <= 8; k++) {
    const int nx = x + d8dx(k), ny = y + d8dy(k);
    if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
    const size_t ni = (size_t)ny * W + nx;
    if (__ldg(dem + ni) == e && !(ft[ni] & FT_NODATA)) uf_union(parent, (int)i, (int)ni);
  }
}

// Two-level variant (flats_uf_tiled = 1): a block first unites the equal-elevation neighbours INSIDE its
// 64x16 tile with the same lock-free union-find running on shared memory (no global atomics), then
// writes every cell's parent as the global index of its in-tile root (the smallest index of its in-tile
// component, so "smaller index wins" still holds); a second kernel unites across tile seams only, on
// those roots.  Replaces uf_init_kernel + uf_union_kernel; the partition is identical.
constexpr int UT_W = 64, UT_H = 16, UT_N = UT_W * UT_H;

__global__ void __launch_bounds__(256) uf_tile_kernel(const float *__restrict__ dem, const uint8_t *__restrict__ ft,
                                                       int *__restrict__ parent, int W, int H) {
  __shared__ float sE[UT_N];
  __shared__ int sP[UT_N];
  __shared__ uint8_t sOk[UT_N];
  const int x0 = blockIdx.x * UT_W, y0 = blockIdx.y * UT_H;
  for (int k = threadIdx.x; k < UT_N; k += blockDim.x) {
    const int lx = k % UT_W, ly = k / UT_W, gx = x0 + lx, gy = y0 + ly;
    float e = 0.f;
    uint8_t ok = 0;
    if (gx < W && gy < H) {
      const size_t i = (size_t)gy * W + gx;
      ok = (ft[i] & FT_NODATA) ? 0 : 1;
      e = __ldg(dem + i);
    }
    sE[k] = e;
    sOk[k] = ok;
    sP[k] = k;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < UT_N; k += blockDim.x) {
    if (!sOk[k]) continue;
    const int lx = k % UT_W, ly = k / UT_W;
    const float e = sE[k];
#pragma unroll
    for (int d = 5; d <= 8; d++) {  // forward half of the 8-neighbourhood: E, SE, S, SW
      const int nx = lx + d8dx(d), ny = ly + d8dy(d);
      if (nx < 0 || nx >= UT_W || ny >= UT_H) continue;
      const int nk = ny * UT_W + nx;
      if (sOk[nk] && sE[nk] == e) uf_union(sP, k, nk);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < UT_N; k += blockDim.x) {
    const int lx = k % UT_W, ly = k / UT_W, gx = x0 + lx, gy = y0 + ly;
    if (gx >= W || gy >= H) continue;
    int r = k;
    for (int p = sP[r]; p != r; p = sP[r]) r = p;  // read-only: the unions are complete
    parent[(size_t)gy * W + gx] = (y0 + r / UT_W) * W + x0 + r % UT_W;
  }
}

// the cells of a tile whose forward neighbours can lie in another tile: left / right column, bottom row
__global__ void __launch_bounds__(128) uf_seams_kernel(const float *__restrict__ dem, const uint8_t *__restrict__ ft, int *parent,
                                                        int W, int H) {
  const int x0 = blockIdx.x * UT_W, y0 = blockIdx.y * UT_H;
  const int t = threadIdx.x;
  int lx, ly;
  if (t < UT_W) {
    lx = t;
    ly = UT_H - 1;
  } else if (t < UT_W + UT_H - 1) {
    lx = 0;
    ly = t - UT_W;
  } else if (t < UT_W + 2 * (UT_H - 1)) {
    lx = UT_W - 1;
    ly = t - (UT_W + UT_H - 1);
  } else {
    return;
  }
  int gx = x0 + lx, gy = y0 + ly;
  // partial tiles at the raster edge: their last real row / column plays the seam role of nothing (no
  // neighbour beyond the raster), so cells outside the raster simply drop out
  if (gx >= W || gy >= H) return;
  const size_t i = (size_t)gy * W + gx;
  if (ft[i] & FT_NODATA) return;
  const float e = __ldg(dem + i);
#pragma unroll
  for (int d = 5; d <= 8; d++) {
    const int nlx = lx + d8dx(d), nly = ly + d8dy(d);
    if (nlx >= 0 && nlx < UT_W && nly < UT_H) continue;  // same tile: done in shared memory
    const int nx = gx + d8dx(d), ny = gy + d8dy(d);
    if (nx < 0 || nx >= W || ny >= H) continue;
    const size_t ni = (size_t)ny * W + nx;
    if (__ldg(dem + ni) == e && !(ft[ni] & FT_NODATA)) uf_union(parent, (int)i, (int)ni);
  }
}

// parent[] for the union-find over exactly-equal elevations, by either variant
void uf_build(const float *d_dem, const uint8_t *ft, int *parent, int w, int h) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (c.params.flats_uf_tiled) {
    dim3 grd((unsigned)((w + UT_W - 1) / UT_W), (unsigned)((h + UT_H - 1) / UT_H));
    uf_tile_kernel<<<grd, 256, 0, c.stream>>>(d_dem, ft, parent, w, h);
    uf_seams_kernel<<<grd, 128, 0, c.stream>>>(d_dem, ft, parent, w, h);
  } else {
    uf_init_kernel<<<blocks, 256, 0, c.stream>>>(parent, n);
    uf_union_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, ft, parent, w, h);
  }
  RDB_CK(cudaGetLastError());
}

// Read-only root lookup (no path compression here: concurrent halving stores could overwrite a
// neighbour's freshly flattened entry with a non-root ancestor).  Writes the root of every data
// cell to `root_of` and flags roots whose component holds a low edge (an outlet).
__global__ void __launch_bounds__(256) uf_roots_kernel(const uint8_t *__restrict__ ft, const int *__restrict__ parent,
                                                        int *__restrict__ root_of, uint8_t *rootflag, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = (int)i;
  for (int p = parent[r]; p != r; p = parent[r]) r = p;
  root_of[i] = r;
  if (ft[i] & FT_LOW) rootflag[r] = 1;
}

// append `item` for the lanes where `pred` holds: one atomicAdd per warp instead of one per lane
__device__ __forceinline__ void warp_append(bool pred, int item, int *queue, int *count) {
  const unsigned bal = __ballot_sync(0xffffffffu, pred);
  if (!bal) return;
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == (__ffs(bal) - 1)) base = atomicAdd(count, __popc(bal));
  base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
  if (pred) queue[base + __popc(bal & ((1u << lane) - 1u))] = item;
}

// distance array of one BFS: 0 = flat cell not reached yet, -1 = not a flat cell (never entered),
// > 0 = level.  Two adjacent IS_A_FLAT cells always have equal elevation (neither has a lower
// neighbour), i.e. the same label, so inside the flood the label test of the reference
// (Barnes2014.hpp:98-104) is implied by "is a flat cell" and one 4-byte load per neighbour suffices.
__global__ void __launch_bounds__(256) bfs_init_kernel(const uint8_t *__restrict__ ft, int *__restrict__ dist, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dist[i] = (ft[i] & FT_FLAT) ? 0 : -1;
}

// ---- BFS ---------------------------------------------------------------------------------------
template <bool AWAY>
__global__ void __launch_bounds__(256) bfs_seed_kernel(const uint8_t *__restrict__ ft, const int *__restrict__ labels,
                                                        int *dist, int *H, int *queue, FlatDev *dev, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool src = false;
  if (i < n) {
    const uint8_t f = ft[i];
    src = AWAY ? ((f & FT_HIGH) && labels[i] != 0)  // Barnes2014.hpp:445-454
               : ((f & FT_LOW) != 0);
    if (src) {
      dist[i] = 1;
      if (AWAY && H[labels[i] - 1] < 1) atomicMax(&H[labels[i] - 1], 1);
    }
  }
  warp_append(src, (int)i, queue, &dev->ctl[0].count);
}

// All BFS levels in ONE cooperative launch: the grid walks the frontier of a level, appends the
// next one (warp-aggregated), and meets at a grid-wide barrier; no host round trip per level.
template <bool AWAY>
__global__ void __launch_bounds__(256) bfs_persistent_kernel(const uint8_t *__restrict__ ft,
                                                              const int *__restrict__ labels, int *dist, int *H, int *q0,
                                                              int *q1, FlatDev *dev, int W, int Hh) {
  cg::grid_group grid = cg::this_grid();
  int round = 0;
  for (;; round++) {
    LevelCtl *cur = &dev->ctl[round % 3];
    LevelCtl *next = &dev->ctl[(round + 1) % 3];
    const int n = *reinterpret_cast<volatile int *>(&cur->count);
    if (n == 0) break;  // every block reads the same, final value (written before the last grid.sync)
    if (blockIdx.x == 0 && threadIdx.x == 0) dev->ctl[(round + 2) % 3].count = 0;
    const int *qc = (round & 1) ? q1 : q0;
    int *qn = (round & 1) ? q0 : q1;
    const int level = round + 1;  // distance value of the cells in the current frontier
    for (int base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
      const int idx = base + threadIdx.x;
      const bool valid = idx < n;
      int c = 0, lab = 0, x = 0, y = 0;
      if (valid) {
        c = __ldcg(qc + idx);  // written by other SMs in the previous level: bypass L1
        lab = labels[c];
        y = c / W;
        x = c - y * W;
      }
      int hmax = 0;
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        const int nx = x + d8dx(k), ny = y + d8dy(k);
        bool won = false;
        int ni = 0;
        if (valid && nx >= 0 && ny >= 0 && nx < W && ny < Hh) {
          ni = ny * W + nx;
          // low-edge sources (first level of the towards-flood) are not flat cells themselves and may
          // touch a lower, different flat: only they need the explicit label test (:196-206)
          if (__ldcg(dist + ni) == 0 && (AWAY || round > 0 || labels[ni] == lab))
            won = atomicCAS(&dist[ni], 0, level + 1) == 0;
        }
        if (won) hmax = level + 1;
        warp_append(won, ni, qn, &next->count);
      }
      if (AWAY && hmax && H[lab - 1] < hmax) atomicMax(&H[lab - 1], hmax);  // flat_height = deepest level, :94
    }
    grid.sync();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) dev->rounds_done = round;
}

__device__ __forceinline__ float advance_ulps(float z, int k) {
  // k successive nextafterf(z, +inf) (Barnes2014.hpp:527-528) as integer arithmetic
  if (k <= 0 || z != z) return z;
  const uint32_t b = __float_as_uint(z);
  const bool neg = (b >> 31) != 0;
  const long long mag = (long long)(b & 0x7fffffffu);
  long long key = neg ? -mag : mag;  // -0.0 and +0.0 share key 0
  key += k;
  if (key >= 0x7f800000ll) return __uint_as_float(0x7f800000u);  // saturate at +inf
  if (key > 0) return __uint_as_float((uint32_t)key);
  if (key == 0) return neg ? __uint_as_float(0x80000000u) : 0.0f;  // a negative value lands on -0.0
  return __uint_as_float(0x80000000u | (uint32_t)(-key));
}

__global__ void __launch_bounds__(256) flats_apply_kernel(float *dem, const int *__restrict__ labels,
                                                           const int *__restrict__ away, const int *__restrict__ tw,
                                                           const int *__restrict__ Hh, int32_t *mask_out,
                                                           int32_t *labels_out, int W, int H, int apply, FlatDev *dev) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int raised = 0;
  if (i < n) {
    const int lab = labels[i];
    int m = 0;
    if (lab != 0) {
      const int t = tw[i];
      if (t > 0) {
        const int a = away[i];
        m = 2 * t + (a > 0 ? Hh[lab - 1] - a : 0);  // :191-194
      }
    }
    if (mask_out) mask_out[i] = m;
    if (labels_out) labels_out[i] = lab;
    if (apply && lab != 0 && m > 0) {
      const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
      if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {  // :511-512 interior only
        const float z = dem[i];
        const float z2 = advance_ulps(z, m);
        dem[i] = z2;
        raised = 1;
      }
    }
  }
  const int cnt = __syncthreads_count(raised);
  if (threadIdx.x == 0 && cnt) atomicAdd(&dev->n_raised, cnt);
}

// 4 cells per thread (W % 4 == 0, no mask / label outputs requested): most quads lie outside every flat and cost one
// 16-byte label load; the others fetch their distances and elevations with 16-byte accesses as well
__global__ void __launch_bounds__(256) flats_apply_x4_kernel(float *dem, const int *__restrict__ labels,
                                                              const int *__restrict__ away, const int *__restrict__ tw,
                                                              const int *__restrict__ Hh, int W, int H, FlatDev *dev) {
  const size_t n4 = (size_t)W * H / 4;
  int raised = 0;
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (size_t)gridDim.x * blockDim.x) {
    const int4 lab = __ldg(reinterpret_cast<const int4 *>(labels) + q);
    if (lab.x | lab.y | lab.z | lab.w) {
      const int4 t4 = __ldg(reinterpret_cast<const int4 *>(tw) + q);
      const int4 a4 = __ldg(reinterpret_cast<const int4 *>(away) + q);
      const int l[4] = {lab.x, lab.y, lab.z, lab.w}, t[4] = {t4.x, t4.y, t4.z, t4.w}, a[4] = {a4.x, a4.y, a4.z, a4.w};
      float4 z4 = reinterpret_cast<float4 *>(dem)[q];
      float z[4] = {z4.x, z4.y, z4.z, z4.w};
      const size_t i0 = q * 4;
      const int y = (int)(i0 / W), x0 = (int)(i0 - (size_t)y * W);
      bool any = false;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (l[j] == 0 || t[j] <= 0) continue;
        const int m = 2 * t[j] + (a[j] > 0 ? __ldg(Hh + l[j] - 1) - a[j] : 0);  // :191-194
        const int x = x0 + j;
        if (m > 0 && x > 0 && y > 0 && x < W - 1 && y < H - 1) {  // :511-512 interior only
          z[j] = advance_ulps(z[j], m);
          raised++;
          any = true;
        }
      }
      if (any) reinterpret_cast<float4 *>(dem)[q] = make_float4(z[0], z[1], z[2], z[3]);
    }
  }
  for (int o = 16; o > 0; o >>= 1) raised += __shfl_xor_sync(0xffffffffu, raised, o);
  __shared__ int sR[8];
  if ((threadIdx.x & 31) == 0) sR[threadIdx.x >> 5] = raised;
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) tot += sR[k];
    if (tot) atomicAdd(&dev->n_raised, tot);  // one atomic per (persistent) block
  }
}

// label = root+1 for data cells of components holding a low edge, else 0 (Barnes2014.hpp:437-441)
__global__ void __launch_bounds__(256) make_labels_kernel(const uint8_t *__restrict__ rootflag,
                                                           const uint8_t *__restrict__ ft, int *labels, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lab = 0;
  if (!(ft[i] & FT_NODATA)) {
    const int r = labels[i];  // root_of[i]
    if (rootflag[r]) lab = r + 1;
  }
  labels[i] = lab;
}

// ---- tiled formulation: the two gradients as geodesic distances solved by the fill's tile engine ----
// away:    seeds = high-edge cells of drainable flats, distance 1            (Barnes2014.hpp:62-110)
// towards: low-edge cells get 1 (set at conversion); the IS_A_FLAT cells next to a low edge of the
//          same elevation (= same flat) are the seeds, distance 2           (Barnes2014.hpp:152-211)
__global__ void __launch_bounds__(256) gradient_seed_kernel(const float *__restrict__ dem, const uint8_t *__restrict__ ft,
                                                             const int *__restrict__ labels, float *__restrict__ winit,
                                                             int W, int H, int away) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float inf = __int_as_float(0x7f800000);
  const uint8_t f = ft[i];
  float w0 = inf;
  if (away) {
    if ((f & FT_HIGH) && labels[i] != 0) w0 = 1.0f;
  } else if (f & FT_FLAT) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const float e = __ldg(dem + i);
#pragma unroll
    for (int k = 1; k <= 8; k++) {
      // (flat cells are interior cells of the raster, but in a row band a ghost row can hold them)
      const int nx = x + d8dx(k), ny = y + d8dy(k);
      if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
      const size_t ni = (size_t)ny * W + nx;
      if ((ft[ni] & FT_LOW) && __ldg(dem + ni) == e) w0 = 2.0f;
    }
  }
  winit[i] = w0;
}

// float distances -> int levels in place (0 = not reached); away also folds the per-flat maximum
__global__ void __launch_bounds__(256) gradient_convert_kernel(const uint8_t *__restrict__ ft, const int *__restrict__ labels,
                                                                int *dist_inout, int *Hh, size_t n, int away, FlatDev *dev) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = __int_as_float(dist_inout[i]);
  int d = (v < __int_as_float(0x7f800000)) ? (int)v : 0;
  // float distances are exact below 2^24 only (w + 1 == w from there on); the reference counts in int32
  if (d >= (1 << 24)) dev->dist_overflow = 1;
  if (!away && (ft[i] & FT_LOW)) d = 1;
  dist_inout[i] = d;
  if (away && d > 0) {
    const int lab = labels[i];
    if (lab != 0 && Hh[lab - 1] < d) atomicMax(&Hh[lab - 1], d);  // flat_height, Barnes2014.hpp:93-94
  }
}

template <bool AWAY>
int run_bfs(const uint8_t *ft, const int *labels, int *dist, int *H, int *q0, int *q1, FlatDev *dev, int w, int h) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  RDB_CK(cudaMemsetAsync(dev->ctl, 0, sizeof(LevelCtl) * 3, c.stream));
  bfs_init_kernel<<<blocks, 256, 0, c.stream>>>(ft, dist, n);
  bfs_seed_kernel<AWAY><<<blocks, 256, 0, c.stream>>>(ft, labels, dist, H, q0, dev, n);
  RDB_CK(cudaGetLastError());
  count_launch();
  FlatDev *hd = (FlatDev *)c.pinned;
  int per_sm = 0;
  RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bfs_persistent_kernel<AWAY>, 256, 0));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 4) per_sm = 4;
  const int grid = c.num_sms * per_sm;
  int wi = w, hi = h;
  void *args[] = {(void *)&ft, (void *)&labels, (void *)&dist, (void *)&H, (void *)&q0, (void *)&q1, (void *)&dev,
                  (void *)&wi, (void *)&hi};
  RDB_CK(cudaLaunchCooperativeKernel((const void *)bfs_persistent_kernel<AWAY>, dim3(grid), dim3(256), args, 0, c.stream));
  count_launch();
  RDB_CK(cudaMemcpyAsync(hd, dev, sizeof(FlatDev), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  const int round = hd->rounds_done;
  return round;
}

}  // namespace

// ResolveFlatsEpsilon (apply=true) / GetFlatMask (apply=false, outputs requested)
void resolve_flats_dev(float *d_dem, int w, int h, float nodata, int32_t *d_mask_out, int32_t *d_labels_out,
                       bool apply, const uint8_t *d_dirs) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  c.stats.cells = (int64_t)n;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  const bool prof = getenv("RDB200_PROFILE") != nullptr;
  auto t_last = std::chrono::steady_clock::now();
  auto lap = [&](const char *what) {
    if (!prof) return;
    cudaStreamSynchronize(c.stream);
    const auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[flats profile] %-24s %8.2f ms\n", what, std::chrono::duration<double, std::milli>(now - t_last).count());
    t_last = now;
  };
  DevBuf<uint8_t> ft(n);
  DevBuf<FlatDev> dev(1);
  RDB_CK(cudaMemsetAsync(dev.p, 0, sizeof(FlatDev), c.stream));
  if (d_dirs) {  // flats as the direction grid defines them (direction-grid flat resolution)
    flats_from_dirs_kernel<<<c.num_sms * 16, 256, 0, c.stream>>>(d_dem, d_dirs, ft.p, w, h, dev.p);
    count_launch();
  } else if (c.params.flats_fused_classify) {
    dim3 grd((unsigned)((w + CE_TX - 1) / CE_TX), (unsigned)((h + CE_TY - 1) / CE_TY));
    flats_classify_edges_kernel<<<grd, 256, 0, c.stream>>>(d_dem, ft.p, w, h, nodata, dev.p);
    count_launch();
  } else {
    flats_classify_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, ft.p, w, h, nodata, dev.p);
    flats_edges_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, ft.p, w, h, dev.p);
    count_launch(2);
  }
  RDB_CK(cudaGetLastError());
  FlatDev *hd = (FlatDev *)c.pinned;
  RDB_CK(cudaMemcpyAsync(hd, dev.p, sizeof(FlatDev), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  const int n_low = hd->n_low, n_flat = hd->n_flat;
  lap("classify+edges");
  if (n_low == 0) {  // Barnes2014.hpp:429-435: nothing to resolve
    if (d_mask_out) RDB_CK(cudaMemsetAsync(d_mask_out, 0, n * sizeof(int32_t), c.stream));
    if (d_labels_out) RDB_CK(cudaMemsetAsync(d_labels_out, 0, n * sizeof(int32_t), c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    return;
  }

  // labels
  DevBuf<int> parent(n), labels(n);
  DevBuf<uint8_t> rootflag(n);
  RDB_CK(cudaMemsetAsync(rootflag.p, 0, n, c.stream));
  uf_build(d_dem, ft.p, parent.p, w, h);
  lap("uf init + union");
  uf_roots_kernel<<<blocks, 256, 0, c.stream>>>(ft.p, parent.p, labels.p, rootflag.p, n);
  make_labels_kernel<<<blocks, 256, 0, c.stream>>>(rootflag.p, ft.p, labels.p, n);
  RDB_CK(cudaGetLastError());
  count_launch(4);

  lap("roots+labels");
  // gradients
  DevBuf<int> away(n), tw(n), Hh(n);
  const size_t qcap = (size_t)n_flat + (size_t)n_low + 16;
  DevBuf<int> q0(qcap), q1(qcap);
  RDB_CK(cudaMemsetAsync(Hh.p, 0, n * sizeof(int), c.stream));
  int levels = 0;
  if (c.params.flats_tiled && c.params.flats_pair) {
    q0.reset();
    q1.reset();
    for (int pass = 0; pass < 2; pass++)
      gradient_seed_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, ft.p, labels.p, reinterpret_cast<float *>(pass == 0 ? away.p : tw.p),
                                                         w, h, pass == 0);
    RDB_CK(cudaGetLastError());
    count_launch(2);
    geodesic_distance_pair_dev(ft.p, FT_FLAT, reinterpret_cast<float *>(away.p), reinterpret_cast<float *>(tw.p), w, h);
    for (int pass = 0; pass < 2; pass++)
      gradient_convert_kernel<<<blocks, 256, 0, c.stream>>>(ft.p, labels.p, pass == 0 ? away.p : tw.p, Hh.p, n, pass == 0, dev.p);
    RDB_CK(cudaGetLastError());
    count_launch(2);
    lap("gradients away + towards (tiled, side by side)");
    levels = (int)c.stats.flat_bfs_levels;
  } else if (c.params.flats_tiled) {
    q0.reset();
    q1.reset();
    for (int pass = 0; pass < 2; pass++) {
      const int is_away = pass == 0;
      int *dist = is_away ? away.p : tw.p;
      gradient_seed_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, ft.p, labels.p, reinterpret_cast<float *>(dist), w, h, is_away);
      RDB_CK(cudaGetLastError());
      count_launch();
      geodesic_distance_dev(ft.p, FT_FLAT, reinterpret_cast<float *>(dist), w, h);
      gradient_convert_kernel<<<blocks, 256, 0, c.stream>>>(ft.p, labels.p, dist, Hh.p, n, is_away, dev.p);
      RDB_CK(cudaGetLastError());
      count_launch();
      lap(is_away ? "gradient away (tiled)" : "gradient towards (tiled)");
    }
    levels = (int)c.stats.flat_bfs_levels;
  } else {
    levels += run_bfs<true>(ft.p, labels.p, away.p, Hh.p, q0.p, q1.p, dev.p, w, h);
    lap("bfs away");
    levels += run_bfs<false>(ft.p, labels.p, tw.p, Hh.p, q0.p, q1.p, dev.p, w, h);
    lap("bfs towards");
  }
  c.stats.flat_bfs_levels = levels;

  if (apply && !d_mask_out && !d_labels_out && (w & 3) == 0 && ((uintptr_t)d_dem & 15) == 0 && c.params.flats_fused_classify)
    flats_apply_x4_kernel<<<(unsigned)std::min<size_t>((n / 4 + 255) / 256, (size_t)c.num_sms * 16), 256, 0, c.stream>>>(
        d_dem, labels.p, away.p, tw.p, Hh.p, w, h, dev.p);
  else
    flats_apply_kernel<<<blocks, 256, 0, c.stream>>>(d_dem, labels.p, away.p, tw.p, Hh.p, d_mask_out, d_labels_out, w, h,
                                                     apply ? 1 : 0, dev.p);
  RDB_CK(cudaGetLastError());
  count_launch();
  RDB_CK(cudaMemcpyAsync(hd, dev.p, sizeof(FlatDev), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  c.stats.flat_cells_raised = hd->n_raised;
  if (hd->dist_overflow)
    fail("resolve_flats: a flat is more than 2^24 cells long; the float distance solver is not exact there "
         "(rdb200_set_param(\"flats_tiled\", 0) selects the int32 level-synchronous solver)");
  lap("apply");
}

// barnes_flat_resolution_d8(elevations, flowdirs, alter) (flats/flat_resolution.hpp:588-607; what apps/rd_d8_flowdirs.cpp
// ships with alter = false): D8 directions, the increment mask and labels of the flats the direction grid shows
// (resolve_flats_barnes, :448-515), then either flow directions inside the flats from the mask (d8_flow_flats, :97-116)
// or the elevations altered by the mask and the directions recomputed (d8_flats_alter_dem, :540-586).
void d8_flow_directions_flats_dev(float *d_dem, uint8_t *d_dirs, int w, int h, float nodata, bool alter) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  d8_flow_directions_dev(d_dem, d_dirs, w, h, nodata);
  if (alter) {
    resolve_flats_dev(d_dem, w, h, nodata, nullptr, nullptr, true, d_dirs);
    d8_flow_directions_dev(d_dem, d_dirs, w, h, nodata);
    return;
  }
  DevBuf<int32_t> mask(n), labels(n);
  resolve_flats_dev(d_dem, w, h, nodata, mask.p, labels.p, false, d_dirs);
  d8_flow_flats_dev(mask.p, labels.p, d_dirs, w, h);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

void d8_flow_flats_dev(const int32_t *d_mask, const int32_t *d_labels, uint8_t *d_dirs, int w, int h) {
  Ctx &c = ctx();
  d8_flow_flats_kernel<<<c.num_sms * 16, 256, 0, c.stream>>>(d_mask, d_labels, d_dirs, w, h);
  RDB_CK(cudaGetLastError());
  count_launch();
}

}  // namespace rdb

// =================================================================================================
// Row-band (multi-GPU) flat resolution.  The stencil / union-find / seeding / conversion / apply
// kernels above run unchanged on the local raster (ghost_top + owned + ghost_bottom rows); what
// crosses a seam moves between the steps below (mgpu_resolve_flats_band drives them over a
// rdb200_comm; the rdb200_dev_flats_* entry points expose them one by one):
//   begin (classify)            -> exchange flag rows (IS_A_FLAT / NoData of the ghost rows)
//   edges                       -> exchange flag rows again (low / high edge bits)
//   components (local union-find over owned + ghost rows, outlet flag per local root)
//                               -> OR the outlet flags of roots that meet at a seam until stable
//   labels
//   gradient_begin(away)        -> band distance protocol (mgpu_relax_band)
//   gradient_end(away)          -> MAX the flat heights of roots that meet at a seam until stable
//   gradient_begin/end(towards) -> band distance protocol
//   apply, finish
// =================================================================================================
struct rdb200_flats_state {
  int W = 0, H = 0, gt = 0, gb = 0;
  float nodata = 0.f;
  float *dem = nullptr;
  rdb::DevBuf<uint8_t> ft, rootflag;
  rdb::DevBuf<int> parent, labels, away, tw, Hh;
  rdb::DevBuf<rdb::FlatDev> dev;
  size_t n() const { return (size_t)W * H; }
  unsigned blocks() const { return (unsigned)((n() + 255) / 256); }
};

namespace rdb {

namespace {

// ---- seam messages: a side's message is [my edge row | my ghost row] (2 x W entries).  The neighbour's edge row is my
// ghost row and its ghost row is my edge row, so entry [0][x] of what arrives belongs to my ghost cell x and [1][x] to
// my edge cell x.  Rows are local row numbers (edge, ghost) of the side.

// outlet flag of the component (local union-find root) of every seam cell
__global__ void __launch_bounds__(256) seam_flag_payload_kernel(const int *__restrict__ root, const uint8_t *__restrict__ rootflag,
                                                                 int W, int edge, int ghost, uint8_t *__restrict__ msg) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int y = blockIdx.y == 0 ? edge : ghost;
  msg[(size_t)blockIdx.y * W + x] = rootflag[root[(size_t)y * W + x]];
}

// a flag the neighbour has for a data cell sets the flag of my component of that cell; *changed = 1 if one went 0 -> 1
// (every writer stores 1: a plain byte store)
__global__ void __launch_bounds__(256) seam_merge_flags_kernel(const uint8_t *__restrict__ ft, const int *__restrict__ root,
                                                                uint8_t *rootflag, int W, int edge, int ghost,
                                                                const uint8_t *__restrict__ theirs, int *changed) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const size_t i = (size_t)(blockIdx.y == 0 ? ghost : edge) * W + x;
  if (!theirs[(size_t)blockIdx.y * W + x] || (ft[i] & FT_NODATA)) return;
  const int r = root[i];
  if (!rootflag[r]) {
    rootflag[r] = 1;
    *changed = 1;
  }
}

// flat height (deepest away level) of the flat of every seam cell, 0 for cells outside a drainable flat
__global__ void __launch_bounds__(256) seam_height_payload_kernel(const int *__restrict__ labels, const int *__restrict__ Hh, int W,
                                                                   int edge, int ghost, int *__restrict__ msg) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int lab = labels[(size_t)(blockIdx.y == 0 ? edge : ghost) * W + x];
  msg[(size_t)blockIdx.y * W + x] = lab > 0 ? Hh[lab - 1] : 0;
}

// the neighbour's flat heights MAX into mine; *changed = 1 if one grew
__global__ void __launch_bounds__(256) seam_merge_heights_kernel(const int *__restrict__ labels, int *Hh, int W, int edge, int ghost,
                                                                  const int *__restrict__ theirs, int *changed) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int lab = labels[(size_t)(blockIdx.y == 0 ? ghost : edge) * W + x];
  if (lab <= 0) return;
  const int v = theirs[(size_t)blockIdx.y * W + x];
  if (v > Hh[lab - 1] && atomicMax(&Hh[lab - 1], v) < v) *changed = 1;  // (heights only grow: a stale read only lets more through)
}

// ---- the steps (shared by the C++ band drivers and the step-wise entry points) ----
// d_dirs: classify from a direction grid (flats_from_dirs_kernel: flags and edge bits in one pass) instead of from the
// elevations
rdb200_flats_state *flats_begin(float *d_dem, int width, int height, float nodata, int ghost_top, int ghost_bottom,
                                const uint8_t *d_dirs = nullptr) {
  Ctx &c = ctx();
  auto *s = new rdb200_flats_state();
  try {
    s->W = width;
    s->H = height;
    s->gt = ghost_top ? 1 : 0;
    s->gb = ghost_bottom ? 1 : 0;
    s->nodata = nodata;
    s->dem = d_dem;
    const size_t n = s->n();
    s->ft.alloc(n);
    s->rootflag.alloc(n);
    s->parent.alloc(n);
    s->labels.alloc(n);
    s->away.alloc(n);
    s->tw.alloc(n);
    s->Hh.alloc(n);
    s->dev.alloc(1);
    RDB_CK(cudaMemsetAsync(s->dev.p, 0, sizeof(FlatDev), c.stream));
    RDB_CK(cudaMemsetAsync(s->rootflag.p, 0, n, c.stream));
    RDB_CK(cudaMemsetAsync(s->Hh.p, 0, n * sizeof(int), c.stream));
    // rows 0 / H-1 are classified as raster-edge cells; for ghost rows the caller overwrites them
    if (d_dirs)
      flats_from_dirs_kernel<<<c.num_sms * 16, 256, 0, c.stream>>>(d_dem, d_dirs, s->ft.p, width, height, s->dev.p);
    else
      flats_classify_kernel<<<s->blocks(), 256, 0, c.stream>>>(d_dem, s->ft.p, width, height, nodata, s->dev.p);
    RDB_CK(cudaGetLastError());
    RDB_CK(cudaStreamSynchronize(c.stream));
  } catch (...) {
    delete s;
    throw;
  }
  return s;
}

void flats_edges(rdb200_flats_state *s) {
  Ctx &c = ctx();
  flats_edges_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->dem, s->ft.p, s->W, s->H, s->dev.p);
  RDB_CK(cudaGetLastError());
  RDB_CK(cudaStreamSynchronize(c.stream));
}

void flats_components(rdb200_flats_state *s) {
  Ctx &c = ctx();
  uf_build(s->dem, s->ft.p, s->parent.p, s->W, s->H);
  uf_roots_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->ft.p, s->parent.p, s->labels.p, s->rootflag.p, s->n());
  RDB_CK(cudaGetLastError());
  RDB_CK(cudaStreamSynchronize(c.stream));
}

void flats_labels(rdb200_flats_state *s) {
  Ctx &c = ctx();
  make_labels_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->rootflag.p, s->ft.p, s->labels.p, s->n());
  RDB_CK(cudaGetLastError());
  RDB_CK(cudaStreamSynchronize(c.stream));
}

rdb200_fill_state *flats_gradient_begin(rdb200_flats_state *s, bool away) {
  Ctx &c = ctx();
  int *dist = away ? s->away.p : s->tw.p;
  gradient_seed_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->dem, s->ft.p, s->labels.p, reinterpret_cast<float *>(dist), s->W, s->H,
                                                          away ? 1 : 0);
  RDB_CK(cudaGetLastError());
  return new_band_distance_state(s->ft.p, FT_FLAT, reinterpret_cast<const float *>(dist), s->W, s->H, s->gt, s->gb);
}

void flats_gradient_end(rdb200_flats_state *s, bool away, rdb200_fill_state *dist_state) {
  Ctx &c = ctx();
  int *dist = away ? s->away.p : s->tw.p;
  finish_band_distance_state(dist_state, reinterpret_cast<float *>(dist));
  gradient_convert_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->ft.p, s->labels.p, dist, s->Hh.p, s->n(), away ? 1 : 0, s->dev.p);
  RDB_CK(cudaGetLastError());
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// d_mask_out: write the increment mask there and leave the elevations alone
void flats_apply(rdb200_flats_state *s, int32_t *d_mask_out = nullptr) {
  Ctx &c = ctx();
  flats_apply_kernel<<<s->blocks(), 256, 0, c.stream>>>(s->dem, s->labels.p, s->away.p, s->tw.p, s->Hh.p, d_mask_out, nullptr,
                                                        s->W, s->H, d_mask_out ? 0 : 1, s->dev.p);
  RDB_CK(cudaGetLastError());
  FlatDev *hd = (FlatDev *)c.pinned;
  RDB_CK(cudaMemcpyAsync(hd, s->dev.p, sizeof(FlatDev), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (hd->dist_overflow) fail("resolve_flats (band): a flat is more than 2^24 cells long; float distances are not exact there");
}

// The band protocol of a begun state up to the increment mask, in the order of the comment above.  Flag rows go straight
// from the flag array into the neighbours' ghost rows; the seam merges are the kernels above, and a merge loop ends when
// a 1-int MAX all-reduce says that no rank's merge changed anything.  The two gradients are band relaxations
// (mgpu_relax_band) of the distance states, with R = 64 sweep rounds between halo exchanges when there are several
// bands.  A state begun from a direction grid already has its edge bits (its ghost rows held the neighbours'
// directions), so one flag exchange suffices.  Returns the flag + height merge iterations (0 for one band).
int flats_band_steps(const rdb200_comm *comm, rdb200_flats_state *s, bool from_dirs) {
  Ctx &c = ctx();
  const int world = comm_world(comm);
  const int w = s->W, hloc = s->H, gt = s->gt, gb = s->gb;
  const int edge[2] = {gt, hloc - 1 - gb}, ghost[2] = {0, hloc - 1};  // per side: 0 = top, 1 = bottom
  const bool side_on[2] = {gt != 0, gb != 0};
  auto exchange_rows = [&](void *p, size_t elem) { exchange_band_rows(comm, p, elem, w, hloc, gt, gb); };
  // message buffers: send up, send down, receive up, receive down; 2 rows of int32 at most
  const size_t msg = (size_t)w * 2 * sizeof(int);
  DevBuf<uint8_t> buf(4 * msg);
  uint8_t *snd[2] = {buf.p, buf.p + msg}, *rcv[2] = {buf.p + 2 * msg, buf.p + 3 * msg};
  DevBuf<int> changed(1);
  int *hchanged = (int *)c.pinned + 1024;
  const dim3 blk(256), grd((unsigned)((w + 255) / 256), 2);
  // merge rounds until no rank changed anything; returns the number of rounds
  auto merge_until_stable = [&](bool heights) {
    int it = 0;
    while (world > 1) {
      if (++it > 1000000) fail("mgpu_resolve_flats: seam merges do not settle");
      RDB_CK(cudaMemsetAsync(changed.p, 0, sizeof(int), c.stream));
      for (int k = 0; k < 2; k++) {
        if (!side_on[k]) continue;
        if (heights)
          seam_height_payload_kernel<<<grd, blk, 0, c.stream>>>(s->labels.p, s->Hh.p, w, edge[k], ghost[k],
                                                                reinterpret_cast<int *>(snd[k]));
        else
          seam_flag_payload_kernel<<<grd, blk, 0, c.stream>>>(s->labels.p, s->rootflag.p, w, edge[k], ghost[k], snd[k]);
      }
      RDB_CK(cudaGetLastError());
      comm_exchange(comm, snd[0], rcv[0], snd[1], rcv[1], heights ? msg : (size_t)w * 2);
      for (int k = 0; k < 2; k++) {
        if (!side_on[k]) continue;
        if (heights)
          seam_merge_heights_kernel<<<grd, blk, 0, c.stream>>>(s->labels.p, s->Hh.p, w, edge[k], ghost[k],
                                                               reinterpret_cast<const int *>(rcv[k]), changed.p);
        else
          seam_merge_flags_kernel<<<grd, blk, 0, c.stream>>>(s->ft.p, s->labels.p, s->rootflag.p, w, edge[k], ghost[k], rcv[k],
                                                             changed.p);
      }
      RDB_CK(cudaGetLastError());
      count_launch(2 * (gt + gb));
      comm_allreduce(comm, changed.p, 1, RDB200_MAX_I32);
      RDB_CK(cudaMemcpyAsync(hchanged, changed.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
      RDB_CK(cudaStreamSynchronize(c.stream));
      if (*hchanged == 0) break;
    }
    return it;
  };
  const int R = world > 1 ? 64 : 0;  // sweep rounds between halo exchanges (0: one band relaxes to its fixed point)

  exchange_rows(s->ft.p, 1);  // IS_A_FLAT / NoData (and, from directions, edge bits) of the ghost rows
  if (!from_dirs) {
    flats_edges(s);
    exchange_rows(s->ft.p, 1);  // low / high edge bits of the ghost rows
  }
  flats_components(s);
  int iters = merge_until_stable(false);  // (labels holds every cell's root until flats_labels)
  flats_labels(s);
  for (const bool away : {true, false}) {
    rdb200_fill_state *ds = flats_gradient_begin(s, away);
    try {
      mgpu_relax_band(comm, ds, gt, gb, R);
    } catch (...) {
      rdb200_dev_fill_finish(ds, nullptr);
      throw;
    }
    flats_gradient_end(s, away, ds);
    if (away) iters += merge_until_stable(true);
  }
  return iters;
}

}  // namespace

// ResolveFlatsEpsilon over row bands, driven from C++ over a rdb200_comm.  On return the ghost rows of d_local hold the
// neighbours' resolved edge rows (one last exchange), so that accumulation can follow without another one.
// *seam_iters: flag + height merge iterations (0 for one band).  With d_mask_out the increment mask goes there instead
// (the float64 bands apply it as double ulps) and d_local is not modified.
void mgpu_resolve_flats_band(const rdb200_comm *comm, float *d_local, int w, int hloc, float nodata, int gt, int gb,
                             int *seam_iters, int32_t *d_mask_out) {
  Ctx &c = ctx();
  check_band_args("mgpu_resolve_flats", comm, d_local, w, hloc, gt, gb);
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  std::unique_ptr<rdb200_flats_state> s(flats_begin(d_local, w, hloc, nodata, gt, gb));
  const int iters = flats_band_steps(comm, s.get(), false);
  flats_apply(s.get(), d_mask_out);
  s.reset();
  if (!d_mask_out) exchange_band_rows(comm, d_local, sizeof(float), w, hloc, gt, gb);  // the neighbours' resolved edge rows
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (seam_iters) *seam_iters = iters;
}

// barnes_flat_resolution_d8 (d8_flow_directions_flats_dev) over row bands.  The DEM's ghost rows hold the neighbours'
// edge rows on entry.  Plain directions of the local raster first: its rows 0 / H-1 get the raster-edge rule, which is
// right for the global top / bottom row and is replaced by the neighbours' directions in a ghost row.  The flats are
// resolved by mgpu_dir_flats_band.  alter = 1: the increments go into the owned rows of the DEM, its edge rows cross the
// seams and the directions are computed again.  On return the ghost rows of d_dirs (and, with alter = 1, of d_dem) hold
// the neighbours' edge rows.
void mgpu_d8_flow_directions_flats_band(const rdb200_comm *comm, float *d_dem, uint8_t *d_dirs, int w, int hloc, float nodata,
                                        int gt, int gb, bool alter, int *seam_iters) {
  Ctx &c = ctx();
  const char *what = "mgpu_d8_flow_directions_flats";
  if (!d_dirs) fail("%s: null pointer", what);
  check_band_args(what, comm, d_dem, w, hloc, gt, gb);
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  d8_flow_directions_dev(d_dem, d_dirs, w, hloc, nodata);
  const int iters = mgpu_dir_flats_band(comm, d_dem, d_dirs, w, hloc, nodata, gt, gb, alter, nullptr);
  if (alter) {
    exchange_band_rows(comm, d_dem, sizeof(float), w, hloc, gt, gb);
    d8_flow_directions_dev(d_dem, d_dirs, w, hloc, nodata);
  }
  exchange_band_rows(comm, d_dirs, 1, w, hloc, gt, gb);
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (seam_iters) *seam_iters = iters;
}

// The flats of a band's plain D8 directions d_dirs (owned rows computed; the ghost rows are exchanged here), classified
// from the directions and resolved by the band protocol on the elevations d_dem, whose ghost rows hold the neighbours'
// rows (float32 elevations, or the order keys of a float64 band).  alter = 0: the increment mask crosses the seams
// (d8_flow_flats compares a cell's mask with its same-label neighbours', ghost cells included; adjacent cells share a
// local label exactly when they share a flat), then the NO_FLOW cells take their masked directions.  alter = 1: the
// increments go into d_dem as float ulps, or, with d_mask_out, the increment mask goes there and d_dem is not modified.
// Returns the flag + height merge iterations.
int mgpu_dir_flats_band(const rdb200_comm *comm, float *d_dem, uint8_t *d_dirs, int w, int hloc, float nodata, int gt, int gb,
                        bool alter, int32_t *d_mask_out) {
  Ctx &c = ctx();
  exchange_band_rows(comm, d_dirs, 1, w, hloc, gt, gb);
  std::unique_ptr<rdb200_flats_state> s(flats_begin(d_dem, w, hloc, nodata, gt, gb, d_dirs));
  const int iters = flats_band_steps(comm, s.get(), true);
  if (alter) {
    flats_apply(s.get(), d_mask_out);
  } else {
    DevBuf<int32_t> mask((size_t)w * hloc);
    flats_apply(s.get(), mask.p);
    exchange_band_rows(comm, mask.p, sizeof(int32_t), w, hloc, gt, gb);
    d8_flow_flats_dev(mask.p, s->labels.p, d_dirs, w, hloc);
    RDB_CK(cudaStreamSynchronize(c.stream));
  }
  return iters;
}

}  // namespace rdb

extern "C" {

int rdb200_dev_flats_begin(rdb200_flats_state **state, float *d_dem, int32_t width, int32_t height, float nodata,
                           int32_t ghost_top, int32_t ghost_bottom) {
  return rdb::capi_call([&] {
    using namespace rdb;
    ensure_init();
    if (!state || !d_dem) fail("flats_begin: null pointer");
    if (height - (ghost_top ? 1 : 0) - (ghost_bottom ? 1 : 0) < 1) fail("flats_begin: band has no owned rows");
    *state = flats_begin(d_dem, width, height, nodata, ghost_top, ghost_bottom);
  });
}

// device addresses of the state arrays the caller moves across seams:
//   out[0] flags (uint8 H x W: bit0 flat, bit1 low edge, bit2 high edge, bit3 NoData)
//   out[1] root of every cell's equal-elevation component, later its label (int32 H x W)
//   out[2] outlet flag per root (uint8, indexed by cell index of the root)
//   out[3] away levels, out[4] towards levels (int32 H x W), out[5] flat height per root (int32)
int rdb200_dev_flats_arrays(rdb200_flats_state *s, uint64_t *out6) {
  return rdb::capi_call([&] {
    if (!s || !out6) rdb::fail("flats_arrays: null pointer");
    out6[0] = (uint64_t)s->ft.p;
    out6[1] = (uint64_t)s->labels.p;
    out6[2] = (uint64_t)s->rootflag.p;
    out6[3] = (uint64_t)s->away.p;
    out6[4] = (uint64_t)s->tw.p;
    out6[5] = (uint64_t)s->Hh.p;
  });
}

int rdb200_dev_flats_edges(rdb200_flats_state *s) {
  return rdb::capi_call([&] { rdb::flats_edges(s); });
}

int rdb200_dev_flats_components(rdb200_flats_state *s) {
  return rdb::capi_call([&] { rdb::flats_components(s); });
}

int rdb200_dev_flats_labels(rdb200_flats_state *s) {
  return rdb::capi_call([&] { rdb::flats_labels(s); });
}

int rdb200_dev_flats_gradient_begin(rdb200_flats_state *s, int32_t away, rdb200_fill_state **dist_state) {
  return rdb::capi_call([&] {
    if (!dist_state) rdb::fail("flats_gradient_begin: null pointer");
    *dist_state = rdb::flats_gradient_begin(s, away != 0);
  });
}

int rdb200_dev_flats_gradient_end(rdb200_flats_state *s, int32_t away, rdb200_fill_state *dist_state) {
  return rdb::capi_call([&] { rdb::flats_gradient_end(s, away != 0, dist_state); });
}

int rdb200_dev_flats_apply(rdb200_flats_state *s) {
  return rdb::capi_call([&] { rdb::flats_apply(s); });
}

int rdb200_dev_flats_finish(rdb200_flats_state *s) {
  return rdb::capi_call([&] {
    if (s) {
      RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
      delete s;
    }
  });
}

}  // extern "C"
