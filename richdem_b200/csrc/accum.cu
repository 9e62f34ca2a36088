// Flow accumulation as a topological wavefront over the flow graph:
//
//     A(c) = w(c) + sum over donors u -> c of p(u,c) * A(u)
//
// (reference methods/flow_accumulation_generic.hpp:33-100 and methods/d8_methods.hpp:47-139).
// Every cell carries a remaining-dependency counter; cells with no donors are the sources.  One
// thread starts at each source and pushes its accumulated value downstream with atomicAdd, then
// decrements the receiver's counter with an atomic; the thread that brings a counter to zero is
// the last donor to arrive, so it owns the receiver and keeps walking.  Receivers that become
// ready while the walker already has a successor (two-receiver D-infinity / multi-receiver
// proportions) are appended to a compacted frontier array that seeds the next launch.
// D8 with unit weights only ever adds integers < 2^53 in double, so the result is exact and
// independent of the order in which atomics land (bit-identical to the serial reference).
#include "flowmet.cuh"

#include <cmath>
#include <cooperative_groups.h>
#include <memory>
namespace cg = cooperative_groups;

namespace rdb {

namespace {

constexpr uint32_t kDepsMask = 0xFFu;
constexpr uint32_t kSrcFlag = 0x80000000u;
constexpr int kCodeSole = 32;  // bit 5 of a code byte: this cell is the only donor of its receiver
constexpr int kCodeSource = 64;  // bit 6: this cell has no donors (set by the fused D8 preparation for the walk's source scan)
constexpr int kLaneChunk = 1024;  // cells a persistent warp fetches per cursor atomic (source scans)

// ---- K1: dem -> compact flow code (+ rmax for D-infinity), weights/NoData initialisation ------
// T: float, or double for the float64 FA_Tarboton (the only stage of that engine that reads the DEM)
template <bool DINF, class T = float>
__global__ void __launch_bounds__(256) flow_code_kernel(const T *__restrict__ dem, uint8_t *__restrict__ code,
                                                         float *__restrict__ rmaxArr, double *__restrict__ accum,
                                                         int W, int H, T nodata, int ones, int tfilter) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
  int cd;
  if (DINF) {
    float rmax = 0;
    const int nm = fm_tarboton_cell(dem, x, y, W, H, nodata, &rmax, tfilter != 0);
    if (nm == kCodeNoData || nm == 0) {
      cd = nm;
    } else if (rmax == 0.0f) {
      cd = nm;  // single receiver, proportion 1 (Tarboton1997.hpp:134-135)
    } else if (rmax == kDang) {
      cd = nwrap(nm + 1);  // :136-137
    } else {
      cd = kCodeTwo | nm;  // :138-141
      rmaxArr[i] = rmax;
    }
  } else {
    cd = fm_d8_cell(dem, x, y, W, H, nodata);
  }
  code[i] = (uint8_t)cd;
  if (cd == kCodeNoData) accum[i] = -1.0;  // flow_accumulation_generic.hpp:95-97 (never touched again)
  else if (ones) accum[i] = 1.0;
}

// D8 fast path: 4 consecutive cells of one row per thread (float4 row loads, uchar4 / double2 stores).
// Requires W % 4 == 0.  Same per-cell rule as fm_d8_cell (reference flowmet/OCallaghan1984.hpp:37-75).
__global__ void __launch_bounds__(256) flow_code_d8_x4_kernel(const float *__restrict__ dem, uint8_t *__restrict__ code,
                                                               double *__restrict__ accum, int W, int H, float nodata,
                                                               int ones) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const size_t i0 = (size_t)y * W + x4;
    float r[3][6];  // rows y-1, y, y+1 ; columns x4-1 .. x4+4
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const int yy = y + j - 1;
      if (yy < 0 || yy >= H) {
#pragma unroll
        for (int k = 0; k < 6; k++) r[j][k] = 0.f;
      } else {
        const float *row = dem + (size_t)yy * W + x4;
        const float4 m = __ldg(reinterpret_cast<const float4 *>(row));
        r[j][1] = m.x; r[j][2] = m.y; r[j][3] = m.z; r[j][4] = m.w;
        r[j][0] = x4 > 0 ? __ldg(row - 1) : 0.f;
        r[j][5] = x4 + 4 < W ? __ldg(row + 4) : 0.f;
      }
    }
    uint8_t cd[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int x = x4 + k;
      const float e = r[1][k + 1];
      int c;
      if (e == nodata) {
        c = kCodeNoData;
      } else if (x == 0 || y == 0 || x == W - 1 || y == H - 1) {
        c = 0;
      } else {
        // neighbours n = 1..8 : W, NW, N, NE, E, SE, S, SW
        const float ne[9] = {0.f, r[1][k], r[0][k], r[0][k + 1], r[0][k + 2], r[1][k + 2], r[2][k + 2], r[2][k + 1], r[2][k]};
        int lowest_n = 0;
        float lowest = 3.402823466e+38f;
#pragma unroll
        for (int n = 1; n <= 8; n++) {
          const float v = ne[n];
          if (v == nodata) continue;
          if (v >= e) continue;
          if (v < lowest) {
            lowest = v;
            lowest_n = n;
          }
        }
        c = lowest_n;
      }
      cd[k] = (uint8_t)c;
    }
    *reinterpret_cast<uchar4 *>(code + i0) = make_uchar4(cd[0], cd[1], cd[2], cd[3]);
    double *ap = accum + i0;
    if (ones) {
      reinterpret_cast<double2 *>(ap)[0] = make_double2(cd[0] == kCodeNoData ? -1.0 : 1.0, cd[1] == kCodeNoData ? -1.0 : 1.0);
      reinterpret_cast<double2 *>(ap)[1] = make_double2(cd[2] == kCodeNoData ? -1.0 : 1.0, cd[3] == kCodeNoData ? -1.0 : 1.0);
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++)
        if (cd[k] == kCodeNoData) ap[k] = -1.0;
    }
  }
}

// ---- K2: dependency counters by gathering over the 8 neighbours' codes; marks sources ----------
__global__ void __launch_bounds__(256) deps_gather_kernel(uint8_t *code, uint32_t *__restrict__ st, int W, int H,
                                                           int y_lo, int y_hi, int mark_sole) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
  if (code[i] == kCodeNoData || y < y_lo || y >= y_hi) {  // NoData, or a ghost row of a row band
    st[i] = 0;
    return;
  }
  uint32_t deps = 0;
  size_t donor = 0;
  int donor_code = 0;
#pragma unroll
  for (int k = 1; k <= 8; k++) {
    const int nx = x + d8dx(k), ny = y + d8dy(k);
    if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
    const int cn = code[(size_t)ny * W + nx];
    if ((cn & 15) == 0 || cn == kCodeNoData) continue;
    const int inv = d8_inverse(k);  // direction from that neighbour to me
    const int first = cn & 15;
    bool hit = first == inv;
    if (!hit && (cn & kCodeTwo) && nwrap(first + 1) == inv) hit = true;
    if (hit) {
      deps++;
      donor = (size_t)ny * W + nx;
      donor_code = cn;
    }
  }
  st[i] = deps | (deps == 0 ? kSrcFlag : 0u);
  // A single-receiver donor that is my only donor may add to me without atomics (nobody else
  // touches my accumulator before I am processed): tell it so.  Only this thread writes that bit
  // of that byte; concurrent readers mask it off.
  if (mark_sole && deps == 1 && !(donor_code & kCodeTwo)) code[donor] = (uint8_t)(donor_code | kCodeSole);
}

// 4 cells per thread version of deps_gather_kernel for W % 4 == 0: the three code rows are read as
// 32-bit words (+ one byte on each side) and the four state words leave as one uint4 store.
__global__ void __launch_bounds__(256) deps_gather_x4_kernel(uint8_t *code, uint32_t *__restrict__ st, int W, int H,
                                                              int y_lo, int y_hi, int mark_sole) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const size_t i0 = (size_t)y * W + x4;
    uint8_t r[3][6];  // rows y-1..y+1, columns x4-1..x4+4 ; 0 = "no flow" for anything off the raster
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const int yy = y + j - 1;
      if (yy < 0 || yy >= H) {
#pragma unroll
        for (int k = 0; k < 6; k++) r[j][k] = 0;
      } else {
        const uint8_t *row = code + (size_t)yy * W + x4;
        const uchar4 m = *reinterpret_cast<const uchar4 *>(row);
        r[j][1] = m.x; r[j][2] = m.y; r[j][3] = m.z; r[j][4] = m.w;
        r[j][0] = x4 > 0 ? row[-1] : (uint8_t)0;
        r[j][5] = x4 + 4 < W ? row[4] : (uint8_t)0;
      }
    }
    uint32_t out[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int cc = r[1][k + 1];
      if (cc == kCodeNoData || y < y_lo || y >= y_hi) {
        out[k] = 0;
        continue;
      }
      // neighbour n = 1..8 : W, NW, N, NE, E, SE, S, SW  -> (row, col) in r
      const int nr[9] = {0, 1, 0, 0, 0, 1, 2, 2, 2};
      const int nc[9] = {0, k, k, k + 1, k + 2, k + 2, k + 2, k + 1, k};
      uint32_t deps = 0;
      int dn = 0, dcode = 0;
#pragma unroll
      for (int n = 1; n <= 8; n++) {
        const int cn = r[nr[n]][nc[n]];
        if ((cn & 15) == 0 || cn == kCodeNoData) continue;
        const int inv = d8_inverse(n);
        const int first = cn & 15;
        bool hit = first == inv;
        if (!hit && (cn & kCodeTwo) && nwrap(first + 1) == inv) hit = true;
        if (hit) {
          deps++;
          dn = n;
          dcode = cn;
        }
      }
      out[k] = deps | (deps == 0 ? kSrcFlag : 0u);
      if (mark_sole && deps == 1 && !(dcode & kCodeTwo))
        code[(size_t)(y + d8dy(dn)) * W + (x4 + k + d8dx(dn))] = (uint8_t)(dcode | kCodeSole);
    }
    *reinterpret_cast<uint4 *>(st + i0) = make_uint4(out[0], out[1], out[2], out[3]);
  }
}

// ---- proportions path: scatter dependency counts, then mark sources ----------------------------
__global__ void __launch_bounds__(256) deps_scatter_props_kernel(const float *__restrict__ props, uint32_t *st, int W,
                                                                  int H) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return;  // generic.hpp:47-48 interior only
  const float *p = props + 9 * i;
  if (p[0] == kNoDataGen) return;
#pragma unroll
  for (int k = 1; k <= 8; k++)
    if (p[k] > 0) atomicAdd(&st[i + (ptrdiff_t)d8dy(k) * W + d8dx(k)], 1u);
}

__global__ void __launch_bounds__(256) mark_sources_props_kernel(const float *__restrict__ props, uint32_t *st,
                                                                  double *accum, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (props[9 * i] == kNoDataGen) {
    st[i] = 0;
    accum[i] = -1.0;  // generic.hpp:95-97
    return;
  }
  const uint32_t d = st[i];
  if ((d & kDepsMask) == 0) st[i] = kSrcFlag;
}

// ---- the walk ----------------------------------------------------------------------------------
// MODE 0: compact code, at most one receiver (D8, direction grids)
// MODE 1: compact code, up to two receivers (D-infinity)
// MODE 2: 9-float proportions, up to eight receivers
template <class A>
struct WalkArgs {
  const uint8_t *code;
  const float *rmaxArr;
  const float *props;
  A *accum;
  uint32_t *st;
  const int *frontier;  // nullptr: round 0, every cell whose st has kSrcFlag
  int nfrontier;        // round 0: number of cells
  int *next_frontier;
  int *next_count;
  int W, H;
  // row-band mode: cells below ghost_lo_end / at or above ghost_hi_start belong to a neighbouring
  // band; flow into them is parked in their accum slot and counted in ghostcnt[2*W]
  int ghost_lo_end, ghost_hi_start;
  int *ghostcnt;
};

template <class A>
__device__ __forceinline__ A ld_acc(const A *p) {
  return __ldcg(p);
}

template <class A>
__device__ __forceinline__ bool park_in_ghost(const WalkArgs<A> &a, int r, A val) {
  if (r < a.ghost_lo_end) {
    atomicAdd(a.accum + r, val);
    atomicAdd(a.ghostcnt + r, 1);
    return true;
  }
  if (r >= a.ghost_hi_start) {
    atomicAdd(a.accum + r, val);
    atomicAdd(a.ghostcnt + a.W + (r - a.ghost_hi_start), 1);
    return true;
  }
  return false;
}

template <int MODE, bool CHECK, class A, bool BAND = false>
__global__ void __launch_bounds__(256) accum_walk_kernel(const WalkArgs<A> a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.nfrontier) return;
  int c;
  if (a.frontier) {
    c = a.frontier[t];
  } else {
    c = t;
    if (!(a.st[c] & kSrcFlag)) return;
  }
  const int W = a.W;
  A acc = ld_acc(a.accum + c);
  // receivers that become ready while this walker already has a successor go to the frontier array
  // of the next launch (row-band D-infinity path; single-GPU multi-receiver graphs use accum_levels_kernel)
  for (;;) {
    int next = -1;
    if (MODE == 0) {
      const int cdraw = a.code[c];
      if (cdraw == kCodeNoData) break;
      const int cd = cdraw & 15;
      if (cd == 0) break;
      const int dx = d8dx(cd), dy = d8dy(cd);
      if (CHECK) {  // direction grids may point off the raster (d8_methods.hpp:121-122)
        const int y = c / W, x = c - y * W;
        const int nx = x + dx, ny = y + dy;
        if (nx < 0 || ny < 0 || nx >= W || ny >= a.H) break;
      }
      const int r = c + dy * W + dx;
      if (cdraw & kCodeSole) {
        // I am the receiver's only donor: no other thread touches accum[r] before I hand it on
        const A sum = ld_acc(a.accum + r) + acc;
        a.accum[r] = sum;
        if (CHECK) a.st[r] = 0;  // released: after the walk, donors left in st mark a direction grid's unreleased cells
        acc = sum;
        c = r;
        continue;
      }
      if (a.code[r] == kCodeNoData) break;  // flow into NoData is dropped
      if (BAND && park_in_ghost(a, r, acc)) break;
      atomicAdd(a.accum + r, acc);
      __threadfence();
      const uint32_t old = atomicSub(a.st + r, 1u);
      if ((old & kDepsMask) == 1u) next = r;
    } else if (MODE == 1) {
      const int cd = a.code[c];
      if (cd == kCodeNoData || (cd & 15) == 0) goto no_receiver;
      const int n1 = cd & 15;
      const int r1 = c + d8dy(n1) * W + d8dx(n1);
      int r2 = -1;
      if (cd & kCodeTwo) {
        const int n2 = nwrap(n1 + 1);
        r2 = c + d8dy(n2) * W + d8dx(n2);
        float p1, p2;
        tarboton_props(a.rmaxArr[c], &p1, &p2);
        // generic.hpp:87  accum(ni) += props(ci,n)*c_accum  (float * double)
        const A v1 = (A)((double)p1 * (double)acc), v2 = (A)((double)p2 * (double)acc);
        bool live1 = p1 > 0, live2 = p2 > 0;
        if (BAND) {
          if (live1 && park_in_ghost(a, r1, v1)) live1 = false;
          if (live2 && park_in_ghost(a, r2, v2)) live2 = false;
        }
        if (live1) atomicAdd(a.accum + r1, v1);
        if (live2) atomicAdd(a.accum + r2, v2);
        __threadfence();
        if (live1) {
          const uint32_t o1 = atomicSub(a.st + r1, 1u);
          if ((o1 & kDepsMask) == 1u) next = r1;
        }
        if (live2) {
          const uint32_t o2 = atomicSub(a.st + r2, 1u);
          if ((o2 & kDepsMask) == 1u) {
            if (next < 0) next = r2;
            else a.next_frontier[atomicAdd(a.next_count, 1)] = r2;
          }
        }
      } else {
        if (BAND && park_in_ghost(a, r1, acc)) goto no_receiver;
        atomicAdd(a.accum + r1, acc);
        __threadfence();
        const uint32_t o1 = atomicSub(a.st + r1, 1u);
        if ((o1 & kDepsMask) == 1u) next = r1;
      }
    } else {
      const int y = c / W, x = c - y * W;
      if (x == 0 || y == 0 || x == W - 1 || y == a.H - 1) goto no_receiver;  // edge cells carry no flow
      const float *p = a.props + (size_t)9 * c;
      uint32_t sent = 0;
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        const float pk = p[k];
        if (pk <= 0) continue;  // generic.hpp:82-83
        const int r = c + d8dy(k) * W + d8dx(k);
        if (a.props[(size_t)9 * r] == kNoDataGen) continue;  // :85-86
        atomicAdd(a.accum + r, (A)((double)pk * (double)acc));
        sent |= 1u << k;
      }
      if (!sent) goto no_receiver;
      __threadfence();
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        if (!(sent & (1u << k))) continue;
        const int r = c + d8dy(k) * W + d8dx(k);
        const uint32_t o = atomicSub(a.st + r, 1u);
        if ((o & kDepsMask) == 1u) {
          if (next < 0) next = r;
          else a.next_frontier[atomicAdd(a.next_count, 1)] = r;
        }
      }
    }
  no_receiver:
    if (next < 0) break;
    // the atomicSub that returned 1 was performed after every other donor's (fenced) add, and this
    // L2 load is issued after it returned: it observes the complete sum
    c = next;
    acc = ld_acc(a.accum + c);
  }
}

// one ready cell: push its flow downstream and keep following the receiver it completes for at most
// `budget` steps; every other receiver it completes (and its own continuation when the budget runs
// out) goes to `push`
template <int MODE, bool BAND, class Push>
__device__ __forceinline__ void levels_follow(const WalkArgs<double> &a, int c, int budget, Push &&push) {
  const int W = a.W;
  double acc = __ldcg(a.accum + c);
  for (int step = 0;; step++) {
    int next = -1;
    if (MODE == 1) {
      const int cd = a.code[c];
      if (cd != kCodeNoData && (cd & 15) != 0) {
        const int n1 = cd & 15;
        const int r1 = c + d8dy(n1) * W + d8dx(n1);
        if (cd & kCodeTwo) {
          const int n2 = nwrap(n1 + 1);
          const int r2 = c + d8dy(n2) * W + d8dx(n2);
          float p1, p2;
          tarboton_props(a.rmaxArr[c], &p1, &p2);
          // generic.hpp:87  accum(ni) += props(ci,n)*c_accum  (float * double)
          bool live1 = p1 > 0, live2 = p2 > 0;
          if (BAND) {
            if (live1 && park_in_ghost(a, r1, (double)p1 * acc)) live1 = false;
            if (live2 && park_in_ghost(a, r2, (double)p2 * acc)) live2 = false;
          }
          if (live1) atomicAdd(a.accum + r1, (double)p1 * acc);
          if (live2) atomicAdd(a.accum + r2, (double)p2 * acc);
          __threadfence();
          if (live1 && (atomicSub(a.st + r1, 1u) & kDepsMask) == 1u) next = r1;
          if (live2 && (atomicSub(a.st + r2, 1u) & kDepsMask) == 1u) {
            if (next < 0) next = r2;
            else push(r2);
          }
        } else if (!(BAND && park_in_ghost(a, r1, acc))) {
          atomicAdd(a.accum + r1, acc);
          __threadfence();
          if ((atomicSub(a.st + r1, 1u) & kDepsMask) == 1u) next = r1;
        }
      }
    } else {
      const int y = c / W, x = c - y * W;
      if (!(x == 0 || y == 0 || x == W - 1 || y == a.H - 1)) {  // edge cells carry no flow
        const float *p = a.props + (size_t)9 * c;
        uint32_t sent = 0;
#pragma unroll
        for (int k = 1; k <= 8; k++) {
          const float pk = p[k];
          if (pk <= 0) continue;  // generic.hpp:82-83
          const int r = c + d8dy(k) * W + d8dx(k);
          if (a.props[(size_t)9 * r] == kNoDataGen) continue;  // :85-86
          // row bands: a share bound for a ghost cell is parked there as one parcel
          if (BAND && park_in_ghost(a, r, (double)pk * acc)) continue;
          atomicAdd(a.accum + r, (double)pk * acc);
          sent |= 1u << k;
        }
        if (sent) {
          __threadfence();
#pragma unroll
          for (int k = 1; k <= 8; k++) {
            if (!(sent & (1u << k))) continue;
            const int r = c + d8dy(k) * W + d8dx(k);
            if ((atomicSub(a.st + r, 1u) & kDepsMask) == 1u) {
              if (next < 0) next = r;
              else push(r);
            }
          }
        }
      }
    }
    if (next < 0) break;
    if (step + 1 >= budget) {  // hand the continuation to the next level
      push(next);
      break;
    }
    c = next;
    acc = __ldcg(a.accum + c);
  }
}

// Multi-receiver graphs (D-infinity: <= 2 receivers, proportions: <= 8): ONE cooperative launch.
// Level L drains the frontier written by level L-1 (level 0: every source); a thread processes a
// ready cell and keeps following the receiver it completed for at most `budget` steps, so long
// single-file reaches cost no extra levels, while every other cell it completes -- and its own
// continuation when the budget runs out -- is appended (coalesced-group atomics) to the next
// frontier, where other threads pick it up in parallel.  Levels meet at grid.sync().
// BAND (row bands, D-infinity and proportions): level 0 can be seeded with the cells completed by a neighbour's flow
// (q0[0..ncells), seeded != 0) and flow into a ghost row is parked there instead of followed.
template <int MODE, bool BAND = false>
__global__ void __launch_bounds__(256) accum_levels_kernel(const WalkArgs<double> a, int *q0, int *q1, int *counts,
                                                            int ncells, int budget, int *levels_out, int seeded) {
  cg::grid_group grid = cg::this_grid();
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
  int level = 0;
  for (;; level++) {
    const int n = level == 0 ? ncells : *reinterpret_cast<volatile int *>(&counts[level % 3]);
    if (n == 0) break;
    if (gtid == 0) counts[(level + 2) % 3] = 0;
    const int *qc = (level & 1) ? q1 : q0;
    int *qn = (level & 1) ? q0 : q1;
    int *cntn = &counts[(level + 1) % 3];
    auto push = [&](int r) {
      cg::coalesced_group g = cg::coalesced_threads();
      int base = 0;
      if (g.thread_rank() == 0) base = atomicAdd(cntn, (int)g.size());
      base = g.shfl(base, 0);
      qn[base + g.thread_rank()] = r;
    };
    for (int idx = gtid; idx < n; idx += gsize) {
      int c;
      if (level == 0 && !(BAND && seeded)) {
        c = idx;
        if (!(a.st[c] & kSrcFlag)) continue;
      } else {
        c = __ldcg(qc + idx);
      }
      levels_follow<MODE, BAND>(a, c, budget, push);
    }
    grid.sync();
  }
  if (gtid == 0) *levels_out = level;
}

template <int MODE>
void run_levels(WalkArgs<double> a, size_t ncells) {
  Ctx &c = ctx();
  DevBuf<int> fr0(ncells), fr1(ncells), cnt(4);
  RDB_CK(cudaMemsetAsync(cnt.p, 0, 4 * sizeof(int), c.stream));
  int per_sm = 0;
  RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, accum_levels_kernel<MODE>, 256, 0));
  if (per_sm < 1) per_sm = 1;
  const int grid = c.num_sms * per_sm;
  int *q0 = fr0.p, *q1 = fr1.p, *counts = cnt.p, *lv = cnt.p + 3;
  int nc = (int)ncells, budget = (int)(c.params.accum_budget > 0 ? c.params.accum_budget : 4);
  int seeded = 0;
  void *args[] = {(void *)&a, (void *)&q0, (void *)&q1, (void *)&counts, (void *)&nc, (void *)&budget, (void *)&lv, (void *)&seeded};
  KernelTimer kt;
  RDB_CK(cudaLaunchCooperativeKernel((const void *)accum_levels_kernel<MODE>, dim3(grid), dim3(256), args, 0, c.stream));
  count_launch();
  kt.stop_async();
  int *h = (int *)c.pinned;
  RDB_CK(cudaMemcpyAsync(h, lv, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  RDB_CK(cudaStreamSynchronize(c.stream));
  c.stats.ms_main_kernel += kt.ms();
  c.stats.accum_rounds = *h;
}

template <int MODE, bool CHECK, class A>
void run_walk(WalkArgs<A> a, size_t ncells) {
  Ctx &c = ctx();
  DevBuf<int> fr0, fr1;
  DevBuf<int> cnt(2);
  int *hcnt = (int *)c.pinned;
  if (MODE != 0) {
    fr0.alloc(ncells);
    fr1.alloc(ncells);
  }
  RDB_CK(cudaMemsetAsync(cnt.p, 0, 2 * sizeof(int), c.stream));
  a.frontier = nullptr;
  a.nfrontier = (int)ncells;
  a.next_frontier = fr0.p;
  a.next_count = cnt.p;
  int rounds = 0;
  KernelTimer kt;
  for (;;) {
    const unsigned blocks = (unsigned)(((size_t)a.nfrontier + 255) / 256);
    accum_walk_kernel<MODE, CHECK, A><<<blocks, 256, 0, c.stream>>>(a);
    RDB_CK(cudaGetLastError());
    count_launch();
    rounds++;
    if (MODE == 0) break;
    RDB_CK(cudaMemcpyAsync(hcnt, a.next_count, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    const int nn = *hcnt;
    if (nn == 0) break;
    // swap frontiers
    a.frontier = a.next_frontier;
    a.nfrontier = nn;
    a.next_frontier = (a.frontier == fr0.p) ? fr1.p : fr0.p;
    a.next_count = (a.next_count == cnt.p) ? cnt.p + 1 : cnt.p;
    RDB_CK(cudaMemsetAsync(a.next_count, 0, sizeof(int), c.stream));
  }
  kt.stop_async();
  RDB_CK(cudaStreamSynchronize(c.stream));
  c.stats.ms_main_kernel += kt.ms();
  c.stats.accum_rounds = rounds;
}

__global__ void area_init_kernel(const uint8_t *__restrict__ dirs, int32_t *__restrict__ area, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) area[i] = (dirs[i] == kCodeNoData) ? -1 : 1;  // d8_methods.hpp:71-74, :111
}

// A direction grid may hold loops.  A cell on a loop, or downstream of one, keeps donors that never complete; the
// reference never takes it off its source queue, so it never adds its own unit (d8_methods.hpp:105-111) and keeps only
// the inflow it received.  After the walk such a cell still has donors left in st: it gives back the 1 of area_init.
__global__ void area_unreleased_kernel(const uint32_t *__restrict__ st, int32_t *__restrict__ area, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (st[i] & kDepsMask) != 0) area[i] -= 1;
}

__global__ void sanitize_dirs_kernel(const uint8_t *__restrict__ dirs, uint8_t *__restrict__ code, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const uint8_t d = dirs[i];
    code[i] = (d <= 8 || d == kCodeNoData) ? d : 0;  // anything else: treated as no flow
  }
}

}  // namespace

// =================================================================================================
// Unit-weight D8 over row bands (the single-GPU path, fa_d8_tiles below, uses the same protocol on shared memory
// inside 64 x 64 tiles): every partial sum is an integer < 2^31, so a cell's accumulator and its remaining-donor count
// share ONE 64-bit word
//     [ 8 bits donors left | 56 bits integer sum ]
// living in the caller's accumulation array.  A donor adds (value - 1<<56) with a single atomicAdd:
// the returned old word tells it whether it was the last donor, and if so the complete sum -- no
// second atomic, no fence, no separate load.  The last donor then overwrites the word with the final
// double (nobody else touches it any more) and walks on.  Results are the same integers the
// reference computes in double arithmetic, bit for bit.
// =================================================================================================
namespace {
constexpr unsigned long long kPkOne = 1ull << 56;
constexpr unsigned long long kPkVal = kPkOne - 1;
constexpr unsigned long long kPkSource = (1ull << 63) | 1ull;  // no donors, own unit of flow, not started yet

__global__ void __launch_bounds__(256) deps_gather_packed_x4_kernel(uint8_t *code, unsigned long long *__restrict__ word,
                                                                     int W, int H, int y_lo, int y_hi) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const size_t i0 = (size_t)y * W + x4;
    uint8_t r[3][6];
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const int yy = y + j - 1;
      if (yy < 0 || yy >= H) {
#pragma unroll
        for (int k = 0; k < 6; k++) r[j][k] = 0;
      } else {
        const uint8_t *row = code + (size_t)yy * W + x4;
        const uchar4 m = *reinterpret_cast<const uchar4 *>(row);
        r[j][1] = m.x; r[j][2] = m.y; r[j][3] = m.z; r[j][4] = m.w;
        r[j][0] = x4 > 0 ? row[-1] : (uint8_t)0;
        r[j][5] = x4 + 4 < W ? row[4] : (uint8_t)0;
      }
    }
    unsigned long long out[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int cc = r[1][k + 1];
      if (y < y_lo || y >= y_hi) {  // ghost row of a row band: an empty parking slot
        out[k] = 0;
        continue;
      }
      if (cc == kCodeNoData) {
        out[k] = 0xBFF0000000000000ull;  // -1.0 (flow_accumulation_generic.hpp:95-97)
        continue;
      }
      const int nr[9] = {0, 1, 0, 0, 0, 1, 2, 2, 2};
      const int nc[9] = {0, k, k, k + 1, k + 2, k + 2, k + 2, k + 1, k};
      unsigned deps = 0;
      int dn = 0, dcode = 0;
#pragma unroll
      for (int n = 1; n <= 8; n++) {
        const int cn = r[nr[n]][nc[n]];
        if ((cn & 15) == 0 || cn == kCodeNoData) continue;
        if ((cn & 15) == d8_inverse(n)) {
          deps++;
          dn = n;
          dcode = cn;
        }
      }
      out[k] = deps == 0 ? kPkSource : (((unsigned long long)deps << 56) | 1ull);
      if (deps == 1) code[(size_t)(y + d8dy(dn)) * W + (x4 + k + d8dx(dn))] = (uint8_t)(dcode | kCodeSole);
    }
    reinterpret_cast<ulonglong2 *>(word + i0)[0] = make_ulonglong2(out[0], out[1]);
    reinterpret_cast<ulonglong2 *>(word + i0)[1] = make_ulonglong2(out[2], out[3]);
  }
}

// Fused replacement of flow_code_d8_x4_kernel + deps_gather_packed_x4_kernel (accum_fused_prep = 1):
// ONE pass over the DEM with a rolling row window.  A block owns 1024 columns (4 per thread, the
// outer 4 on each side are halo: blocks overlap by 8 columns) and walks down a chunk of rows.  Per
// row step g it (A) loads DEM row g+1 (one float4 per thread, neighbours by shuffle) and computes
// the flow codes of row g into a 5-row ring in shared memory, (B) counts the donors of row g-1 from
// the code rows g-2..g into a 4-row ring, and (C) writes row g-2: the packed word from its donor
// count, and its code byte with the sole-donor bit looked up at the receiver (rows g-3..g-1 of the
// rings).  Every DEM row is fetched once per block, all stores are coalesced, and the scattered
// one-byte sole-donor marks of the two-pass version disappear: 4 B read + 9 B written per cell.
constexpr int kPrepCols = 1024;
constexpr int kPrepOut = kPrepCols - 8;
constexpr int kPrepRows = 64;

__global__ void __launch_bounds__(256) fa_d8_prep_rolling_kernel(const float *__restrict__ dem, uint8_t *__restrict__ code,
                                                                  unsigned long long *__restrict__ word, int W, int H,
                                                                  float nodata, int y_lo, int y_hi) {
  // Row bands (y_lo > 0 / y_hi < H): rows outside [y_lo, y_hi) are ghost rows.  Their flow codes are NOT computed here
  // (the row beyond them is unknown): `code` already holds the neighbouring band's codes for them, they are read back
  // in step A, their words become empty parking slots and they are never a sole-donor target.
  // ring rows carry 4 guard bytes on each side (column c of the block lives at byte c + 4)
  __shared__ __align__(16) uint8_t sCode[5][kPrepCols + 8];
  __shared__ __align__(16) uint8_t sDeps[4][kPrepCols + 8];
  const unsigned full = 0xffffffffu;
  const int t = threadIdx.x, lane = t & 31;
  const int xc = (int)blockIdx.x * kPrepOut - 4 + 4 * t;  // first of this thread's 4 columns
  const int y0 = (int)blockIdx.y * kPrepRows;
  const bool col_in = xc >= 0 && xc < W;  // W % 4 == 0: the 4 columns are inside or outside together
  const bool writer = t >= 1 && t <= 254 && col_in;
  if (t < 4) {
#pragma unroll
    for (int r = 0; r < 5; r++) sCode[r][t] = sCode[r][kPrepCols + 4 + t] = 0;
#pragma unroll
    for (int r = 0; r < 4; r++) sDeps[r][t] = sDeps[r][kPrepCols + 4 + t] = 0;
  }
  // DEM rows g-1, g, g+1 ; columns xc-1 .. xc+4.  NoData cells are held as NaN -- as a neighbour a NaN fails every
  // comparison of the steepest-descent scan, which is exactly "skip NoData neighbours" -- and remembered in a bit mask
  // per row for the cell's own NoData test (a NaN that is data, or a NaN NoData value, keeps the reference's behaviour:
  // `== nodata` is false for it).
  float d[3][6];
  unsigned ndm[3];
  const float kNaN = __int_as_float(0x7fc00000);
  auto load_row = [&](int gy, float(&o)[6], unsigned &mask) {
    const bool rin = gy >= 0 && gy < H;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rin && col_in) m = __ldg(reinterpret_cast<const float4 *>(dem + (size_t)gy * W + xc));
    float left = __shfl_up_sync(full, m.w, 1), right = __shfl_down_sync(full, m.x, 1);
    if (lane == 0) left = (rin && xc - 1 >= 0 && xc - 1 < W) ? __ldg(dem + (size_t)gy * W + xc - 1) : 0.f;
    if (lane == 31) right = (rin && xc + 4 >= 0 && xc + 4 < W) ? __ldg(dem + (size_t)gy * W + xc + 4) : 0.f;
    const float in[6] = {left, m.x, m.y, m.z, m.w, right};
    mask = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) {
      const bool nd = in[k] == nodata;
      o[k] = nd ? kNaN : in[k];
      if (k >= 1 && k <= 4 && nd) mask |= 1u << k;
    }
  };
  load_row(y0 - 3, d[0], ndm[0]);
  load_row(y0 - 2, d[1], ndm[1]);
  for (int g = y0 - 2; g <= y0 + kPrepRows + 1; g++) {
    if (g - 2 >= H) break;  // no row left to write (uniform across the block)
    load_row(g + 1, d[2], ndm[2]);
    // ---- A: flow codes of row g (same per-cell rule as flow_code_d8_x4_kernel) ----
    {
      uint8_t cd[4];
      const bool row_in = g >= 0 && g < H;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int x = xc + k;
        const float e = d[1][k + 1];
        int c = 0;
        if (row_in && col_in && (g < y_lo || g >= y_hi)) {
          c = code[(size_t)g * W + x];  // a neighbouring band's row: its codes were installed by the caller
        } else if (row_in && col_in) {
          if (ndm[1] & (1u << (k + 1))) {
            c = kCodeNoData;
          } else if (!(x == 0 || g == 0 || x == W - 1 || g == H - 1)) {
            // neighbours n = 1..8 : W, NW, N, NE, E, SE, S, SW.  The first strictly lowest neighbour below the cell
            // wins: starting the running minimum at the cell's own value folds the reference's `>= e` skip into it
            // (capped at FLT_MAX, the reference's starting value, which only matters for an infinite cell)
            const float ne[9] = {0.f, d[1][k], d[0][k], d[0][k + 1], d[0][k + 2], d[1][k + 2], d[2][k + 2], d[2][k + 1], d[2][k]};
            float lowest = fminf(e, 3.402823466e+38f);
#pragma unroll
            for (int n = 1; n <= 8; n++) {
              const float v = ne[n];
              if (v < lowest) {
                lowest = v;
                c = n;
              }
            }
          }
        }
        cd[k] = (uint8_t)c;
      }
      *reinterpret_cast<uchar4 *>(&sCode[(g + 10) % 5][4 + 4 * t]) = make_uchar4(cd[0], cd[1], cd[2], cd[3]);
#pragma unroll
      for (int k = 0; k < 6; k++) {
        d[0][k] = d[1][k];
        d[1][k] = d[2][k];
      }
      ndm[0] = ndm[1];
      ndm[1] = ndm[2];
    }
    __syncthreads();
    // ---- B: donors of row g-1 from code rows g-2, g-1, g, four cells at a time on packed bytes ----
    if (g >= y0) {
      // m[j]: this thread's 4 codes of row g-2+j; wl / wr: the same row seen one column to the left / right
      uint32_t m[3], wl[3], wr[3];
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const uint8_t *row = &sCode[(g - 2 + j + 10) % 5][4 + 4 * t];
        m[j] = *reinterpret_cast<const uint32_t *>(row);
        wl[j] = (m[j] << 8) | (uint32_t)row[-1];
        wr[j] = (m[j] >> 8) | ((uint32_t)row[4] << 24);
      }
      // byte k of the result is 1 where the neighbour's direction (low 4 bits; NoData 255 -> 15 and "no flow" 0 never
      // equal an inverse direction) points back at cell k: x is 0..15 per byte, x + 0x7f sets bit 7 exactly where x != 0
      auto points_back = [](uint32_t w, uint32_t inv) -> uint32_t {
        const uint32_t x = (w & 0x0f0f0f0fu) ^ (inv * 0x01010101u);
        return (~(x + 0x7f7f7f7fu) & 0x80808080u) >> 7;
      };
      // neighbours n = 1..8 : W, NW, N, NE, E, SE, S, SW, each against d8_inverse(n) = 5, 6, 7, 8, 1, 2, 3, 4
      const uint32_t deps4 = points_back(wl[1], 5) + points_back(wl[0], 6) + points_back(m[0], 7) + points_back(wr[0], 8) +
                             points_back(wr[1], 1) + points_back(wr[2], 2) + points_back(m[2], 3) + points_back(wl[2], 4);
      *reinterpret_cast<uint32_t *>(&sDeps[(g - 1 + 8) % 4][4 + 4 * t]) = deps4;
    }
    __syncthreads();
    // ---- C: write row g-2 ----
    if (g >= y0 + 2 && writer) {
      const int yy = g - 2;
      const uchar4 c4 = *reinterpret_cast<const uchar4 *>(&sCode[(yy + 10) % 5][4 + 4 * t]);
      const uchar4 d4 = *reinterpret_cast<const uchar4 *>(&sDeps[(yy + 8) % 4][4 + 4 * t]);
      int cc[4] = {c4.x, c4.y, c4.z, c4.w};
      const int dd[4] = {d4.x, d4.y, d4.z, d4.w};
      unsigned long long out[4];
      const bool ghost = yy < y_lo || yy >= y_hi;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        if (ghost) {
          out[k] = 0;  // an empty parking slot for flow that leaves the band
          continue;
        }
        if (cc[k] == kCodeNoData) {
          out[k] = 0xBFF0000000000000ull;  // -1.0 (flow_accumulation_generic.hpp:95-97)
          continue;
        }
        out[k] = dd[k] == 0 ? kPkSource : (((unsigned long long)dd[k] << 56) | 1ull);
        if (dd[k] == 0) cc[k] |= kCodeSource;
        const int dir = cc[k] & 15;
        if (dir != 0) {
          const int ry = yy + d8dy(dir), ro = 4 + 4 * t + k + d8dx(dir);
          const int rc = sCode[(ry + 10) % 5][ro];
          // I am my receiver's only donor (a receiver in a ghost row is a parking slot that several bands' worth of
          // cells may add to: never "sole")
          if (rc != kCodeNoData && sDeps[(ry + 8) % 4][ro] == 1 && ry >= y_lo && ry < y_hi) cc[k] |= kCodeSole;
        }
      }
      const size_t i0 = (size_t)yy * W + xc;
      if (!ghost)
        *reinterpret_cast<uchar4 *>(code + i0) = make_uchar4((uint8_t)cc[0], (uint8_t)cc[1], (uint8_t)cc[2], (uint8_t)cc[3]);
      reinterpret_cast<ulonglong2 *>(word + i0)[0] = make_ulonglong2(out[0], out[1]);
      reinterpret_cast<ulonglong2 *>(word + i0)[1] = make_ulonglong2(out[2], out[3]);
    }
  }
}

// flow codes of single rows (the first / last owned row of a row band, which the neighbouring band needs before it
// can count the donors of its own edge row)
__global__ void __launch_bounds__(256) flow_code_rows_kernel(const float *__restrict__ dem, uint8_t *__restrict__ code, int W,
                                                              int H, float nodata, int ya, int yb) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int y = blockIdx.y == 0 ? ya : yb;
  if (y < 0) return;
  code[(size_t)y * W + x] = (uint8_t)fm_d8_cell(dem, x, y, W, H, nodata);
}

// BAND: cells below ghost_lo_end / from ghost_hi_start on belong to a neighbouring row band; flow
// into them is parked in their word as [parcel count | sum] for the caller to ship.  `frontier`
// (optional) lists cells completed by a neighbour's flow; their word already holds the final double.
template <bool BAND>
__global__ void __launch_bounds__(256) accum_walk_packed_kernel(const uint8_t *__restrict__ code, unsigned long long *word,
                                                                 int W, int ncells, const int *__restrict__ frontier,
                                                                 int ghost_lo_end, int ghost_hi_start) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ncells) return;
  int c;
  unsigned long long acc;
  if (BAND && frontier) {
    c = frontier[t];
    acc = (unsigned long long)__longlong_as_double((long long)word[c]);
  } else {
    c = t;
    if (word[c] != kPkSource) return;
    acc = 1;
    word[c] = (unsigned long long)__double_as_longlong(1.0);
  }
  for (;;) {
    const int cdraw = code[c];
    const int cd = cdraw & 15;
    if (cdraw == kCodeNoData || cd == 0) break;
    const int r = c + d8dy(cd) * W + d8dx(cd);
    unsigned long long total;
    if (cdraw & kCodeSole) {
      total = acc + 1;  // the receiver holds its own unit and waits for me alone
    } else {
      if (code[r] == kCodeNoData) break;  // flow into NoData is dropped (FM_D8 never produces it)
      if (BAND && (r < ghost_lo_end || r >= ghost_hi_start)) {
        atomicAdd(word + r, acc + kPkOne);  // one more parcel, `acc` more flow
        break;
      }
      const unsigned long long old = atomicAdd(word + r, acc - kPkOne);
      if ((old >> 56) != 1ull) break;     // other donors are still to come: the last one carries on
      total = (old & kPkVal) + acc;
    }
    word[r] = (unsigned long long)__double_as_longlong((double)total);
    acc = total;
    c = r;
  }
}
// Same walk with persistent, always-busy lanes (accum_walk_lanes = 1).  In the kernel above a thread
// that is not a source exits at once and a walk ends as soon as its thread is not the last donor, so
// most resident warps hold one or two live lanes and the walk is bound by how few dependent atomics
// are in flight.  Here a warp pulls chunks of cells from a global cursor, compacts their sources
// (ballot + popc) into a small queue in shared memory, and every lane whose walk has ended takes
// the next source from that queue; the loop body is one converged walk step for all 32 lanes.
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

constexpr int kLaneQueue = 256;   // per-warp source queue (power of two, >= 160: a refill adds up to 128 cells)

// `src_in_code`: the preparation marked the cells without donors with kCodeSource in their code byte (the fused
// preparation does), so the source scan reads 1 B/cell -- four cells per lane and load -- instead of the 8 B words.
// A walking lane holds the code byte of its cell: the receiver's byte is fetched while the atomic on the receiver's
// word is in flight (flow codes of this path never point at NoData -- the steepest-descent rule skips NoData
// neighbours -- so nothing has to be known about the receiver before the add), which takes one of the two dependent
// memory round trips out of every step.
template <bool BAND>
__global__ void __launch_bounds__(256) accum_walk_packed_lanes_kernel(const uint8_t *__restrict__ code,
                                                                       unsigned long long *word, int W, int ncells,
                                                                       const int *__restrict__ frontier, int ghost_lo_end,
                                                                       int ghost_hi_start, int *cursor, int src_in_code,
                                                                       int ahead) {
  __shared__ int sQ[8][kLaneQueue];
  __shared__ uint8_t sQc[8][kLaneQueue];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  int *q = sQ[threadIdx.x >> 5];
  uint8_t *qc = sQc[threadIdx.x >> 5];
  const unsigned lt = (1u << lane) - 1u;
  const bool listed = BAND && frontier;
  const int per_lane = (!listed && src_in_code) ? 4 : 1;  // candidates a lane looks at per refill step
  int head = 0, count = 0;           // warp-uniform queue state
  int pos = 0, end = 0;              // warp-uniform: next candidate, end of the current chunk
  bool more = true;                  // the cursor may still hold chunks
  bool walking = false;
  int c = 0, cdraw = 0;
  unsigned long long acc = 0;
  for (;;) {
    // ---- refill: keep `ahead` sources queued while candidates last -- no more: a source waits in the queue while the
    // words its walk will touch, fetched around the time it was scanned, sit in L2; with every warp a full queue ahead of
    // its walks those lines are gone again when they are needed ----
    while (count < ahead) {
      if (pos >= end) {
        if (!more) break;
        int b = 0;
        if (lane == 0) b = atomicAdd(cursor, kLaneChunk);
        b = __shfl_sync(full, b, 0);
        if (b >= ncells) {
          more = false;
          break;
        }
        pos = b;
        end = b + kLaneChunk < ncells ? b + kLaneChunk : ncells;
      }
      const int i = pos + per_lane * lane;
      unsigned flags = 0;            // bit k: candidate i + k is a source
      uint32_t bytes = 0;            // its code byte(s)
      int cell = i;
      if (i < end) {
        if (listed) {
          cell = frontier[i];
          bytes = code[cell];
          flags = 1;
        } else if (per_lane == 4) {  // chunks and ncells are multiples of 4 here (W % 4 == 0)
          // the walks that start here push into words of this and the neighbouring rows: have the 1 KB of words that
          // belong to these 128 cells on their way into L2 (the 8 B/cell scan used to do that as a side effect; without
          // it every first atomic on a line waits for DRAM) -- fire and forget, nothing depends on it
          if (src_in_code == 1 && lane < 8 && pos + 16 * lane < end) prefetch_l2(word + pos + 16 * lane);
          bytes = __ldg(reinterpret_cast<const uint32_t *>(code + i));
          // a source byte has kCodeSource (bit 6) set and is not NoData (255, the only value with bit 7)
          const uint32_t sb = (bytes >> 6) & ~(bytes >> 7) & 0x01010101u;
          flags = (sb & 1u) | ((sb >> 7) & 2u) | ((sb >> 14) & 4u) | ((sb >> 21) & 8u);
        } else if (word[i] == kPkSource) {
          bytes = code[i];
          flags = 1;
        }
      }
#pragma unroll
      for (int k = 0; k < 4; k++) {
        if (k >= per_lane) break;
        const bool src = (flags >> k) & 1u;
        const unsigned bal = __ballot_sync(full, src);
        if (src) {
          const int slot = (head + count + __popc(bal & lt)) & (kLaneQueue - 1);
          q[slot] = cell + k;
          qc[slot] = (uint8_t)(bytes >> (8 * k));
        }
        count += __popc(bal);
      }
      pos += 32 * per_lane;
    }
    __syncwarp();  // queue entries written above are read by other lanes below
    // ---- hand queued sources to the lanes that are not walking ----
    const unsigned idle = __ballot_sync(full, !walking);
    if (idle == full && count == 0 && !more && pos >= end) break;
    const int rank = __popc(idle & lt);
    if (!walking && rank < count) {
      const int slot = (head + rank) & (kLaneQueue - 1);
      c = q[slot];
      cdraw = qc[slot];
      if (listed) {
        acc = (unsigned long long)__longlong_as_double((long long)word[c]);  // completed by a neighbour's flow
      } else {
        acc = 1;
        word[c] = (unsigned long long)__double_as_longlong(1.0);
      }
      walking = true;
    }
    {
      const int nidle = __popc(idle);
      const int taken = nidle < count ? nidle : count;
      head = (head + taken) & (kLaneQueue - 1);
      count -= taken;
    }
    __syncwarp();  // everyone has read its queue slot before the next refill overwrites the ring
    // ---- one walk step ----
    if (walking) {
      const int cd = cdraw & 15;
      if (cdraw == kCodeNoData || cd == 0) {
        walking = false;
      } else {
        const int r = c + d8dy(cd) * W + d8dx(cd);
        const int cnext = code[r];  // in flight together with the atomic
        unsigned long long total = 0;
        if (cdraw & kCodeSole) {
          total = acc + 1;  // the receiver holds its own unit and waits for me alone
        } else if (BAND && (r < ghost_lo_end || r >= ghost_hi_start)) {
          atomicAdd(word + r, acc + kPkOne);  // park in the ghost row: one more parcel, `acc` more flow
          walking = false;
        } else {
          const unsigned long long old = atomicAdd(word + r, acc - kPkOne);
          if ((old >> 56) != 1ull) walking = false;  // other donors are still to come
          else total = (old & kPkVal) + acc;
        }
        if (walking) {
          word[r] = (unsigned long long)__double_as_longlong((double)total);
          acc = total;
          c = r;
          cdraw = cnext;
        }
      }
    }
  }
}

// =================================================================================================
// Unit-weight D-infinity on packed words (accum_dinf_packed, the default for FA_Tarboton without weights).
// The level-synchronous kernel needs ~7000 grid barriers at 32768^2 and, per cell, two double atomics, a fence and two
// counter atomics.  With unit weights every accumulation is a sum of products of proportions, so it is carried as a
// 56-bit fixed-point number (24 fractional bits) next to the 8-bit donor count, exactly like the D8 words:
//     [ 8 bits donors left | 56 bits sum * 2^24 ]
// A donor's single atomicAdd(word, share - 2^56) delivers its share AND tells it whether it was the last donor.  The
// walk has no levels: persistent lanes take sources from a per-warp queue; a lane follows the first receiver it completes
// and queues the second one.  A cell with two receivers sends each share rounded to the nearest 2^-24, off by <= 2^-25; a
// sole receiver gets the sum unrounded.  A cell may take up to 8 rounded shares however small its accumulation (a
// neighbour whose flow runs almost parallel to it sends it a share of ~1e-7), so the error of a cell c obeys
//     err(c) <= sum over donors d of p(d) err(d) + k(c) 2^-25,   k(c) <= 8 rounded shares taken,
// and as every accumulation is at least 1 (the cell's own unit), induction gives a relative error below 8 * 2^-25 =
// 2^-22 (~2.4e-7), against the 1e-5 the results are specified to.  Measured on an H100: 6.1e-8 at most on fBm and on the
// Beauford crop, 5.9e-8 on terrain searched for the worst case (tests/test_accum_exact.py, tools/dinf_packed_worst.py).
// The sums are integers, so the result does not depend on the order of the atomics.  Weighted accumulations keep the
// double-precision path.
// =================================================================================================
constexpr unsigned long long kFxOne = 1ull << 24;                    // one unit of flow
constexpr unsigned long long kFxSource = (1ull << 63) | kFxOne;      // no donors, own unit, not started yet
constexpr int kLaneQueueD = 256;                                      // per-warp ring (power of two)

// (row bands: rows outside [y_lo, y_hi) are ghost rows -- empty parking slots for the flow that leaves the band)
__global__ void __launch_bounds__(256) deps_gather_packed_dinf_x4_kernel(const uint8_t *__restrict__ code,
                                                                          unsigned long long *__restrict__ word, int W, int H,
                                                                          int y_lo, int y_hi) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const size_t i0 = (size_t)y * W + x4;
    uint8_t r[3][6];
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const int yy = y + j - 1;
      if (yy < 0 || yy >= H) {
#pragma unroll
        for (int k = 0; k < 6; k++) r[j][k] = 0;
      } else {
        const uint8_t *row = code + (size_t)yy * W + x4;
        const uchar4 m = *reinterpret_cast<const uchar4 *>(row);
        r[j][1] = m.x; r[j][2] = m.y; r[j][3] = m.z; r[j][4] = m.w;
        r[j][0] = x4 > 0 ? row[-1] : (uint8_t)0;
        r[j][5] = x4 + 4 < W ? row[4] : (uint8_t)0;
      }
    }
    unsigned long long out[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int cc = r[1][k + 1];
      if (y < y_lo || y >= y_hi) {
        out[k] = 0;
        continue;
      }
      if (cc == kCodeNoData) {
        out[k] = 0xBFF0000000000000ull;  // -1.0 (flow_accumulation_generic.hpp:95-97)
        continue;
      }
      const int nr[9] = {0, 1, 0, 0, 0, 1, 2, 2, 2};
      const int nc[9] = {0, k, k, k + 1, k + 2, k + 2, k + 2, k + 1, k};
      unsigned deps = 0;
#pragma unroll
      for (int n = 1; n <= 8; n++) {
        const int cn = r[nr[n]][nc[n]];
        if ((cn & 15) == 0 || cn == kCodeNoData) continue;
        const int inv = d8_inverse(n);
        const int first = cn & 15;
        if (first == inv || ((cn & kCodeTwo) && nwrap(first + 1) == inv)) deps++;
      }
      out[k] = deps == 0 ? kFxSource : (((unsigned long long)deps << 56) | kFxOne);
    }
    reinterpret_cast<ulonglong2 *>(word + i0)[0] = make_ulonglong2(out[0], out[1]);
    reinterpret_cast<ulonglong2 *>(word + i0)[1] = make_ulonglong2(out[2], out[3]);
  }
}

__device__ __forceinline__ double fx_to_double(unsigned long long fx) { return (double)fx * (1.0 / 16777216.0); }

// Work sharing.  A lane follows the first receiver it completes; a second one goes to its warp's ring in shared memory,
// where idle lanes of the warp pick it up.  What a warp completes stays with that warp, so after the source scan the
// remaining work -- the big rivers and the resolved lakes -- sits with the few warps that happened to complete their
// upstream ends: measured at 32768^2 after flat resolution, one warp walked 115 000 iterations at 30 busy lanes while
// 7 000 warps had nothing to do (470 ms), and routing the hand-overs through a global ticket queue that every idle warp
// polls cost more than it saved (3.8 s with most hand-overs shared).  So the work is rebalanced by stopping the world
// instead: the kernel runs in PHASES separated by grid barriers.  A warp that has nothing left waits at the barrier; a
// warp that holds more cells than it has lanes for (`excess_above` queued) while a quarter of the warps wait there asks
// for the phase to end; every warp then appends what it holds -- ring entries and the cells its lanes stand on -- to a
// list in global memory, and after the barrier all warps draw from that list in equal portions (a cell's fixed-point
// sum is recovered from its final double).  The walk is over when a phase ends with an empty list.  No warp polls a
// shared line while it works except one read every 16 iterations.
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct alignas(16) DinfShare {
  int cursor;          // source scan
  int n_data;          // cells that have to be walked (every cell that is not NoData)
  int n_noflow;        // data cells without a receiver (flat cells of an unresolved DEM, raster edge)
  int done;            // cells walked, reported at the end of every phase (checked by the host)
  unsigned list_head;  // hand-over list: entries claimed
  unsigned list_tail;  //                 entries appended
  unsigned cons_end;   //                 [list_head, cons_end) may be claimed in the current phase
  int quota;           // entries a warp claims at a time in the current phase
  int stop;            // a warp asked for phase `stop - 1` to end
  int n_waiting;       // warps at the barrier
  int finished;        // the phase ended with an empty list
  int phases;          // statistics
};

__global__ void __launch_bounds__(256) dinf_count_data_kernel(const uint8_t *__restrict__ code, size_t n, DinfShare *sh) {
  int k = 0, z = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int cd = code[i];
    k += cd != kCodeNoData;
    z += cd == 0;
  }
  for (int o = 16; o > 0; o >>= 1) {
    k += __shfl_xor_sync(0xffffffffu, k, o);
    z += __shfl_xor_sync(0xffffffffu, z, o);
  }
  __shared__ int sk[2][8];
  if ((threadIdx.x & 31) == 0) {
    sk[0][threadIdx.x >> 5] = k;
    sk[1][threadIdx.x >> 5] = z;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    int t = 0;
    for (int w = 0; w < 8; w++) t += sk[threadIdx.x][w];
    if (t) atomicAdd(threadIdx.x == 0 ? &sh->n_data : &sh->n_noflow, t);
  }
}

template <bool STATS>
__global__ void __launch_bounds__(256, 6) accum_walk_dinf_lanes_kernel(const uint8_t *__restrict__ code,
                                                                     const float *__restrict__ rmaxArr,
                                                                     unsigned long long *word, int W, int ncells, int *list,
                                                                     unsigned cap, DinfShare *sh, int excess_above,
                                                                     int wait_div, unsigned long long *stats, int ghost_lo_end,
                                                                     int ghost_hi_start, int seeded) {
  cg::grid_group grid = cg::this_grid();
  __shared__ int sQ[8][kLaneQueueD];
  __shared__ unsigned long long sQa[8][kLaneQueueD];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  int *q = sQ[threadIdx.x >> 5];
  unsigned long long *qa = sQa[threadIdx.x >> 5];
  const unsigned lt = (1u << lane) - 1u;
  const int n_warps = (int)gridDim.x * 8;
  int head = 0, count = 0;        // warp-uniform ring state
  int pos = 0, end = 0;           // warp-uniform: next source candidate, end of the current chunk
  // Row bands: cells below ghost_lo_end / from ghost_hi_start on belong to a neighbouring band; flow into them is parked in
  // their word as [parcels | sum] for the caller to ship.  `seeded`: no source scan, the list already holds the cells an
  // inflow completed (the host put their number into list_tail / cons_end and a portion into quota).
  bool more = seeded == 0;        // the source cursor may still hold chunks
  int walked = 0;                 // warp-uniform: cells walked since the last report
  bool walking = false;
  int c = 0;
  unsigned long long acc = 0;
  int phase = 0, quota = 0;
  unsigned cons_end = 0;
  bool list_dry = true;           // nothing to claim from the list in this phase (phase 0: the list is empty)
  if (seeded) {
    quota = *reinterpret_cast<volatile int *>(&sh->quota);
    cons_end = *reinterpret_cast<volatile unsigned *>(&sh->cons_end);
    list_dry = false;
  }
  // optional counters (accum_dinf_stats): what the warps spent their loop iterations on
  unsigned long long st_iters = 0, st_steps = 0, st_list = 0, st_loc = 0, st_got = 0;
  for (;;) {  // phases
    unsigned iter = 0;
    for (;;) {  // iterations of this phase
      iter++;
      if (STATS) st_iters++;
      // ---- sources: refill from the scan only when the lanes would otherwise starve ----
      while (count < 32 && (more || pos < end)) {
        if (pos >= end) {
          int b = 0;
          if (lane == 0) b = atomicAdd(&sh->cursor, kLaneChunk);
          b = __shfl_sync(full, b, 0);
          if (b >= ncells) {
            more = false;
            break;
          }
          pos = b;
          end = b + kLaneChunk < ncells ? b + kLaneChunk : ncells;
        }
        const int i = pos + lane;
        const bool src = i < end && word[i] == kFxSource;
        const unsigned bal = __ballot_sync(full, src);
        if (src) {
          const int slot = (head + count + __popc(bal & lt)) & (kLaneQueueD - 1);
          q[slot] = i;
          qa[slot] = kFxOne;
          word[i] = (unsigned long long)__double_as_longlong(1.0);
        }
        count += __popc(bal);
        pos += 32;
      }
      // ---- the hand-over list of this phase: a warp with lanes it cannot feed claims its portion ----
      const int hungry = __popc(__ballot_sync(full, !walking));
      if (!list_dry && !more && pos >= end && count < hungry) {
        unsigned h = 0;
        if (lane == 0) h = atomicAdd(&sh->list_head, (unsigned)quota);
        h = __shfl_sync(full, h, 0);
        const int avail = (int)(cons_end - h);
        if (avail <= 0) {
          list_dry = true;
        } else {
          const int k = avail < quota ? avail : quota;
          if (lane < k) {
            const int cell = __ldcg(list + (h + (unsigned)lane) % cap);
            const int slot = (head + count + lane) & (kLaneQueueD - 1);
            q[slot] = cell;
            qa[slot] = (unsigned long long)(__longlong_as_double((long long)__ldcg(word + cell)) * 16777216.0 + 0.5);
          }
          count += k;
          if (STATS) st_got += k;
        }
      }
      __syncwarp();
      // ---- hand queued cells to the lanes that are not walking ----
      const unsigned idle = __ballot_sync(full, !walking);
      const int rank = __popc(idle & lt);
      if (!walking && rank < count) {
        const int slot = (head + rank) & (kLaneQueueD - 1);
        c = q[slot];
        acc = qa[slot];
        walking = true;
      }
      {
        const int nidle = __popc(idle);
        const int taken = nidle < count ? nidle : count;
        head = (head + taken) & (kLaneQueueD - 1);
        count -= taken;
      }
      __syncwarp();
      const unsigned busy = __ballot_sync(full, walking);
      if (busy == 0) {
        if (!more && pos >= end && list_dry) break;  // nothing left for this warp in this phase
        continue;
      }
      // ---- has the end of the phase been asked for?  shall this warp ask? ----
      if ((iter & 15u) == 0) {
        int st = 0;
        if (lane == 0) {
          st = *reinterpret_cast<volatile int *>(&sh->stop) > phase ? 1 : 0;
          if (!st && count >= excess_above && (iter >= 64u || count >= kLaneQueueD - 64) &&
              *reinterpret_cast<volatile int *>(&sh->n_waiting) * wait_div >= n_warps) {
            atomicMax(&sh->stop, phase + 1);
            st = 1;
          }
        }
        st = __shfl_sync(full, st, 0);
        if (st) break;
      }
      // ---- one walk step: push this cell's flow to its receiver(s) ----
      walked += __popc(busy);
      if (STATS) st_steps += __popc(busy);
      int extra = -1;  // a second receiver completed by this lane in this step
      unsigned long long extra_acc = 0;
      if (walking) {
        const int cd = code[c];
        const int n1 = cd & 15;
        if (cd == kCodeNoData || n1 == 0) {
          walking = false;
        } else {
          const int r1 = c + d8dy(n1) * W + d8dx(n1);
          int next = -1;
          unsigned long long next_acc = 0;
          if (cd & kCodeTwo) {
            const int n2 = nwrap(n1 + 1);
            const int r2 = c + d8dy(n2) * W + d8dx(n2);
            float p1, p2;
            tarboton_props(rmaxArr[c], &p1, &p2);
            const double ad = (double)acc;
            const unsigned long long v1 = p1 > 0 ? (unsigned long long)((double)p1 * ad + 0.5) : 0ull;
            const unsigned long long v2 = p2 > 0 ? (unsigned long long)((double)p2 * ad + 0.5) : 0ull;
            if (p1 > 0) {
              if (r1 < ghost_lo_end || r1 >= ghost_hi_start) {
                atomicAdd(word + r1, v1 + kPkOne);  // park: one more parcel, v1 more flow
              } else {
                const unsigned long long old = atomicAdd(word + r1, v1 - kPkOne);
                if ((old >> 56) == 1ull) {
                  next = r1;
                  next_acc = (old & kPkVal) + v1;
                }
              }
            }
            if (p2 > 0 && (r2 < ghost_lo_end || r2 >= ghost_hi_start)) {
              atomicAdd(word + r2, v2 + kPkOne);
            } else if (p2 > 0) {
              const unsigned long long old = atomicAdd(word + r2, v2 - kPkOne);
              if ((old >> 56) == 1ull) {
                const unsigned long long tot = (old & kPkVal) + v2;
                if (next < 0) {
                  next = r2;
                  next_acc = tot;
                } else {
                  extra = r2;
                  extra_acc = tot;
                }
              }
            }
          } else if (r1 < ghost_lo_end || r1 >= ghost_hi_start) {
            atomicAdd(word + r1, acc + kPkOne);
          } else {
            const unsigned long long old = atomicAdd(word + r1, acc - kPkOne);
            if ((old >> 56) == 1ull) {
              next = r1;
              next_acc = (old & kPkVal) + acc;
            }
          }
          if (next >= 0) {
            word[next] = (unsigned long long)__double_as_longlong(fx_to_double(next_acc));
            c = next;
            acc = next_acc;
          } else {
            walking = false;
          }
          if (extra >= 0) word[extra] = (unsigned long long)__double_as_longlong(fx_to_double(extra_acc));
        }
      }
      // ---- hand-overs: to the warp's ring; what the ring cannot take goes straight to the list of the next phase ----
      {
        const unsigned pb = __ballot_sync(full, extra >= 0);
        if (pb) {
          const int k = __popc(pb & lt), np = __popc(pb);
          const int room = kLaneQueueD - 32 - count;
          const int local = np < room ? np : (room > 0 ? room : 0);
          unsigned gbase = 0;
          if (np > local) {
            if (lane == 0) gbase = atomicAdd(&sh->list_tail, (unsigned)(np - local));
            gbase = __shfl_sync(full, gbase, 0);
          }
          if (extra >= 0) {
            if (k < local) {
              const int slot = (head + count + k) & (kLaneQueueD - 1);
              q[slot] = extra;
              qa[slot] = extra_acc;
            } else {
              list[(gbase + (unsigned)(k - local)) % cap] = extra;
            }
          }
          count += local;
          if (STATS) {
            st_list += np - local;
            st_loc += local;
          }
        }
      }
    }
    // ---- end of the phase for this warp: everything it holds goes to the list ----
    {
      const unsigned wb = __ballot_sync(full, walking);
      const int total = count + __popc(wb);
      if (total) {
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(&sh->list_tail, (unsigned)total);
        base = __shfl_sync(full, base, 0);
        for (int j = lane; j < count; j += 32) list[(base + (unsigned)j) % cap] = q[(head + j) & (kLaneQueueD - 1)];
        if (walking) list[(base + (unsigned)(count + __popc(wb & lt))) % cap] = c;
        if (STATS) st_list += total;
      }
      if (lane == 0) {
        if (walked) atomicAdd(&sh->done, walked);
        atomicAdd(&sh->n_waiting, 1);
      }
      walked = 0;
      count = 0;
      head = 0;
      walking = false;
      __threadfence();
    }
    grid.sync();
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      unsigned hd = sh->list_head;
      const unsigned ce = sh->cons_end, tl = sh->list_tail;
      if ((int)(hd - ce) > 0) hd = ce;  // claims past the end of the last portion
      const unsigned left = tl - hd;
      int qv = (int)((left + (unsigned)n_warps - 1u) / (unsigned)n_warps);
      sh->list_head = hd;
      sh->cons_end = tl;
      sh->quota = qv < 1 ? 1 : (qv > 32 ? 32 : qv);
      sh->n_waiting = 0;
      sh->finished = left == 0 ? 1 : 0;
      sh->phases = phase + 1;
      __threadfence();
    }
    grid.sync();
    phase++;
    if (*reinterpret_cast<volatile int *>(&sh->finished)) break;
    quota = *reinterpret_cast<volatile int *>(&sh->quota);
    cons_end = *reinterpret_cast<volatile unsigned *>(&sh->cons_end);
    list_dry = false;
  }
  if (STATS && lane == 0) {
    atomicAdd(stats + 0, st_iters);
    atomicAdd(stats + 2, st_steps);
    atomicMax(stats + 3, st_iters);
    atomicAdd(stats + 4, 1ull);
    atomicAdd(stats + 6, st_got);
    atomicAdd(stats + 7, st_list);
    atomicAdd(stats + 8, st_loc);
  }
}

// seeds the shared block for a walk from a list of cells (row bands: the cells an inflow completed)
__global__ void dinf_share_seed_kernel(DinfShare *sh, int n_list, int n_warps, int ncells) {
  sh->cursor = ncells;
  sh->done = 0;
  sh->list_head = 0;
  sh->list_tail = (unsigned)n_list;
  sh->cons_end = (unsigned)n_list;
  const int q = (n_list + n_warps - 1) / n_warps;
  sh->quota = q < 1 ? 1 : (q > 32 ? 32 : q);
  sh->stop = 0;
  sh->n_waiting = 0;
  sh->finished = 0;
  sh->phases = 0;
}

// Queues the packed D-infinity walk on the library's stream (a cooperative launch: the phases meet at grid barriers, so
// every block has to be resident).  seeded < 0: sources come from the scan over the words (`share` zeroed by the caller,
// or holding the cell counts); seeded >= 0: the first `seeded` entries of `list` are the cells to start from.
void launch_walk_dinf(const uint8_t *code, const float *rmax, unsigned long long *word, int W, int ncells, int *list,
                      DinfShare *share, unsigned long long *stats, int ghost_lo_end, int ghost_hi_start, int seeded) {
  Ctx &c = ctx();
  int per_sm = 0;
  if (stats) RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, accum_walk_dinf_lanes_kernel<true>, 256, 0));
  else RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, accum_walk_dinf_lanes_kernel<false>, 256, 0));
  if (per_sm < 1) per_sm = 1;
  long long nb = (long long)c.num_sms * per_sm;
  const long long work = seeded >= 0 ? ((long long)seeded + 31) / 32 : ((long long)ncells + kLaneChunk - 1) / kLaneChunk;
  if (nb * 8 > work) nb = (work + 7) / 8;  // no more warps than chunks of sources / than warps' worth of listed cells
  // (a listed cell may be the head of a river through the whole band: keep a block per SM for the phases to spread it over)
  if (seeded >= 0 && nb < c.num_sms) nb = c.num_sms;
  if (nb < 1) nb = 1;
  if (seeded >= 0) {
    dinf_share_seed_kernel<<<1, 1, 0, c.stream>>>(share, seeded, (int)nb * 8, ncells);
    RDB_CK(cudaGetLastError());
  }
  const uint8_t *a_code = code;
  const float *a_rmax = rmax;
  int a_w = W, a_n = ncells;
  int *a_list = list;
  unsigned a_cap = (unsigned)ncells;
  DinfShare *a_sh = share;
  int a_excess = (int)(c.params.accum_dinf_share >= 0 ? c.params.accum_dinf_share : 1);  // measured at 32768^2 after flat resolution: 0 / 1 / 2 / 4 / 8 -> 140 / 135 / 141 / 185 / 189 ms
  int a_wait = (int)(c.params.accum_dinf_wait > 0 ? c.params.accum_dinf_wait : 4);  // 1 / this share of the warps waiting
  if (a_excess > kLaneQueueD - 96) a_excess = kLaneQueueD - 96;
  unsigned long long *a_stats = stats;
  int a_lo = ghost_lo_end, a_hi = ghost_hi_start, a_seeded = seeded >= 0 ? 1 : 0;
  void *args[] = {(void *)&a_code, (void *)&a_rmax, (void *)&word, (void *)&a_w, (void *)&a_n, (void *)&a_list, (void *)&a_cap,
                  (void *)&a_sh, (void *)&a_excess, (void *)&a_wait, (void *)&a_stats, (void *)&a_lo, (void *)&a_hi, (void *)&a_seeded};
  if (stats)
    RDB_CK(cudaLaunchCooperativeKernel((const void *)accum_walk_dinf_lanes_kernel<true>, dim3((unsigned)nb), dim3(256), args, 0, c.stream));
  else
    RDB_CK(cudaLaunchCooperativeKernel((const void *)accum_walk_dinf_lanes_kernel<false>, dim3((unsigned)nb), dim3(256), args, 0, c.stream));
  RDB_CK(cudaGetLastError());
}

// `cursor_buf` (optional): a device int the caller owns; the launch is then left in flight (no stream sync)
template <bool BAND>
void launch_walk_packed(const uint8_t *code, unsigned long long *word, int W, int ncells, const int *frontier,
                        int ghost_lo_end, int ghost_hi_start, bool src_in_code, int *cursor_buf = nullptr) {
  Ctx &c = ctx();
  if (ncells <= 0) return;
  if (c.params.accum_walk_lanes) {
    DevBuf<int> cursor;
    if (!cursor_buf) cursor.alloc(1);
    int *cur = cursor_buf ? cursor_buf : cursor.p;
    RDB_CK(cudaMemsetAsync(cur, 0, sizeof(int), c.stream));
    int per_sm = 0;
    RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, accum_walk_packed_lanes_kernel<BAND>, 256, 0));
    if (per_sm < 1) per_sm = 1;
    long long blocks = (long long)c.num_sms * per_sm;
    const long long need = ((long long)ncells + kLaneChunk - 1) / kLaneChunk;  // no more warps than chunks
    if (blocks * 8 > need) blocks = (need + 7) / 8;
    // accum_walk_scan: 0 (default) scan the 8 B words for sources, 1 scan the flagged code bytes and prefetch the words, 2 no prefetch.
    // The byte scan moves 7 B/cell less and still loses 3.5 ms at 32768^2: the word scan is what brings the lines the walks
    // are about to hit with atomics into L2, and a prefetch instruction does not replace it.
    const int in_code = src_in_code && c.params.accum_walk_scan && (ncells & 3) == 0 && ((uintptr_t)code & 3) == 0 ? (int)c.params.accum_walk_scan : 0;
    int ahead = (int)(c.params.accum_walk_ahead > 0 ? c.params.accum_walk_ahead : 64);
    if (ahead > kLaneQueue - 128) ahead = kLaneQueue - 128;  // one refill step adds up to 128 cells
    if (ahead < 32) ahead = 32;
    accum_walk_packed_lanes_kernel<BAND><<<(unsigned)blocks, 256, 0, c.stream>>>(code, word, W, ncells, frontier, ghost_lo_end,
                                                                               ghost_hi_start, cur, in_code, ahead);
    RDB_CK(cudaGetLastError());
    if (!cursor_buf) RDB_CK(cudaStreamSynchronize(c.stream));  // `cursor` goes out of scope
  } else {
    accum_walk_packed_kernel<BAND><<<(unsigned)((ncells + 255) / 256), 256, 0, c.stream>>>(code, word, W, ncells, frontier,
                                                                                        ghost_lo_end, ghost_hi_start);
  }
}

// packed ghost row -> (sum, parcels) rows for shipping; clears the slots; counts the parcels
__global__ void __launch_bounds__(256) band_take_packed_kernel(unsigned long long *ghost, double *sum, int *cnt, int W,
                                                                int *total) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  int k = 0;
  if (x < W) {
    const unsigned long long wv = ghost[x];
    k = (int)(wv >> 56);
    sum[x] = (double)(wv & kPkVal);
    cnt[x] = k;
    ghost[x] = 0;
  }
  for (int o = 16; o > 0; o >>= 1) k += __shfl_down_sync(0xffffffffu, k, o);
  if ((threadIdx.x & 31) == 0 && k) atomicAdd(total, k);
}

__global__ void __launch_bounds__(256) band_count_packed_kernel(const unsigned long long *__restrict__ gtop,
                                                                 const unsigned long long *__restrict__ gbot, int W,
                                                                 int *sums) {
  int s0 = 0, s1 = 0;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < W; x += gridDim.x * blockDim.x) {
    if (gtop) s0 += (int)(gtop[x] >> 56);
    if (gbot) s1 += (int)(gbot[x] >> 56);
  }
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_down_sync(0xffffffffu, s0, o);
    s1 += __shfl_down_sync(0xffffffffu, s1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (s0) atomicAdd(&sums[0], s0);
    if (s1) atomicAdd(&sums[1], s1);
  }
}

// neighbour's flow arrives at my edge row: fold it into the packed words, release completed cells
__global__ void __launch_bounds__(256) band_apply_packed_kernel(unsigned long long *row, const double *__restrict__ sum,
                                                                 const int *__restrict__ cnt, int W, int base_index,
                                                                 int *frontier, int *fcount, double scale) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int k = cnt[x];
  if (k <= 0) return;
  const unsigned long long wv = row[x];
  const unsigned long long val = (wv & kPkVal) + (unsigned long long)sum[x];
  const unsigned long long left = (wv >> 56) - (unsigned long long)k;
  if (left == 0) {
    row[x] = (unsigned long long)__double_as_longlong((double)val * scale);  // (D-infinity sums carry 24 fractional bits)
    frontier[atomicAdd(fcount, 1)] = base_index + x;
  } else {
    row[x] = (left << 56) | val;
  }
}

// =================================================================================================
// Unit-weight D8 on one GPU, tile by tile: the perimeter method of Barnes (2017) for out-of-core D8 accumulation
// (the reference's programs/parallel_d8_accum) with shared memory as the "core".  The raster is cut into 64 x 64
// tiles; the cells on a tile's edge are its *slots*.  Almost every D8 path is short, so almost all the work stays in
// shared memory and only the flow that crosses tile edges goes through a small global solve:
//   1. fa_tile_codes_kernel: per tile, the flow codes from the DEM window (tile + one-cell apron) -> code bytes
//      (tile-major scratch), then every cell's root (the last in-tile cell on its path) by pointer jumping.  Per slot
//      it records in `link`: for an *exit* slot (receiver in another tile) the receiver's slot, for any other slot the
//      exit slot of the same tile where its in-tile path leaves the tile (or none), and in `lword` the exit slot's
//      local accumulation, the number of the tile's data cells whose root it is.
//   2. fa_link_count_kernel + fa_link_walk_kernel: exit slot p drains into next(p), the exit slot where the in-tile
//      path from its receiver's slot leaves that tile.  The exit slots form a forest, solved by the packed countdown
//      walk over slots; each exit's total outflow is added to the inflow of its receiver's slot.
//   3. fa_tile_final_kernel: per tile, the codes again, every cell seeded with 1 plus the inflow on its slot, the
//      in-tile accumulation by pointer doubling (fa_tile_jump with SUM), the result written as doubles.
// Per cell, HBM sees 4 B (DEM) + 2 x 1 B (codes) + 8 B (result); per slot (1/16 of the cells) 16 B of link data.  No
// global atomic touches the cell raster.  All sums are integers < 2^31, so the result is exact whatever the order.
// =================================================================================================
constexpr int kFaT = 64;                           // tile side
constexpr int kFaCells = kFaT * kFaT;
constexpr int kFaSlots = 4 * kFaT;                 // slot numbers per tile: top row, bottom row, left, right column
constexpr unsigned long long kLkOne = 1ull << 32;  // link words: [32 bits donors left | 32 bits sum]; an exit slot can
                                                   // have hundreds of donors, more than the 8-bit field of kPkOne holds

// width (height) of a tile that starts `left` columns (rows) before the raster's edge
__device__ __forceinline__ int fa_side(int left) { return left < kFaT ? left : kFaT; }

// slot of the edge cell (lx, ly) of a tw x th tile, -1 for an inner cell (a corner belongs to its row)
__device__ __forceinline__ int fa_slot_of(int lx, int ly, int tw, int th) {
  if (ly == 0) return lx;
  if (ly == th - 1) return kFaT + lx;
  if (lx == 0) return 2 * kFaT + ly;
  if (lx == tw - 1) return 3 * kFaT + ly;
  return -1;
}

// the cell of slot s; false where s names no cell of a tw x th tile
__device__ __forceinline__ bool fa_slot_cell(int s, int tw, int th, int &lx, int &ly) {
  const int k = s & (kFaT - 1), side = s / kFaT;
  if (side < 2) {
    lx = k;
    ly = side == 0 ? 0 : th - 1;
    return k < tw && (side == 0 || th > 1);
  }
  lx = side == 2 ? 0 : tw - 1;
  ly = k;
  return k > 0 && k < th - 1 && (side == 2 || tw > 1);
}

// Flags of a root in a tile's parent array (cell indices need 12 bits): the path leaves the tile here, or it ends here
// (no receiver, or NoData).  An entry that carries a flag names the root of its cell's path.
constexpr int kFaRootExit = 0x8000, kFaRootEnd = 0x4000, kFaRoot = kFaRootExit | kFaRootEnd;

// the parent array entry of tile cell c with code cd: its in-tile receiver, or c itself flagged as a root
__device__ __forceinline__ int fa_tile_parent(int c, int cd, int tw, int th) {
  const int d = cd & 15;
  if (cd == kCodeNoData || d == 0) return c | kFaRootEnd;
  const int x = (c & (kFaT - 1)) + d8dx(d), y = c / kFaT + d8dy(d);
  if (x < 0 || y < 0 || x >= tw || y >= th) return c | kFaRootExit;
  return y * kFaT + x;
}

// Pointer jumping over a tile's parent array sPar, 16 cells per thread: bit k of `live` says that cell t + 256 k's
// entry carries no flag.  After r rounds such an *exact* entry names p_r, the cell exactly 2^r steps down its in-tile
// path; a round sets p[c] = p[p[c]], and an entry that reads a flag has reached its root in fewer steps and keeps it
// from then on.  The loop ends when every entry names its flagged root, after at most ceil(log2 4096) = 12 rounds.
// With SUM, sAcc holds every cell's weight on entry and its in-tile accumulation on exit.  Writing A_r(c) for the sum of
// the weights of the cells fewer than 2^r steps upstream of c (c included),
//     A_{r+1}(c) = A_r(c) + sum of A_r(d) over the cells d with an exact p_r(d) = c,
// since every cell 2^r to 2^{r+1} - 1 steps upstream of c is fewer than 2^r steps upstream of exactly one such d.  Each
// round reads A_r and p_r before anything is added or replaced, so it takes two barriers; a cell's work is one shared
// atomicAdd per round in which its entry is exact, about log2 of its distance to the root, instead of a walk as long as
// the path.  Without SUM any ancestor read is as good as the one a round intended, so the entry is replaced in place,
// one barrier per round.
template <bool SUM>
__device__ __forceinline__ void fa_tile_jump(uint16_t *sPar, unsigned *sAcc, unsigned live) {
  constexpr int kPer = kFaCells / 256;
  const int t = threadIdx.x;
  while (__syncthreads_or(live)) {
    unsigned pq[kPer], a[kPer];  // SUM: [p_r(c) | p_r(p_r(c)) << 16] and A_r(c), kept across the barrier
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      if (live >> k & 1) {
        const int c = t + 256 * k, p = sPar[c], q = sPar[p];
        if (SUM) {
          pq[k] = (unsigned)p | (unsigned)q << 16;
          a[k] = sAcc[c];
        } else {
          sPar[c] = (uint16_t)q;
          if (q & kFaRoot) live &= ~(1u << k);
        }
      }
    }
    if (SUM) {
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kPer; k++) {
        if (live >> k & 1) {
          const int q = pq[k] >> 16;
          atomicAdd(&sAcc[pq[k] & 0xffffu], a[k]);
          sPar[t + 256 * k] = (uint16_t)q;
          if (q & kFaRoot) live &= ~(1u << k);
        }
      }
    }
  }
}

// Pass 1 needs no accumulation.  Per slot the link solve needs the exit slot where its in-tile path leaves the tile, and
// per exit slot the number of the tile's data cells whose in-tile path ends there.  Both follow from each cell's *root*,
// the last in-tile cell on its path, which pointer jumping (fa_tile_jump without SUM) finds in at most 12 rounds of
// shared-memory loads; a walk would take as many dependent steps as the tile's longest in-tile path.
__global__ void __launch_bounds__(256) fa_tile_codes_kernel(const float *__restrict__ dem, uint8_t *__restrict__ code,
                                                             int *__restrict__ link, unsigned long long *__restrict__ lword,
                                                             unsigned *__restrict__ inflow, int W, int H, float nodata,
                                                             int tiles_x) {
  constexpr int kWin = kFaT + 2;  // DEM window: the tile and a one-cell apron
  static_assert(kFaCells * sizeof(uint16_t) <= kWin * kWin * sizeof(float), "the parent array lives in the DEM window");
  __shared__ __align__(16) float sDem[kWin * kWin];  // first the DEM window, then the parent array
  __shared__ __align__(16) uint8_t sCode[kFaCells];
  __shared__ unsigned sCount[kFaSlots];  // per exit slot: the data cells whose in-tile path ends there
  const int t = threadIdx.x, tile = blockIdx.x;
  sCount[t] = 0;
  const int bx = tile % tiles_x, by = tile / tiles_x;
  const int x0 = bx * kFaT, y0 = by * kFaT;
  const int tw = fa_side(W - x0), th = fa_side(H - y0);
  // NoData (and the apron beyond the raster) is held as the NaN kFaNoDataBits, every NaN of the DEM as the canonical
  // one: as a neighbour any NaN fails every comparison of the steepest-descent scan, which is exactly "skip NoData", and
  // the cell's own NoData test is one integer compare.  A NaN no-data value matches nothing, as in the reference.
  constexpr unsigned kFaNoDataBits = 0x7fffffffu;
  for (int i = t; i < kWin * kWin; i += 256) {
    const int wy = i / kWin, wx = i - wy * kWin;
    const int gy = y0 - 1 + wy, gx = x0 - 1 + wx;
    float v = __uint_as_float(kFaNoDataBits);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      v = __ldg(dem + (size_t)gy * W + gx);
      v = v == nodata ? __uint_as_float(kFaNoDataBits) : v != v ? __uint_as_float(0x7fc00000u) : v;
    }
    sDem[i] = v;
  }
  __syncthreads();
  // flow codes, the rule of fa_d8_prep_rolling_kernel: the first strictly lowest data neighbour; raster-border cells have
  // no receiver.  Thread t: columns 4 (t % 16) .. + 3, a strip of 4 rows, a rolling 3 x 6 register window; the 4 codes of
  // a row leave as one 32-bit word.
  {
    const int lx0 = (t & 15) * 4, ly0 = (t >> 4) * 4;
    float a[3][6];
#pragma unroll
    for (int j = 1; j < 3; j++)
#pragma unroll
      for (int k = 0; k < 6; k++) a[j][k] = sDem[(ly0 + j - 1) * kWin + lx0 + k];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int ly = ly0 + j, gy = y0 + ly;
#pragma unroll
      for (int k = 0; k < 6; k++) {
        a[0][k] = a[1][k];
        a[1][k] = a[2][k];
        a[2][k] = sDem[(ly + 2) * kWin + lx0 + k];
      }
      unsigned word = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int lx = lx0 + k, gx = x0 + lx;
        const float e = a[1][k + 1];
        int cd = 0;
        if (lx >= tw || ly >= th || __float_as_uint(e) == kFaNoDataBits) {
          cd = kCodeNoData;
        } else if (!(gx == 0 || gy == 0 || gx == W - 1 || gy == H - 1)) {
          // neighbours n = 1..8 : W, NW, N, NE, E, SE, S, SW.  Starting the running minimum at the cell's own value
          // folds the reference's `>= e` skip into it (capped at FLT_MAX, the reference's starting value)
          const float ne[9] = {0.f, a[1][k], a[0][k], a[0][k + 1], a[0][k + 2], a[1][k + 2], a[2][k + 2], a[2][k + 1], a[2][k]};
          float lowest = fminf(e, 3.402823466e+38f);
#pragma unroll
          for (int n = 1; n <= 8; n++) {
            if (ne[n] < lowest) {
              lowest = ne[n];
              cd = n;
            }
          }
        }
        word |= (unsigned)cd << (8 * k);
      }
      *reinterpret_cast<unsigned *>(&sCode[ly * kFaT + lx0]) = word;
    }
  }
  __syncthreads();  // the DEM window is dead from here on
  reinterpret_cast<uint4 *>(code + (size_t)tile * kFaCells)[t] = reinterpret_cast<const uint4 *>(sCode)[t];
  uint16_t *sPar = reinterpret_cast<uint16_t *>(sDem);
  unsigned live = 0;
#pragma unroll
  for (int k = 0; k < kFaCells / 256; k++) {
    const int c = t + 256 * k, p = fa_tile_parent(c, sCode[c], tw, th);
    sPar[c] = (uint16_t)p;
    if (!(p & kFaRoot)) live |= 1u << k;
  }
  fa_tile_jump<false>(sPar, nullptr, live);
#pragma unroll
  for (int k = 0; k < kFaCells / 256; k++) {
    const int r = sPar[t + 256 * k];
    if (r & kFaRootExit) atomicAdd(&sCount[fa_slot_of(r & (kFaT - 1), (r & (kFaCells - 1)) / kFaT, tw, th)], 1u);
  }
  __syncthreads();
  // ---- per slot (one per thread): where its in-tile path leaves the tile ----
  const size_t gs = (size_t)tile * kFaSlots + t;
  int lk = -1;  // -1: the path ends inside the tile (or the slot is NoData / unused)
  unsigned long long out = 0;
  int lx, ly;
  if (fa_slot_cell(t, tw, th, lx, ly)) {
    const int c = ly * kFaT + lx, r = sPar[c];
    if (r == (c | kFaRootExit)) {  // an exit slot: link to the receiver's slot (encoded as -2 - slot)
      const int d = sCode[c] & 15;
      const int gx = x0 + lx + d8dx(d), gy = y0 + ly + d8dy(d), rbx = gx / kFaT, rby = gy / kFaT;
      const int rs = fa_slot_of(gx - rbx * kFaT, gy - rby * kFaT, fa_side(W - rbx * kFaT), fa_side(H - rby * kFaT));
      lk = -2 - ((rby * tiles_x + rbx) * kFaSlots + rs);
      out = kLkOne | sCount[t];  // the count starts at 1: the slot's own token (fa_link_walk_kernel)
    } else if (r & kFaRootExit) {
      const int e = r & (kFaCells - 1);
      lk = tile * kFaSlots + fa_slot_of(e & (kFaT - 1), e / kFaT, tw, th);
    }
  }
  link[gs] = lk;
  lword[gs] = out;
  inflow[gs] = 0;
}

// the exit slot where the in-tile path from slot r leaves its tile, -1 if it ends inside
__device__ __forceinline__ int fa_link_next(const int *link, int r) {
  const int l = link[r];
  return l <= -2 ? r : l;
}

__global__ void __launch_bounds__(256) fa_link_count_kernel(const int *__restrict__ link, unsigned long long *lword,
                                                             int nslots) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nslots) return;
  const int l = link[p];
  if (l > -2) return;  // not an exit slot
  const int q = fa_link_next(link, -2 - l);
  if (q >= 0) atomicAdd(&lword[q], kLkOne);
}

// Every exit slot delivers its own token first: the party that brings a count to zero -- the slot itself when all its
// donors have arrived, else its last donor -- owns the total and walks on.  Its outflow goes to the receiver's inflow.
__global__ void __launch_bounds__(256) fa_link_walk_kernel(const int *__restrict__ link, unsigned long long *lword,
                                                            unsigned *inflow, int nslots) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nslots) return;
  int l = link[p];
  if (l > -2) return;
  const unsigned long long old = atomicAdd(&lword[p], 0ull - kLkOne);
  if ((old >> 32) != 1ull) return;
  unsigned long long acc = old & (kLkOne - 1);
  for (;;) {
    const int r = -2 - l;
    atomicAdd(&inflow[r], (unsigned)acc);
    const int q = fa_link_next(link, r);
    if (q < 0) break;
    const unsigned long long o = atomicAdd(&lword[q], acc - kLkOne);
    if ((o >> 32) != 1ull) break;
    acc = (o & (kLkOne - 1)) + acc;
    l = link[q];
  }
}

__global__ void __launch_bounds__(256) fa_tile_final_kernel(const uint8_t *__restrict__ code,
                                                             const unsigned *__restrict__ inflow, double *__restrict__ accum,
                                                             int W, int H, int tiles_x) {
  constexpr unsigned kNoDataAcc = 0xffffffffu;  // a NoData cell's sum: no data cell's sum comes near it (< 2^31)
  __shared__ __align__(16) unsigned sAcc[kFaCells];
  __shared__ __align__(16) uint16_t sPar[kFaCells];
  __shared__ __align__(16) uint8_t sCode[kFaCells];
  const int t = threadIdx.x, tile = blockIdx.x;
  const int bx = tile % tiles_x, by = tile / tiles_x;
  const int x0 = bx * kFaT, y0 = by * kFaT;
  const int tw = fa_side(W - x0), th = fa_side(H - y0);
  reinterpret_cast<uint4 *>(sCode)[t] = __ldg(reinterpret_cast<const uint4 *>(code + (size_t)tile * kFaCells) + t);
  __syncthreads();
  // weights: 1 per data cell (plus the inflow on its slot, below), none for NoData, whose entry is a root from the start
  unsigned live = 0;
#pragma unroll
  for (int k = 0; k < kFaCells / 256; k++) {
    const int c = t + 256 * k, cd = sCode[c], p = fa_tile_parent(c, cd, tw, th);
    sPar[c] = (uint16_t)p;
    sAcc[c] = cd == kCodeNoData ? kNoDataAcc : 1u;
    if (!(p & kFaRoot)) live |= 1u << k;
  }
  __syncthreads();
  int lx, ly;
  if (fa_slot_cell(t, tw, th, lx, ly) && sCode[ly * kFaT + lx] != kCodeNoData)
    sAcc[ly * kFaT + lx] += __ldg(inflow + (size_t)tile * kFaSlots + t);
  fa_tile_jump<true>(sPar, sAcc, live);
  // two cells per thread and step, one 16-byte store where the row's address allows it (odd widths, unaligned rasters)
  for (int c = 2 * t; c < kFaCells; c += 512) {
    const int cx = c & (kFaT - 1), cy = c / kFaT;
    if (cx >= tw || cy >= th) continue;
    const unsigned s0 = sAcc[c], s1 = sAcc[c + 1];
    const double a0 = s0 == kNoDataAcc ? -1.0 : (double)s0, a1 = s1 == kNoDataAcc ? -1.0 : (double)s1;  // -1: flow_accumulation_generic.hpp:95-97
    double *out = accum + (size_t)(y0 + cy) * W + x0 + cx;
    if (cx + 1 < tw && ((uintptr_t)out & 15) == 0) {
      *reinterpret_cast<double2 *>(out) = make_double2(a0, a1);
    } else {
      out[0] = a0;
      if (cx + 1 < tw) out[1] = a1;
    }
  }
}

// the number of slots fa_d8_tiles needs for a w x h raster (slots are numbered with int)
long long fa_tile_slots(int w, int h) {
  return (long long)((w + kFaT - 1) / kFaT) * ((h + kFaT - 1) / kFaT) * kFaSlots;
}

void fa_d8_tiles(const float *d_dem, double *d_accum, int w, int h, float nodata) {
  Ctx &c = ctx();
  const int tiles_x = (w + kFaT - 1) / kFaT;
  const long long nslots = fa_tile_slots(w, h);
  const unsigned ntiles = (unsigned)(nslots / kFaSlots);
  DevBuf<uint8_t> code((size_t)ntiles * kFaCells);
  DevBuf<int> link((size_t)nslots);
  DevBuf<unsigned long long> lword((size_t)nslots);
  DevBuf<unsigned> inflow((size_t)nslots);
  const unsigned sblocks = (unsigned)((nslots + 255) / 256);
  fa_tile_codes_kernel<<<ntiles, 256, 0, c.stream>>>(d_dem, code.p, link.p, lword.p, inflow.p, w, h, nodata, tiles_x);
  fa_link_count_kernel<<<sblocks, 256, 0, c.stream>>>(link.p, lword.p, (int)nslots);
  KernelTimer kt;
  fa_link_walk_kernel<<<sblocks, 256, 0, c.stream>>>(link.p, lword.p, inflow.p, (int)nslots);
  kt.stop_async();
  fa_tile_final_kernel<<<ntiles, 256, 0, c.stream>>>(code.p, inflow.p, d_accum, w, h, tiles_x);
  RDB_CK(cudaGetLastError());
  count_launch(4);
  RDB_CK(cudaStreamSynchronize(c.stream));
  c.stats.ms_main_kernel += kt.ms();
  c.stats.accum_rounds = 1;
}
}  // namespace

// FA_D8 / FA_Tarboton fused (reference methods/flow_accumulation.hpp:27,16): no 36 B/cell props.  T is the DEM's type;
// only the code pass (flow_code_kernel) reads the DEM, everything after it works on the codes.  The D8 engines exist for
// T = float only (the float64 FA_D8 runs on order-preserving float keys, f64.cu).
template <class T>
static void fa_fused(const T *d_dem, double *d_accum, int w, int h, T nodata, bool ones, bool dinf) {
  constexpr bool F32 = sizeof(T) == 4;
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  if constexpr (F32) {
    if (!dinf && ones && c.params.accum_packed && fa_tile_slots(w, h) < INT32_MAX) {
      fa_d8_tiles(d_dem, d_accum, w, h, nodata);  // unit-weight D8: tile by tile (see above)
      return;
    }
  } else if (!dinf) {
    fail("FA_D8 on doubles runs on float keys (fa_fused_dev)");
  }
  DevBuf<uint8_t> code(n);
  DevBuf<float> rmax;
  bool have_codes = false;
  // Unit-weight D-infinity has two engines.  The packed fixed-point walk (accum_walk_dinf_lanes_kernel) is throughput
  // bound: 75 ms against 490 ms at 32768^2 on a filled DEM, whose flats end every flow path early.  After flat
  // resolution every cell flows on, the longest dependency chains have tens of thousands of cells, and the level kernel's
  // barriers (540 ms) still beat the walk's long tail (780 ms).  accum_dinf_packed: 0 level kernel, 1 packed walk,
  // 2 (default) packed walk when more than 5 % of the data cells have no receiver.
  if (dinf && ones && (w & 3) == 0 && ((uintptr_t)d_accum & 15) == 0 && c.params.accum_dinf_packed) {
    rmax.alloc(n);
    const unsigned blocks = (unsigned)((n + 255) / 256);
    unsigned long long *word = reinterpret_cast<unsigned long long *>(d_accum);
    flow_code_kernel<true, T><<<blocks, 256, 0, c.stream>>>(d_dem, code.p, rmax.p, d_accum, w, h, nodata, 1, (int)c.params.flowmet_tarboton_filter);
    have_codes = true;
    DevBuf<DinfShare> share(1);
    RDB_CK(cudaMemsetAsync(share.p, 0, sizeof(DinfShare), c.stream));
    dinf_count_data_kernel<<<c.num_sms * 8, 256, 0, c.stream>>>(code.p, n, share.p);
    RDB_CK(cudaGetLastError());
    count_launch(2);
    DinfShare *hs0 = reinterpret_cast<DinfShare *>(c.pinned);
    RDB_CK(cudaMemcpyAsync(hs0, share.p, sizeof(DinfShare), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    const bool use_packed = c.params.accum_dinf_packed == 1 || (long long)hs0->n_noflow * 20 > (long long)hs0->n_data;
    if (use_packed) {
    dim3 blk(256), grd((w / 4 + 255) / 256, h < 8192 ? h : 8192);
    deps_gather_packed_dinf_x4_kernel<<<grd, blk, 0, c.stream>>>(code.p, word, w, h, 0, h);
    RDB_CK(cudaGetLastError());
    count_launch();
    DevBuf<int> list(n);  // the hand-over list (a ring: at most one entry per ready cell is alive)
    DevBuf<unsigned long long> dstats;
    if (c.params.accum_dinf_stats) {
      dstats.alloc(16);
      RDB_CK(cudaMemsetAsync(dstats.p, 0, 16 * sizeof(unsigned long long), c.stream));
    }
    KernelTimer kt;
    launch_walk_dinf(code.p, rmax.p, word, w, (int)n, list.p, share.p, dstats.p, 0, (int)n, -1);
    RDB_CK(cudaGetLastError());
    count_launch(2);
    DinfShare *hs = reinterpret_cast<DinfShare *>(c.pinned);
    RDB_CK(cudaMemcpyAsync(hs, share.p, sizeof(DinfShare), cudaMemcpyDeviceToHost, c.stream));
    kt.stop_async();
    RDB_CK(cudaStreamSynchronize(c.stream));
    c.stats.ms_main_kernel += kt.ms();
    c.stats.accum_rounds = hs->phases;
    if (dstats.p) {
      unsigned long long hsx[16];
      RDB_CK(cudaMemcpy(hsx, dstats.p, sizeof(hsx), cudaMemcpyDeviceToHost));
      fprintf(stderr,
              "[dinf walk] %.2f ms, %llu warps, %d phases: iterations sum %llu max %llu, lane-steps %llu (%.1f %% of the lanes), "
              "hand-overs %llu in the rings, %llu through the list (%llu claimed back)\n",
              kt.ms(), hsx[4], hs->phases, hsx[0], hsx[3], hsx[2], 100.0 * (double)hsx[2] / (32.0 * (double)(hsx[0] ? hsx[0] : 1)),
              hsx[8], hsx[7], hsx[6]);
    }
    if (hs->done != hs->n_data)
      fail("D-infinity accumulation (packed walk): %d of %d cells walked after %d phases", hs->done, hs->n_data, hs->phases);
    return;
    }
  }
  DevBuf<uint32_t> st(n);
  if (dinf && !have_codes) rmax.alloc(n);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (have_codes) {
    // flow codes, rmax and the unit weights are in place already
  } else if (dinf)
    flow_code_kernel<true, T><<<blocks, 256, 0, c.stream>>>(d_dem, code.p, rmax.p, d_accum, w, h, nodata, ones ? 1 : 0, (int)c.params.flowmet_tarboton_filter);
  else if constexpr (F32) {
    if ((w & 3) == 0 && ((uintptr_t)d_dem & 15) == 0 && ((uintptr_t)d_accum & 15) == 0) {
      dim3 blk(256), grd((w / 4 + 255) / 256, h < 8192 ? h : 8192);
      flow_code_d8_x4_kernel<<<grd, blk, 0, c.stream>>>(d_dem, code.p, d_accum, w, h, nodata, ones ? 1 : 0);
    } else
      flow_code_kernel<false><<<blocks, 256, 0, c.stream>>>(d_dem, code.p, nullptr, d_accum, w, h, nodata, ones ? 1 : 0, (int)c.params.flowmet_tarboton_filter);
  }
  RDB_CK(cudaGetLastError());
  if ((w & 3) == 0) {
    dim3 blk(256), grd((w / 4 + 255) / 256, h < 8192 ? h : 8192);
    deps_gather_x4_kernel<<<grd, blk, 0, c.stream>>>(code.p, st.p, w, h, 0, h, dinf ? 0 : 1);
  } else {
    deps_gather_kernel<<<blocks, 256, 0, c.stream>>>(code.p, st.p, w, h, 0, h, dinf ? 0 : 1);
  }
  RDB_CK(cudaGetLastError());
  count_launch(2);
  WalkArgs<double> a;
  memset(&a, 0, sizeof(a));
  a.code = code.p;
  a.rmaxArr = rmax.p;
  a.accum = d_accum;
  a.st = st.p;
  a.W = w;
  a.H = h;
  if (dinf) run_levels<1>(a, n);
  else run_walk<0, false, double>(a, n);
}

void fa_fused_dev(const float *d_dem, double *d_accum, int w, int h, float nodata, bool ones, bool dinf) {
  fa_fused(d_dem, d_accum, w, h, nodata, ones, dinf);
}
// FA_Tarboton<double, double>: the same engine after a code pass on the doubles.  FA_D8<double, double> on the key raster:
// the accumulation carries no elevation values.
void fa_fused_dev(const double *d_dem, double *d_accum, int w, int h, double nodata, bool ones, bool dinf) {
  if (dinf) return fa_fused(d_dem, d_accum, w, h, nodata, ones, true);
  const size_t n = (size_t)w * h;
  DevBuf<float> key(n);
  const float nd = f64_keys_dev(d_dem, key.p, n, nodata, nullptr, nullptr);
  fa_fused(key.p, d_accum, w, h, nd, ones, false);
}

// FlowAccumulation(props, accum) (reference methods/flow_accumulation_generic.hpp:33-100)
void flow_accumulation_props_dev(const float *d_props, double *d_accum, int w, int h) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  DevBuf<uint32_t> st(n);
  RDB_CK(cudaMemsetAsync(st.p, 0, n * sizeof(uint32_t), c.stream));
  const unsigned blocks = (unsigned)((n + 255) / 256);
  deps_scatter_props_kernel<<<blocks, 256, 0, c.stream>>>(d_props, st.p, w, h);
  RDB_CK(cudaGetLastError());
  mark_sources_props_kernel<<<blocks, 256, 0, c.stream>>>(d_props, st.p, d_accum, n);
  RDB_CK(cudaGetLastError());
  count_launch(2);
  WalkArgs<double> a;
  memset(&a, 0, sizeof(a));
  a.props = d_props;
  a.accum = d_accum;
  a.st = st.p;
  a.W = w;
  a.H = h;
  run_levels<2>(a, n);
}

// d8_flow_accum(dirs, area) (reference methods/d8_methods.hpp:47-139)
void d8_flow_accum_dev(const uint8_t *d_dirs, int32_t *d_area, int w, int h) {
  Ctx &c = ctx();
  const size_t n = (size_t)w * h;
  DevBuf<uint8_t> code(n);
  DevBuf<uint32_t> st(n);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  sanitize_dirs_kernel<<<blocks, 256, 0, c.stream>>>(d_dirs, code.p, n);
  area_init_kernel<<<blocks, 256, 0, c.stream>>>(d_dirs, d_area, n);
  deps_gather_kernel<<<blocks, 256, 0, c.stream>>>(code.p, st.p, w, h, 0, h, 1);
  RDB_CK(cudaGetLastError());
  count_launch(3);
  WalkArgs<int32_t> a;
  memset(&a, 0, sizeof(a));
  a.code = code.p;
  a.accum = d_area;
  a.st = st.p;
  a.W = w;
  a.H = h;
  run_walk<0, true, int32_t>(a, n);
  area_unreleased_kernel<<<blocks, 256, 0, c.stream>>>(st.p, d_area, n);
  RDB_CK(cudaGetLastError());
  count_launch();
}

}  // namespace rdb

// =================================================================================================
// Row-band (multi-GPU) accumulation.  The local raster is (ghost_top + owned + ghost_bottom) rows;
// the ghost rows carry the neighbouring bands' flow codes (so dependency counts are complete) and
// act as parking slots for flow that leaves the band.  Per global round: walk -> take_outflow ->
// (caller exchanges rows) -> apply_inflow -> walk from the cells that just became ready.
// =================================================================================================
namespace rdb {
namespace {

__global__ void __launch_bounds__(256) band_apply_inflow_kernel(double *accum_row, uint32_t *st_row,
                                                                 const double *__restrict__ sum,
                                                                 const int *__restrict__ cnt, int W, int base_index,
                                                                 int *frontier, int *fcount) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const int k = cnt[x];
  if (k <= 0) return;
  accum_row[x] += sum[x];
  const uint32_t old = st_row[x];
  st_row[x] = old - (uint32_t)k;
  if ((old & kDepsMask) == (uint32_t)k) frontier[atomicAdd(fcount, 1)] = base_index + x;
}

// An empty parking slot holds -0.0, the identity of IEEE addition: x + -0.0 == x for every x, -0.0 included, so a
// parcel of -0.0 weights stays -0.0 across a seam, as in the single-band sum (+0.0 would turn it into +0.0).
__global__ void __launch_bounds__(256) band_clear_ghost_kernel(double *row, int W) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x < W) row[x] = -0.0;
}

// ---- proportions (D4, Quinn, Holmgren, Freeman) over row bands ----
// The ghost rows are local edge rows, so their proportions carry no flow and they donate to nobody here: flow from the
// neighbour's edge row into my edge row is announced by a seam donor mask instead, one byte per cell of the sender's
// edge row.  Bit j (j = 0, 1, 2) set: the cell sends a share across the seam to column x + j - 1, whose cell is not
// NoData -- exactly the shares the sender's walk parks in its ghost row.
__global__ void __launch_bounds__(256) band_seam_mask_kernel(const float *__restrict__ props, uint8_t *__restrict__ mask,
                                                              int W, int row, int dy) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  uint32_t m = 0;
  if (x > 0 && x < W - 1) {  // edge columns carry no flow
    const size_t i = (size_t)row * W + x;
    const float *p = props + 9 * i;
    if (p[0] != kNoDataGen) {
#pragma unroll
      for (int k = 1; k <= 8; k++) {
        if (d8dy(k) != dy || !(p[k] > 0)) continue;
        const size_t r = i + (ptrdiff_t)dy * W + d8dx(k);
        if (props[9 * r] == kNoDataGen) continue;  // the walk drops flow into NoData
        m |= 1u << (d8dx(k) + 1);
      }
    }
  }
  mask[x] = (uint8_t)m;
}

// my edge row's donor counts += the neighbour's shares that point at each cell
__global__ void __launch_bounds__(256) band_add_seam_donors_kernel(const uint8_t *__restrict__ mask, uint32_t *st_row, int W) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  uint32_t k = (mask[x] >> 1) & 1u;               // straight across
  if (x + 1 < W) k += mask[x + 1] & 1u;            // from x + 1, one column left
  if (x > 0) k += (mask[x - 1] >> 2) & 1u;         // from x - 1, one column right
  st_row[x] += k;
}

// weights: ghost rows become empty parking slots (-0.0, see band_clear_ghost_kernel), NoData cells -1 (generic.hpp:95-97),
// unit weights 1.0
__global__ void __launch_bounds__(256) band_init_props_accum_kernel(const float *__restrict__ props, double *accum, int W,
                                                                     int H, int y_lo, int y_hi, int ones) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W);
  if (y < y_lo || y >= y_hi) accum[i] = -0.0;
  else if (props[9 * i] == kNoDataGen) accum[i] = -1.0;
  else if (ones) accum[i] = 1.0;
}

// after the seam donors are in: ghost and NoData cells take no part in the walk, cells without donors are its sources
__global__ void __launch_bounds__(256) band_mark_sources_props_kernel(const float *__restrict__ props, uint32_t *st, int W,
                                                                       int H, int y_lo, int y_hi) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W);
  if (y < y_lo || y >= y_hi || props[9 * i] == kNoDataGen) st[i] = 0;
  else if ((st[i] & kDepsMask) == 0) st[i] = kSrcFlag;
}

// ---- direction grids (d8_flow_accum) over row bands ----
// unit weights: ghost rows become empty parking slots (-0.0), NoData cells -1 (d8_methods.hpp:71-74, :111)
__global__ void __launch_bounds__(256) band_init_dirs_accum_kernel(const uint8_t *__restrict__ code, double *accum, int W, int H,
                                                                    int y_lo, int y_hi) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = (int)(i / W);
  accum[i] = (y < y_lo || y >= y_hi) ? -0.0 : (code[i] == kCodeNoData ? -1.0 : 1.0);
}

// (only directions 1..8 are cleared, and only NoData (255) is tested at the receiver: concurrent clears are harmless)
__global__ void __launch_bounds__(256) band_settle_dir_codes_kernel(uint8_t *code, int W, int H) {
  const size_t n = (size_t)W * H;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = code[i];
  if (d == 0 || d > 8) return;
  const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
  const int nx = x + d8dx(d), ny = y + d8dy(d);
  if (nx < 0 || ny < 0 || nx >= W || ny >= H || code[(size_t)ny * W + nx] == kCodeNoData) code[i] = 0;
}

// the int32 areas from the accumulator: doubles, or -- packed words of cells that never completed, which only a loop in
// the direction grid leaves behind -- [donors left (1..8) | integer sum].  Such an unreleased cell (on a loop or
// downstream of one; unpacked: donors left in st) keeps only the inflow it received, without its own unit, as in
// d8_flow_accum (area_unreleased_kernel).
__global__ void __launch_bounds__(256) band_area_from_accum_kernel(const unsigned long long *__restrict__ word,
                                                                    const uint32_t *__restrict__ st,
                                                                    int32_t *__restrict__ area, size_t n, int packed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long v = word[i];
  const unsigned top = (unsigned)(v >> 56);
  if (packed)
    area[i] = (top >= 1 && top <= 8) ? (int32_t)(v & kPkVal) - 1 : (int32_t)__longlong_as_double((long long)v);
  else
    area[i] = (int32_t)__longlong_as_double((long long)v) - ((st[i] & kDepsMask) != 0 ? 1 : 0);
}

}  // namespace

// Flow accumulation methods of the band entry points, numbered as rdb200_dev_fa_method_f32_f64: 0 D8, 1 Tarboton,
// 2 D4, 3 Holmgren (xparam; Quinn = 1.0), 4 Freeman (xparam).
enum : int { FA_BAND_D8 = 0, FA_BAND_DINF = 1, FA_BAND_D4 = 2, FA_BAND_HOLMGREN = 3, FA_BAND_FREEMAN = 4 };

void check_fa_method(int method, double xparam) {
  if (method < FA_BAND_D8 || method > FA_BAND_FREEMAN) fail("flow accumulation: unknown method %d", method);
  if ((method == FA_BAND_HOLMGREN || method == FA_BAND_FREEMAN) && !std::isfinite(xparam))
    fail("flow accumulation: method %d needs a finite exponent, got %g", method, xparam);
}

struct FaccState {
  int W = 0, H = 0, gt = 0, gb = 0;
  bool dinf = false;
  int method = FA_BAND_D8;
  bool mfd = false;       // D4 / Holmgren / Freeman: 9-float proportions, accum_levels_kernel<2, true>
  double *accum = nullptr;
  DevBuf<uint8_t> code;
  DevBuf<float> rmax;
  DevBuf<float> props;
  const float *pr = nullptr;  // the proportions the walk reads: props.p, or the caller's (begin_given_props)
  DevBuf<uint32_t> st;
  DevBuf<int> ghostcnt, fr0, fr1, cnt;
  bool prepared = false;
  bool packed = false;    // unit-weight D8: accumulator words are [donors left | integer sum] until final
  bool packed_dinf = false;  // unit-weight D-infinity: the same words with 24 fractional bits (accum_walk_dinf_lanes_kernel)
  DevBuf<DinfShare> dshare;
  bool fused = false;     // ... and codes + donor counts come from the fused rolling-window pass at the first run
  const float *dem = nullptr;
  float nodata_v = 0.f;
  int n_frontier = 0;     // cells waiting in fr0 (seeded by apply_inflow)
  int rounds = 0;

  size_t n() const { return (size_t)W * H; }

  void begin(const float *d_dem, double *d_accum, int w, int h, float nodata, int ghost_top, int ghost_bottom,
             int method_, double xparam, bool ones) {
    Ctx &c = ctx();
    check_fa_method(method_, xparam);
    W = w;
    H = h;
    gt = ghost_top ? 1 : 0;
    gb = ghost_bottom ? 1 : 0;
    method = method_;
    dinf = method == FA_BAND_DINF;
    mfd = method >= FA_BAND_D4;
    accum = d_accum;
    if (h - gt - gb < 1) fail("facc_begin: band has no owned rows");
    if (mfd) return begin_props(d_dem, nodata, xparam, ones);
    packed = !dinf && ones && (w & 3) == 0 && ((uintptr_t)d_accum & 15) == 0 && c.params.accum_packed != 0;
    packed_dinf = dinf && ones && (w & 3) == 0 && ((uintptr_t)d_accum & 15) == 0 && c.params.accum_dinf_packed != 0;
    if (packed_dinf) {
      packed = true;  // same protocol as packed D8: parked parcels in the ghost words, take / apply on the words
      dshare.alloc(1);
    }
    code.alloc(n());
    if (!packed) st.alloc(n());
    if (dinf) rmax.alloc(n());
    ghostcnt.alloc(2 * (size_t)W);
    fr0.alloc(n());
    fr1.alloc(n());
    cnt.alloc(4);
    RDB_CK(cudaMemsetAsync(ghostcnt.p, 0, 2 * (size_t)W * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(cnt.p, 0, 4 * sizeof(int), c.stream));
    const unsigned blocks = (unsigned)((n() + 255) / 256);
    fused = packed && !packed_dinf && c.params.accum_fused_prep != 0 && ((uintptr_t)d_dem & 15) == 0;
    dem = d_dem;
    nodata_v = nodata;
    if (fused) {
      // only the rows the neighbours ask for now; everything else in ONE rolling-window pass at the first run, after
      // the neighbours' edge codes have been installed in the ghost rows
      dim3 grd((unsigned)((W + 255) / 256), 2);
      flow_code_rows_kernel<<<grd, 256, 0, c.stream>>>(d_dem, code.p, w, h, nodata, gt ? edge_row(0) : -1, gb ? edge_row(1) : -1);
      RDB_CK(cudaGetLastError());
      count_launch();
      return;
    }
    // rows 0 / H-1 of the local raster are either true raster edges (no ghost) or ghost rows whose
    // codes are replaced below, so the per-cell functions' own edge test is exactly right here
    if (dinf)
      flow_code_kernel<true><<<blocks, 256, 0, c.stream>>>(d_dem, code.p, rmax.p, d_accum, w, h, nodata, ones ? 1 : 0, (int)c.params.flowmet_tarboton_filter);
    else
      flow_code_kernel<false><<<blocks, 256, 0, c.stream>>>(d_dem, code.p, nullptr, d_accum, w, h, nodata, ones ? 1 : 0, (int)c.params.flowmet_tarboton_filter);
    RDB_CK(cudaGetLastError());
    count_launch();
    if (packed) return;  // the packed gather (first run) initialises every accumulator word
    const unsigned rb = (unsigned)((W + 255) / 256);
    if (gt) band_clear_ghost_kernel<<<rb, 256, 0, c.stream>>>(accum, W);
    if (gb) band_clear_ghost_kernel<<<rb, 256, 0, c.stream>>>(accum + (size_t)(H - 1) * W, W);
    RDB_CK(cudaGetLastError());
  }

  // D4 / Holmgren / Freeman: the proportions of the whole local raster by the single-GPU kernels.  The owned rows see
  // their full 3 x 3 neighbourhood (the ghost rows hold the neighbours' elevations), so theirs are the single-GPU bits.
  // Ghost rows are local edge rows: no flow, except that a NoData ghost cell still gets slot 0 == NO_DATA_GEN (every
  // FM_* cell function tests NoData before the edge), so the walk drops flow into it as on one GPU.  Donor counts of
  // the owned rows are scattered here; the seam masks (set_ghost_codes) add the neighbours' shares to the edge rows.
  void begin_props(const float *d_dem, float nodata, double xparam, bool ones) {
    props.alloc(9 * n());
    fm_method_dev(method, d_dem, props.p, W, H, nodata, xparam);
    init_props_walk(props.p, ones);
  }

  // FlowAccumulation(props, accum) of a band whose proportions the caller supplies (d_props, 9 floats per cell).  Only
  // slot 0 of the ghost rows is read here, by the NoData test at the receiver, so the ghost rows must hold the neighbours'
  // edge-row proportions (mgpu_flow_accumulation_props_band copies them in); deps_scatter_props_kernel skips the local
  // edge rows, so the shares of those ghost cells are never counted, and the seam donor masks bring them in instead.
  void begin_given_props(const float *d_props, double *d_accum, int w, int h, int ghost_top, int ghost_bottom) {
    W = w;
    H = h;
    gt = ghost_top ? 1 : 0;
    gb = ghost_bottom ? 1 : 0;
    method = FA_BAND_D4;  // any proportions method: the walk and the seam protocol do not depend on it
    mfd = true;
    accum = d_accum;
    if (h - gt - gb < 1) fail("facc_begin: band has no owned rows");
    init_props_walk(d_props, false);
  }

  // donor counts of the proportions `p`, and the weights (ghost rows: empty parking slots; NoData: -1)
  void init_props_walk(const float *p, bool ones) {
    Ctx &c = ctx();
    pr = p;
    st.alloc(n());
    ghostcnt.alloc(2 * (size_t)W);
    fr0.alloc(n());
    fr1.alloc(n());
    cnt.alloc(4);
    RDB_CK(cudaMemsetAsync(ghostcnt.p, 0, 2 * (size_t)W * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(cnt.p, 0, 4 * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(st.p, 0, n() * sizeof(uint32_t), c.stream));
    const unsigned blocks = (unsigned)((n() + 255) / 256);
    deps_scatter_props_kernel<<<blocks, 256, 0, c.stream>>>(pr, st.p, W, H);
    RDB_CK(cudaGetLastError());
    band_init_props_accum_kernel<<<blocks, 256, 0, c.stream>>>(pr, accum, W, H, gt, H - gb, ones ? 1 : 0);
    RDB_CK(cudaGetLastError());
    count_launch(2);
  }

  // d8_flow_accum of a direction grid (unit weights): the codes are the directions, codes other than 0..8 / NoData
  // meaning no flow.  settle_dir_codes() must follow once the ghost rows hold the neighbours' codes.
  void begin_dirs(const uint8_t *d_dirs, double *d_accum, int w, int h, int ghost_top, int ghost_bottom) {
    Ctx &c = ctx();
    W = w;
    H = h;
    gt = ghost_top ? 1 : 0;
    gb = ghost_bottom ? 1 : 0;
    accum = d_accum;
    from_dirs = true;
    if (h - gt - gb < 1) fail("facc_begin: band has no owned rows");
    packed = (w & 3) == 0 && ((uintptr_t)d_accum & 15) == 0 && c.params.accum_packed != 0;
    code.alloc(n());
    if (!packed) st.alloc(n());
    ghostcnt.alloc(2 * (size_t)W);
    fr0.alloc(n());
    fr1.alloc(n());
    cnt.alloc(4);
    RDB_CK(cudaMemsetAsync(ghostcnt.p, 0, 2 * (size_t)W * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(cnt.p, 0, 4 * sizeof(int), c.stream));
    const unsigned blocks = (unsigned)((n() + 255) / 256);
    sanitize_dirs_kernel<<<blocks, 256, 0, c.stream>>>(d_dirs, code.p, n());
    // the packed gather (first run) initialises every accumulator word
    if (!packed) band_init_dirs_accum_kernel<<<blocks, 256, 0, c.stream>>>(code.p, accum, W, H, gt, H - gb);
    RDB_CK(cudaGetLastError());
    count_launch(packed ? 1 : 2);
  }
  bool from_dirs = false;

  // A direction that leaves the local raster or points at a NoData cell becomes "no flow".  For an owned cell that is
  // exactly the flow d8_flow_accum drops: off the global raster (a seam row is inside the local raster) or into NoData,
  // a NoData ghost cell included.  For a ghost cell it only drops flow that never reaches this band.  The walks then
  // need no bounds test and never add into a NoData word, as with codes computed from a DEM.
  void settle_dir_codes() {
    Ctx &c = ctx();
    band_settle_dir_codes_kernel<<<(unsigned)((n() + 255) / 256), 256, 0, c.stream>>>(code.p, W, H);
    RDB_CK(cudaGetLastError());
    count_launch();
  }

  int edge_row(int which) const { return which == 0 ? gt : H - 1 - gb; }   // my first / last owned row
  int ghost_row(int which) const { return which == 0 ? 0 : H - 1; }

  // D8 / D-infinity: the flow codes (and rmax) of my edge row; proportions: its seam donor mask (d_rmax_row unused)
  void get_edge_codes(int which, uint8_t *d_code_row, float *d_rmax_row) {
    Ctx &c = ctx();
    if (mfd) {
      const int row = edge_row(which);
      if (row == 0 || row == H - 1) {
        // the band's one owned row is the raster's first or last row: raster-edge cells carry no flow (the walk skips
        // them), so they announce none.  FM_* never give an edge cell flow; caller-supplied proportions may.
        RDB_CK(cudaMemsetAsync(d_code_row, 0, W, c.stream));
        return;
      }
      band_seam_mask_kernel<<<(unsigned)((W + 255) / 256), 256, 0, c.stream>>>(pr, d_code_row, W, row, which == 0 ? -1 : 1);
      RDB_CK(cudaGetLastError());
      count_launch();
      return;
    }
    const size_t o = (size_t)edge_row(which) * W;
    RDB_CK(cudaMemcpyAsync(d_code_row, code.p + o, W, cudaMemcpyDeviceToDevice, c.stream));
    if (dinf && d_rmax_row)
      RDB_CK(cudaMemcpyAsync(d_rmax_row, rmax.p + o, (size_t)W * 4, cudaMemcpyDeviceToDevice, c.stream));
  }
  void set_ghost_codes(int which, const uint8_t *d_code_row, const float *d_rmax_row) {
    Ctx &c = ctx();
    if ((which == 0 && !gt) || (which == 1 && !gb)) fail("facc_set_ghost_codes: no ghost row on that side");
    if (mfd) {  // the neighbour's seam donor mask: its shares that flow into my edge row
      if (prepared) fail("facc_set_ghost_codes: the seam donors must be in before the first run");
      band_add_seam_donors_kernel<<<(unsigned)((W + 255) / 256), 256, 0, c.stream>>>(d_code_row,
                                                                                      st.p + (size_t)edge_row(which) * W, W);
      RDB_CK(cudaGetLastError());
      count_launch();
      return;
    }
    const size_t o = (size_t)ghost_row(which) * W;
    RDB_CK(cudaMemcpyAsync(code.p + o, d_code_row, W, cudaMemcpyDeviceToDevice, c.stream));
    if (dinf && d_rmax_row)
      RDB_CK(cudaMemcpyAsync(rmax.p + o, d_rmax_row, (size_t)W * 4, cudaMemcpyDeviceToDevice, c.stream));
  }

  template <int MODE>
  void walk(WalkArgs<double> a) {
    Ctx &c = ctx();
    int *hcnt = (int *)c.pinned;
    for (;;) {
      const unsigned blocks = (unsigned)(((size_t)a.nfrontier + 255) / 256);
      if (blocks) {
        // a direction grid walks with CHECK (the sole-donor steps clear st, which tells unreleased cells at the end)
        if (from_dirs) accum_walk_kernel<MODE, true, double, true><<<blocks, 256, 0, c.stream>>>(a);
        else accum_walk_kernel<MODE, false, double, true><<<blocks, 256, 0, c.stream>>>(a);
        RDB_CK(cudaGetLastError());
        count_launch();
      }
      if (MODE == 0) break;
      RDB_CK(cudaMemcpyAsync(hcnt, a.next_count, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
      RDB_CK(cudaStreamSynchronize(c.stream));
      const int nn = *hcnt;
      if (nn == 0) break;
      a.frontier = a.next_frontier;
      a.nfrontier = nn;
      a.next_frontier = (a.frontier == fr0.p) ? fr1.p : fr0.p;
      RDB_CK(cudaMemsetAsync(a.next_count, 0, sizeof(int), c.stream));
    }
  }

  void run_packed(int *sent_top, int *sent_bottom) {
    Ctx &c = ctx();
    unsigned long long *word = reinterpret_cast<unsigned long long *>(accum);
    const int lo_end = gt ? W : 0, hi_start = gb ? (H - 1) * W : H * W;
    if (packed_dinf) {
      walk_packed_async(n_frontier);
    } else if (!prepared && fused) {
      dim3 pgrd((unsigned)((W + kPrepOut - 1) / kPrepOut), (unsigned)((H + kPrepRows - 1) / kPrepRows));
      fa_d8_prep_rolling_kernel<<<pgrd, 256, 0, c.stream>>>(dem, code.p, word, W, H, nodata_v, gt, H - gb);
      launch_walk_packed<true>(code.p, word, W, (int)n(), nullptr, lo_end, hi_start, true);
      count_launch(2);
      prepared = true;
    } else if (!prepared) {
      dim3 blk(256), grd((W / 4 + 255) / 256, H < 8192 ? H : 8192);
      deps_gather_packed_x4_kernel<<<grd, blk, 0, c.stream>>>(code.p, word, W, H, gt, H - gb);
      launch_walk_packed<true>(code.p, word, W, (int)n(), nullptr, lo_end, hi_start, false);
      count_launch(2);
      prepared = true;
    } else if (n_frontier > 0) {
      launch_walk_packed<true>(code.p, word, W, n_frontier, fr0.p, lo_end, hi_start, false);
      count_launch();
    }
    RDB_CK(cudaGetLastError());
    n_frontier = 0;
    if (!packed_dinf) rounds++;  // (walk_packed_async counted it)
    int *h = (int *)c.pinned;
    DevBuf<int> sums(2);
    RDB_CK(cudaMemsetAsync(sums.p, 0, 2 * sizeof(int), c.stream));
    band_count_packed_kernel<<<64, 256, 0, c.stream>>>(gt ? word : nullptr, gb ? word + (size_t)(H - 1) * W : nullptr, W,
                                                       sums.p);
    RDB_CK(cudaMemcpyAsync(h, sums.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (sent_top) *sent_top = h[0];
    if (sent_bottom) *sent_bottom = h[1];
    c.stats.accum_rounds = rounds;
  }

  // packed unit-weight D8, for the C++ band driver: queue the preparation (first call) / the walk from the cells an
  // inflow completed, without waiting for it
  void walk_packed_async(int frontier_cells) {
    Ctx &c = ctx();
    unsigned long long *word = reinterpret_cast<unsigned long long *>(accum);
    const int lo_end = gt ? W : 0, hi_start = gb ? (H - 1) * W : H * W;
    if (packed_dinf) {
      // fr0 is both the list the inflow appended the completed cells to and the walk's hand-over ring
      if (!prepared) {
        dim3 blk(256), grd((W / 4 + 255) / 256, H < 8192 ? H : 8192);
        deps_gather_packed_dinf_x4_kernel<<<grd, blk, 0, c.stream>>>(code.p, word, W, H, gt, H - gb);
        RDB_CK(cudaMemsetAsync(dshare.p, 0, sizeof(DinfShare), c.stream));
        launch_walk_dinf(code.p, rmax.p, word, W, (int)n(), fr0.p, dshare.p, nullptr, lo_end, hi_start, -1);
        count_launch(2);
        prepared = true;
      } else if (frontier_cells > 0) {
        launch_walk_dinf(code.p, rmax.p, word, W, (int)n(), fr0.p, dshare.p, nullptr, lo_end, hi_start, frontier_cells);
        count_launch(2);
      }
      rounds++;
      c.stats.accum_rounds = rounds;
      return;
    }
    if (!prepared) {
      if (fused) {
        dim3 pgrd((unsigned)((W + kPrepOut - 1) / kPrepOut), (unsigned)((H + kPrepRows - 1) / kPrepRows));
        fa_d8_prep_rolling_kernel<<<pgrd, 256, 0, c.stream>>>(dem, code.p, word, W, H, nodata_v, gt, H - gb);
      } else {
        dim3 blk(256), grd((W / 4 + 255) / 256, H < 8192 ? H : 8192);
        deps_gather_packed_x4_kernel<<<grd, blk, 0, c.stream>>>(code.p, word, W, H, gt, H - gb);
      }
      launch_walk_packed<true>(code.p, word, W, (int)n(), nullptr, lo_end, hi_start, fused, cnt.p);
      count_launch(2);
      prepared = true;
    } else if (frontier_cells > 0) {
      launch_walk_packed<true>(code.p, word, W, frontier_cells, fr0.p, lo_end, hi_start, false, cnt.p);
      count_launch();
    }
    RDB_CK(cudaGetLastError());
    rounds++;
    c.stats.accum_rounds = rounds;
  }

  // multi-receiver graphs (D-infinity: MODE 1, proportions: MODE 2): one cooperative launch, levels of the frontier
  // inside the band (accum_levels_kernel); the first run starts from every source, later ones from the cells the
  // neighbours' inflow completed (fr0)
  template <int MODE>
  void run_levels_band(WalkArgs<double> &a) {
    Ctx &c = ctx();
    DevBuf<int> lc(4);
    RDB_CK(cudaMemsetAsync(lc.p, 0, 4 * sizeof(int), c.stream));
    int per_sm = 0;
    RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, accum_levels_kernel<MODE, true>, 256, 0));
    if (per_sm < 1) per_sm = 1;
    const int grid = c.num_sms * per_sm;
    int *q0 = fr0.p, *q1 = fr1.p, *counts = lc.p, *lv = lc.p + 3;
    int seeded = a.frontier ? 1 : 0;
    int nc = a.nfrontier, budget = (int)(c.params.accum_budget > 0 ? c.params.accum_budget : 4);
    if (nc > 0) {
      void *args[] = {(void *)&a, (void *)&q0, (void *)&q1, (void *)&counts, (void *)&nc, (void *)&budget, (void *)&lv, (void *)&seeded};
      RDB_CK(cudaLaunchCooperativeKernel((const void *)accum_levels_kernel<MODE, true>, dim3(grid), dim3(256), args, 0,
                                         c.stream));
      count_launch();
    }
  }

  // returns the number of flow parcels parked in the ghost rows by this run: [top, bottom]
  void run(int *sent_top, int *sent_bottom) {
    if (packed) return run_packed(sent_top, sent_bottom);
    Ctx &c = ctx();
    WalkArgs<double> a;
    memset(&a, 0, sizeof(a));
    a.code = code.p;
    a.rmaxArr = rmax.p;
    a.props = pr;
    a.accum = accum;
    a.st = st.p;
    a.W = W;
    a.H = H;
    a.ghost_lo_end = gt ? W : 0;
    a.ghost_hi_start = gb ? (H - 1) * W : H * W;
    a.ghostcnt = ghostcnt.p;
    a.next_count = cnt.p + 1;
    if (!prepared) {
      const unsigned blocks = (unsigned)((n() + 255) / 256);
      if (mfd)
        band_mark_sources_props_kernel<<<blocks, 256, 0, c.stream>>>(pr, st.p, W, H, gt, H - gb);
      else
        deps_gather_kernel<<<blocks, 256, 0, c.stream>>>(code.p, st.p, W, H, gt, H - gb, dinf ? 0 : 1);
      RDB_CK(cudaGetLastError());
      count_launch();
      prepared = true;
      a.frontier = nullptr;
      a.nfrontier = (int)n();
      a.next_frontier = fr1.p;
    } else {
      a.frontier = fr0.p;
      a.nfrontier = n_frontier;
      a.next_frontier = fr1.p;
    }
    RDB_CK(cudaMemsetAsync(cnt.p, 0, 2 * sizeof(int), c.stream));
    if (mfd) {
      run_levels_band<2>(a);
    } else if (dinf) {
      run_levels_band<1>(a);
    } else {
      walk<0>(a);
    }
    n_frontier = 0;
    rounds++;
    // how much left the band?
    // (cheap: reduce the two count rows on the host side of a tiny kernel-free copy is overkill;
    //  the caller exchanges the rows anyway, so only a boolean is needed -> thrust-free sum)
    int *h = (int *)c.pinned;
    DevBuf<int> sums(2);
    RDB_CK(cudaMemsetAsync(sums.p, 0, 2 * sizeof(int), c.stream));
    sum_rows(sums.p);
    RDB_CK(cudaMemcpyAsync(h, sums.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (sent_top) *sent_top = h[0];
    if (sent_bottom) *sent_bottom = h[1];
    c.stats.accum_rounds = rounds;
  }

  void sum_rows(int *d_sums);

  void take_outflow(int which, double *d_sum_row, int *d_cnt_row) {
    Ctx &c = ctx();
    if ((which == 0 && !gt) || (which == 1 && !gb)) fail("facc_take_outflow: no ghost row on that side");
    if (packed) {
      unsigned long long *g = reinterpret_cast<unsigned long long *>(accum) + (size_t)ghost_row(which) * W;
      band_take_packed_kernel<<<(unsigned)((W + 255) / 256), 256, 0, c.stream>>>(g, d_sum_row, d_cnt_row, W, cnt.p + 3);
      RDB_CK(cudaGetLastError());
      count_launch();
      return;
    }
    double *grow = accum + (size_t)ghost_row(which) * W;
    int *crow = ghostcnt.p + (which == 0 ? 0 : W);
    RDB_CK(cudaMemcpyAsync(d_sum_row, grow, (size_t)W * 8, cudaMemcpyDeviceToDevice, c.stream));
    RDB_CK(cudaMemcpyAsync(d_cnt_row, crow, (size_t)W * 4, cudaMemcpyDeviceToDevice, c.stream));
    band_clear_ghost_kernel<<<(unsigned)((W + 255) / 256), 256, 0, c.stream>>>(grow, W);
    RDB_CK(cudaGetLastError());
    count_launch();
    RDB_CK(cudaMemsetAsync(crow, 0, (size_t)W * 4, c.stream));
  }

  void apply_inflow(int which, const double *d_sum_row, const int *d_cnt_row) {
    Ctx &c = ctx();
    if ((which == 0 && !gt) || (which == 1 && !gb)) fail("facc_apply_inflow: no neighbour on that side");
    const int row = edge_row(which);
    const unsigned rb = (unsigned)((W + 255) / 256);
    if (packed) {
      band_apply_packed_kernel<<<rb, 256, 0, c.stream>>>(reinterpret_cast<unsigned long long *>(accum) + (size_t)row * W,
                                                         d_sum_row, d_cnt_row, W, row * W, fr0.p, cnt.p + 2,
                                                         packed_dinf ? 1.0 / 16777216.0 : 1.0);
      RDB_CK(cudaGetLastError());
      count_launch();
      pending_apply = true;
      return;
    }
    // frontier count lives in cnt[2]; cells are appended to fr0 after whatever is already waiting
    band_apply_inflow_kernel<<<rb, 256, 0, c.stream>>>(accum + (size_t)row * W, st.p + (size_t)row * W, d_sum_row,
                                                       d_cnt_row, W, row * W, fr0.p, cnt.p + 2);
    RDB_CK(cudaGetLastError());
    count_launch();
    pending_apply = true;
  }
  bool pending_apply = false;

  void collect_frontier() {
    Ctx &c = ctx();
    if (!pending_apply) return;
    int *h = (int *)c.pinned;
    RDB_CK(cudaMemcpyAsync(h, cnt.p + 2, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    n_frontier = h[0];
    RDB_CK(cudaMemsetAsync(cnt.p + 2, 0, sizeof(int), c.stream));
    pending_apply = false;
  }
};

namespace {
__global__ void __launch_bounds__(256) band_sum_counts_kernel(const int *__restrict__ ghostcnt, int W, int *sums) {
  int s0 = 0, s1 = 0;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < W; x += gridDim.x * blockDim.x) {
    s0 += ghostcnt[x];
    s1 += ghostcnt[W + x];
  }
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_down_sync(0xffffffffu, s0, o);
    s1 += __shfl_down_sync(0xffffffffu, s1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (s0) atomicAdd(&sums[0], s0);
    if (s1) atomicAdd(&sums[1], s1);
  }
}
}  // namespace

void FaccState::sum_rows(int *d_sums) {
  Ctx &c = ctx();
  band_sum_counts_kernel<<<64, 256, 0, c.stream>>>(ghostcnt.p, W, d_sums);
  RDB_CK(cudaGetLastError());
}

// Row-band (multi-GPU) flow accumulation driven from C++ over a rdb200_comm, for every method of check_fa_method: the
// protocol of FaccState (edge codes -- or, for proportions, seam donor masks -- to the neighbours once, then rounds of:
// walk | parked outflow of the two seams in ONE message per neighbour (sums and parcel counts) | neighbours' inflow
// releases cells of the edge rows | a 1-int all-reduce says whether anyone shipped).
static void fa_band_rounds(const rdb200_comm *comm, FaccState &A, int *xrounds) {
  Ctx &c = ctx();
  const int world = comm_world(comm);
  const int w = A.W, gt = A.gt, gb = A.gb;
  // message layout per side: [w doubles: sums | w ints: parcel counts]; codes: [w floats: rmax | w bytes: codes or seam
  // donor masks] (the float half is unused for proportions).  Each of the four messages starts 16-byte aligned, so that
  // the sums of the second one are aligned doubles for an odd width too.
  const size_t msg = ((size_t)w * 12 + 15) & ~(size_t)15;
  DevBuf<uint8_t> buf(4 * msg);
  uint8_t *su = buf.p, *sd = buf.p + msg, *ru = buf.p + 2 * msg, *rd = buf.p + 3 * msg;
  auto rmaxp = [&](uint8_t *m) { return reinterpret_cast<float *>(m); };
  auto codep = [&](uint8_t *m) { return m + (size_t)w * 4; };
  auto sump = [&](uint8_t *m) { return reinterpret_cast<double *>(m); };
  auto cntp = [&](uint8_t *m) { return reinterpret_cast<int *>(m + (size_t)w * 8); };
  if (world > 1) {
    RDB_CK(cudaMemsetAsync(buf.p, 0, 4 * msg, c.stream));
    if (gt) A.get_edge_codes(0, codep(su), rmaxp(su));
    if (gb) A.get_edge_codes(1, codep(sd), rmaxp(sd));
    comm_exchange(comm, su, ru, sd, rd, (size_t)w * 5);
    if (gt) A.set_ghost_codes(0, codep(ru), rmaxp(ru));
    if (gb) A.set_ghost_codes(1, codep(rd), rmaxp(rd));
  }
  if (A.from_dirs) A.settle_dir_codes();
  DevBuf<int> flag(1);
  int *hflag = (int *)c.pinned + 1024;
  int rounds = 0;
  if (A.packed && world > 1) {
    // unit-weight D8: one stream synchronisation per exchange round.  Everything of a round is queued back to back --
    // walk | take the parked outflow (and count the parcels) | exchange | apply the inflow (device-side frontier) | 1-int
    // all-reduce -- and the host reads {any parcels anywhere, my new frontier length} in one copy.
    int frontier_cells = 0;
    for (;;) {
      A.walk_packed_async(frontier_cells);
      rounds++;
      if (getenv("RDB_MGPU_DEBUG")) fprintf(stderr, "[mgpu fa] rank %d round %d frontier %d\n", comm_rank(comm), rounds, frontier_cells);
      RDB_CK(cudaMemsetAsync(A.cnt.p + 2, 0, 2 * sizeof(int), c.stream));  // [2] frontier length, [3] parcels taken
      if (gt) A.take_outflow(0, sump(su), cntp(su));
      if (gb) A.take_outflow(1, sump(sd), cntp(sd));
      comm_exchange(comm, su, ru, sd, rd, msg);
      if (gt) A.apply_inflow(0, sump(ru), cntp(ru));
      if (gb) A.apply_inflow(1, sump(rd), cntp(rd));
      RDB_CK(cudaMemcpyAsync(flag.p, A.cnt.p + 3, sizeof(int), cudaMemcpyDeviceToDevice, c.stream));
      comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
      RDB_CK(cudaMemcpyAsync(hflag, flag.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
      RDB_CK(cudaMemcpyAsync(hflag + 1, A.cnt.p + 2, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
      RDB_CK(cudaStreamSynchronize(c.stream));
      A.pending_apply = false;
      if (getenv("RDB_MGPU_DEBUG")) fprintf(stderr, "[mgpu fa] rank %d round %d sent-anywhere %d new frontier %d\n", comm_rank(comm), rounds, hflag[0], hflag[1]);
      if (hflag[0] == 0) break;
      frontier_cells = hflag[1];
      if (rounds > 1000000) fail("mgpu_fa: exchange rounds exceeded");
    }
    if (xrounds) *xrounds = rounds;
    return;
  }
  for (;;) {
    A.collect_frontier();
    int a = 0, b = 0;
    A.run(&a, &b);
    rounds++;
    if (world == 1) break;
    RDB_CK(cudaMemsetAsync(flag.p, 0, sizeof(int), c.stream));
    if (a + b > 0) count_launch();
    {
      const int mine = a + b > 0 ? 1 : 0;
      RDB_CK(cudaMemcpyAsync(flag.p, &mine, sizeof(int), cudaMemcpyHostToDevice, c.stream));  // (pageable 4 bytes: staged at once)
    }
    comm_allreduce(comm, flag.p, 1, RDB200_MAX_I32);
    RDB_CK(cudaMemcpyAsync(hflag, flag.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (*hflag == 0) break;
    if (gt) A.take_outflow(0, sump(su), cntp(su));
    if (gb) A.take_outflow(1, sump(sd), cntp(sd));
    comm_exchange(comm, su, ru, sd, rd, msg);
    if (gt) A.apply_inflow(0, sump(ru), cntp(ru));
    if (gb) A.apply_inflow(1, sump(rd), cntp(rd));
    if (rounds > 1000000) fail("mgpu_fa: exchange rounds exceeded");
  }
  RDB_CK(cudaStreamSynchronize(c.stream));
  if (xrounds) *xrounds = rounds;
}

void mgpu_fa_band(const rdb200_comm *comm, const float *d_dem, double *d_accum, int w, int hloc, float nodata, int gt, int gb,
                  int method, double xparam, bool ones, int *xrounds) {
  FaccState A;
  A.begin(d_dem, d_accum, w, hloc, nodata, gt, gb, method, xparam, ones);
  fa_band_rounds(comm, A, xrounds);
}

// FlowAccumulation(props, accum) over row bands, with the proportions supplied by the caller: the proportions protocol of
// mgpu_fa_band (seam donor masks, the level walk, parcels parked in the ghost rows) on d_props instead of FM_x of a DEM.
// The caller's ghost rows are not trusted: one exchange of the edge rows (36 B per cell) puts the neighbours' owned
// proportions there first, so that the seam masks and the walk see which ghost cells are NoData.
void mgpu_flow_accumulation_props_band(const rdb200_comm *comm, float *d_props, double *d_accum, int w, int hloc, int gt, int gb,
                                       int *xrounds) {
  const char *what = "mgpu_flow_accumulation_props";
  if (!d_accum) fail("%s: null pointer", what);
  check_band_args(what, comm, d_props, w, hloc, gt, gb);
  exchange_band_rows(comm, d_props, 9 * sizeof(float), w, hloc, gt, gb);
  FaccState A;
  A.begin_given_props(d_props, d_accum, w, hloc, gt, gb);
  fa_band_rounds(comm, A, xrounds);
}

// d8_flow_accum over row bands: the protocol above on the codes of a direction grid, whose ghost rows are not trusted
// (the edge-code exchange installs the neighbours' rows).  The walk runs on a float64 accumulator -- packed
// [donors | integer sum] words where the width allows -- and the int32 areas are written at the end; the ghost rows of
// d_area are scratch.
void mgpu_d8_flow_accum_band(const rdb200_comm *comm, const uint8_t *d_dirs, int32_t *d_area, int w, int hloc, int gt, int gb,
                             int *xrounds) {
  Ctx &c = ctx();
  const char *what = "mgpu_d8_flow_accum";
  if (!d_area) fail("%s: null pointer", what);
  check_band_args(what, comm, d_dirs, w, hloc, gt, gb);
  const size_t n = (size_t)w * hloc;
  DevBuf<double> acc(n);
  {
    FaccState A;
    A.begin_dirs(d_dirs, acc.p, w, hloc, gt, gb);
    fa_band_rounds(comm, A, xrounds);
    band_area_from_accum_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(
        reinterpret_cast<const unsigned long long *>(acc.p), A.st.p, d_area, n, A.packed ? 1 : 0);
    RDB_CK(cudaGetLastError());
    count_launch();
  }
  RDB_CK(cudaStreamSynchronize(c.stream));
}

}  // namespace rdb

struct rdb200_facc_state {
  rdb::FaccState st;
};

extern "C" {

int rdb200_dev_facc_begin_method(rdb200_facc_state **state, const float *d_dem, double *d_accum_inout, int32_t width,
                                 int32_t height, float nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t method,
                                 double xparam, int32_t accum_is_ones) {
  return rdb::capi_call([&] {
    rdb::ensure_init();
    if (!state || !d_dem || !d_accum_inout) rdb::fail("facc_begin: null pointer");
    auto s = std::make_unique<rdb200_facc_state>();
    s->st.begin(d_dem, d_accum_inout, width, height, nodata, ghost_top, ghost_bottom, method, xparam, accum_is_ones != 0);
    *state = s.release();
  });
}

int rdb200_dev_facc_begin(rdb200_facc_state **state, const float *d_dem, double *d_accum_inout, int32_t width,
                          int32_t height, float nodata, int32_t ghost_top, int32_t ghost_bottom, int32_t dinf,
                          int32_t accum_is_ones) {
  return rdb200_dev_facc_begin_method(state, d_dem, d_accum_inout, width, height, nodata, ghost_top, ghost_bottom,
                                      dinf ? rdb::FA_BAND_DINF : rdb::FA_BAND_D8, 0.0, accum_is_ones);
}

int rdb200_dev_facc_get_edge_codes(rdb200_facc_state *state, int32_t which, uint8_t *d_code_row, float *d_rmax_row) {
  return rdb::capi_call([&] {
    state->st.get_edge_codes(which, d_code_row, d_rmax_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_facc_set_ghost_codes(rdb200_facc_state *state, int32_t which, const uint8_t *d_code_row,
                                    const float *d_rmax_row) {
  return rdb::capi_call([&] {
    state->st.set_ghost_codes(which, d_code_row, d_rmax_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_facc_run(rdb200_facc_state *state, int32_t *sent_top, int32_t *sent_bottom) {
  return rdb::capi_call([&] {
    state->st.collect_frontier();
    int a = 0, b = 0;
    state->st.run(&a, &b);
    if (sent_top) *sent_top = a;
    if (sent_bottom) *sent_bottom = b;
  });
}

int rdb200_dev_facc_take_outflow(rdb200_facc_state *state, int32_t which, double *d_sum_row, int32_t *d_cnt_row) {
  return rdb::capi_call([&] {
    state->st.take_outflow(which, d_sum_row, d_cnt_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_facc_apply_inflow(rdb200_facc_state *state, int32_t which, const double *d_sum_row,
                                 const int32_t *d_cnt_row) {
  return rdb::capi_call([&] {
    state->st.apply_inflow(which, d_sum_row, d_cnt_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_facc_finish(rdb200_facc_state *state) {
  return rdb::capi_call([&] {
    if (state) {
      RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
      delete state;
    }
  });
}

}  // extern "C"
