// Depression filling on H100: the Priority-Flood result computed as the greatest fixed point of
//
//     W(c) = max( Z(c), min over the 8 neighbours n of W(n) ),   W = Z on the raster border,
//
// reached from above (W0 = +inf on interior cells).  The fixed point is the unique
// min-over-paths-of-max-elevation surface, i.e. exactly what the reference's serial
// priority-queue flood produces (include/richdem/depressions/Zhou2016.hpp:125-191 via
// depressions.hpp:13-21), and only comparisons/copies of input values are involved, so the
// result is bit-identical.  See DESIGN.md section "fill" for the proof sketch and layout.
//
// Formulation ("spill-scan"): the raster is cut into 64x64 tiles.  One sweep round is ONE
// persistent kernel launch that walks a compacted worklist of active tiles; for each tile it
//   1. stages W (with a one-cell apron) and Z into shared memory with two TMA tile loads
//      (cp.async.bulk.tensor.2d + mbarrier),
//   2. relaxes the tile to its local fixed point entirely in shared memory / registers: a
//      compacted list of dirty 4x4 blocks is kept in shared memory; every pass hands one dirty
//      block to a thread, which runs a forward+backward Gauss-Seidel pass over its 16 cells in
//      registers and marks the blocks that read what it changed,
//   3. writes the changed block rows back with coalesced float4 stores, and
//   4. appends the neighbouring tiles whose apron it changed to the next round's worklist,
//      together with the apron side(s) that changed and the lowest water level that arrived.
// Between tiles the iteration is chaotic (asynchronous Jacobi); every value ever stored is an
// upper bound of the answer and updates are monotone, so any schedule converges to the same
// fixed point.  The device-wide "anything changed" signal is the next worklist's length.
// fill_admit_kernel orders the flood by rising water level (see DESIGN.md 3.1); the same engine
// with the "+1" operator (fill_sweep_kernel<1>) computes the geodesic distances of the flat
// resolution (csrc/flats.cu), and FillState doubles as the row-band (multi-GPU) solver.
#include "common.cuh"

#include <chrono>
#include <memory>

namespace rdb {

namespace {

#ifndef RDB_TX
#define RDB_TX 64
#endif
#ifndef RDB_TY
#define RDB_TY 64
#endif
#ifndef RDB_FILL_THREADS
#define RDB_FILL_THREADS 128
#endif
#ifndef RDB_FILL_MIN_CTAS
#define RDB_FILL_MIN_CTAS 6
#endif
constexpr int TX = RDB_TX;       // tile width  (cells), multiple of 4, <= 248
constexpr int TY = RDB_TY;       // tile height (cells), multiple of 4
constexpr int BXN = TX / 4;      // 4x4 blocks per tile row
constexpr int BYN = TY / 4;      // block rows per tile (<= 16: they are tracked in a 16-bit mask)
constexpr int PADL = 4;          // cell (x,y) lives at padded (x+PADL, y+1)
constexpr int SP = TX + 2 * PADL;  // shared-memory row pitch of the W tile (floats): 72
constexpr int SROWS = TY + 2;    // W tile rows incl. apron: 66
constexpr int FILL_THREADS = RDB_FILL_THREADS;  // threads per CTA; each pass hands one dirty 4x4 block to a thread
constexpr int FILL_MIN_CTAS = RDB_FILL_MIN_CTAS;
static_assert(BYN <= 16 && BXN * BYN <= 256 && TX % 4 == 0 && TY % 4 == 0, "tile shape");
constexpr uint32_t W_TILE_BYTES = SP * SROWS * 4;
constexpr uint32_t Z_TILE_BYTES = TX * TY * 4;

struct RoundCtl {
  int count;  // tiles in this round's worklist
  int take;   // next worklist slot to hand out
};

struct FillDev {
  RoundCtl ctl[3];  // rotating: cur = round%3, next = (round+1)%3, being-zeroed = (round+2)%3
  RoundCtl proc[3]; // level-ordered mode: tiles of the current worklist admitted this round
  unsigned long long visits;
  unsigned long long iters;
  unsigned long long block_updates;  // 4x4 blocks relaxed (threads that did not skip a pass)
  unsigned long long warp_updates;   // warps with at least one such thread
  unsigned long long idle_visits;    // tile visits that changed nothing
  unsigned long long wakes_dropped;  // changed tile sides / corners whose neighbour the wake test left asleep
  unsigned long long iter_hist[8];   // visits by pass count: 1,2,3-4,5-8,9-16,17-32,33-64,65+
  int edge_changed;  // bit0: raster row 1 changed, bit1: raster row H-2 changed
  int zmin_ord, zmax_ord;  // ordered-int min / max of the finite input elevations
  unsigned long long deferred;  // tile visits postponed by the level schedule
  unsigned long long live_rounds;  // sweep launches that found a non-empty worklist
  // level-ordered admission (device-side feedback loop, see fill_admit_kernel)
  float level, step, step_min, level_max;
  int target, ordered;
  int ndefer[3];  // tiles postponed by the admit kernel, by round%3
};

struct FillArgs {
  // Z of cell (x, y) is Z[(y + zoy) * zpitch + x + zox] and its water level Wp[(y + woy) * pitch + x + wox].  Padded
  // layout: both padded arrays (pitch, offsets PADL and 1).  In place (`inplace`): W is the caller's w x h raster and Z a
  // compact w x h array (row stride W, no offsets); cells outside the raster read as +inf.
  const float *Z;
  int zpitch, zox, zoy;
  int inplace;
  // round 1 of a lifted start (in place only): W is built from the coarse surface instead of loaded (null: load it);
  // `staged` flags the tiles whose cells are in W already.  Z is then still the caller's raster, and every tile saves its
  // Z to `zcopy` (the compact Z of the later rounds) before its W overwrites it.
  const float *coarse;
  int Wc, pool, yoff;
  int *staged;
  float *zcopy;
  float *Wp;
  int pitch;  // floats
  int wox, woy;
  int W, H;
  int tilesX, tilesY;
  int *list0, *list1;
  int *stamp;
  int *sides;  // [2][tiles]: apron sides that changed, by round parity
  int *keys;   // [2][tiles]: ordered-int min of the water levels that arrived at the tile's apron
  float level; // tiles whose key is above this level are postponed to a later round (+inf: none)
  int *plist;  // level-ordered mode: admitted tiles of this round (filled by fill_admit_kernel)
  int use_proc;
  FillDev *dev;
  int round;
  int max_iters;
  int use_tma;
  int profile;
  int *dirty;  // per tile: a visit wrote cells back since the flags were last cleared (V-cycle bookkeeping; may be null)
  // fill only (null: every changed side wakes its neighbour): per tile, one word per edge line -- N row, S row, W column,
  // E column -- with bit i set while cell i of that line may still be above its Z (see fill_wake_neighbours)
  unsigned long long *edge_above;
};

// ---- PTX helpers: mbarrier + TMA ----------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
  uint32_t ok;
  const uint32_t addr = smem_u32(bar);
  do {
    asm volatile(
        "{\n"
        "  .reg .pred p;\n"
        "  mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "  selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, int c0, int c1,
                                            unsigned long long *bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(smem_dst)),
      "l"((unsigned long long)map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// shared -> global tile store (cells of the box outside the tensor are not written), committed as its own bulk group
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, int c0, int c1, const void *smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"((unsigned long long)map),
               "r"(c0), "r"(c1), "r"(smem_u32(smem_src))
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// the shared memory of every bulk store issued by this thread may be overwritten
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every bulk store issued by this thread is complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- the sweep kernel --------------------------------------------------------------------
// A tile is 16x16 "blocks" of 4x4 cells.  Relaxation is driven by a compacted list of dirty
// blocks kept in shared memory: a pass hands one dirty block to each thread (so warps stay full
// however sparse the activity is), the thread pulls the block and its rim into registers, runs a
// forward and a backward Gauss-Seidel pass over the 16 cells, writes back the rows that changed
// and marks the blocks that read the cells it changed.  Marks are compacted (ballot + popc) into
// the next pass's list.  A visit starts from the blocks along the apron sides that changed since
// the tile was last relaxed (the interior is still at its local fixed point).
constexpr int NBLK = BXN * BYN;  // blocks per tile
constexpr int MKP = BXN + 2;       // pitch of the mark array (one spare entry all round)
constexpr int NWARP = FILL_THREADS / 32;
constexpr int SEG = ((NBLK + NWARP - 1) / NWARP + 31) / 32 * 32;  // blocks scanned / listed per warp
// apron sides (and corners) of a tile that changed; SIDE_FULL = relax every block
enum : int { SIDE_N = 1, SIDE_S = 2, SIDE_W = 4, SIDE_E = 8, SIDE_NW = 16, SIDE_NE = 32, SIDE_SW = 64,
             SIDE_SE = 128, SIDE_FULL = 256 };

// order-preserving float <-> int map (so atomicMin/Max on ints orders floats, negatives included)
__host__ __device__ __forceinline__ int f2ord(float f) {
  int b;
  memcpy(&b, &f, 4);
  return b >= 0 ? b : (b ^ 0x7fffffff);
}
__host__ __device__ __forceinline__ float ord2f(int o) {
  const int b = o >= 0 ? o : (o ^ 0x7fffffff);
  float f;
  memcpy(&f, &b, 4);
  return f;
}
constexpr int ORD_POS_INF = 0x7f800000;

__device__ __forceinline__ void enqueue_tile(const FillArgs &a, RoundCtl *next, int *list_next, int t,
                                             int stampval, int side_bits, int key_ord) {
  atomicOr(&a.sides[(stampval & 1) * a.tilesX * a.tilesY + t], side_bits);
  atomicMin(&a.keys[(stampval & 1) * a.tilesX * a.tilesY + t], key_ord);
  if (atomicExch(&a.stamp[t], stampval) != stampval) {
    const int idx = atomicAdd(&next->count, 1);
    list_next[idx] = t;
  }
}

__device__ __forceinline__ float min3f(float a, float b, float c) { return fminf(fminf(a, b), c); }

// std::nextafter(x, +inf) on the float bits: +inf (and NaN) stay, -0 goes to +denorm_min, a negative value one step
// towards zero (-denorm_min to -0, -inf to -FLT_MAX), a positive one (and +0) one step up (FLT_MAX to +inf)
__host__ __device__ __forceinline__ float next_up(float x) {
  int b;
  memcpy(&b, &x, 4);
  b = b < 0 ? (b == (int)0x80000000 ? 1 : b - 1) : (b < 0x7f800000 ? b + 1 : b);
  float r;
  memcpy(&r, &b, 4);
  return r;
}

// the neighbour term of fill_sweep_kernel<STEP>: W(c) <- min(W(c), max(Z(c), fill_step(min over the neighbours of W)))
template <int STEP>
__device__ __forceinline__ float fill_step(float w) {
  if constexpr (STEP == 1) return w + 1.0f;
  else if constexpr (STEP == 2) return next_up(w);
  else return w;
}

// ---- the wake test (fill only) ----------------------------------------------------------------------------------------
// A changed tile edge used to wake the neighbour across it whatever the new values were, and most of those visits found
// nothing to do: the neighbour's cell next to the edge already sat at its Z (W == Z never moves again) or at or below
// the new edge.  Now the neighbour N across a changed side or corner is only woken if one of its cells `a` next to the
// edge has
//     its bit set in N's edge_above word   and   min(this tile's own cells adjacent to a) < W(a),
// i.e. if the new edge can lower a.  W(a) is taken from this visit's apron: the copy of N's cells the visit started from.
// No fence protocol is needed:
//   * N's cells only decrease, so the apron value is at least every value N holds now or later -- whether N is idle or
//     in a visit of its own (each cell read before or after N's store of it): e >= W_apron(a) means the new edge
//     cannot lower a in either case;
//   * a bit is cleared only for a cell at W == Z, which relaxation never moves again (Z only changes on the ghost rows
//     of a row band, border cells whose W drops with it), so a stale word only has bits set that could be clear: an
//     extra wake, never a lost one;
//   * when N is woken, its visit in the next launch sees this tile's stores.
// The staged first round needs no exception: the apron of a neighbour that had not stored its cells when the window was
// built holds the lifted level that neighbour starts from -- never the raster's Z, which is below it -- and so bounds
// every value the neighbour stores from above; a tile's words read all ones until its first visit stores them.
// Only the tile's own cells count (three for D8, one for D4; one against one at a corner, and no D4 corner wake: that
// stencil never reads the corner aprons): an apron cell belongs to another tile, which tests its own edge.
constexpr bool WAKE_WORDS = TX <= 64 && TY <= 64;  // one 64-bit word per edge line

// edge line s of the W window (0: N row, 1: S row, 2: W column, 3: E column): cell i at sW[o + i * st], the neighbour's
// adjacent cell at sW[o + i * st + da], its Z at sZ[zo + i * zs]
struct EdgeLine {
  int len, o, st, da, zo, zs;
};
__device__ __forceinline__ EdgeLine edge_line(int s) {
  switch (s) {
    case 0: return {TX, SP + PADL, 1, -SP, 0, 1};
    case 1: return {TX, TY * SP + PADL, 1, SP, (TY - 1) * TX, 1};
    case 2: return {TY, SP + PADL, SP, -1, 0, TX};
    default: return {TY, SP + PADL + TX - 1, SP, 1, TX - 1, TX};
  }
}

// ---- staged first round: drain the lifted tile with column sweeps -----------------------------------------------------
// A tile of the staged round starts from the lifted surface (constant pool x pool plateaus) and must drain nearly every
// cell down towards Z, with all of its blocks dirty.  Before the dirty-block relaxation (which then runs unchanged from
// SIDE_FULL and finishes the local fixed point), an N->S and an S->N sweep carry the drain down and up the whole tile:
// one column per lane, a 64-row recurrence on the row before, W(x, y) <- min(W, max(Z, min of W(x-1..x+1, y -+ 1)))
// (D4: W(x, y -+ 1) only -- a diagonal would lower cells below the D4 answer).  Every update is
// W(c) <- min(W(c), max(Z(c), W(n))) for a neighbour n, which keeps W >= W* (W*(c) <= max(Z(c), W*(n))), leaves pinned
// border cells (W = Z) and cells outside the raster (+inf) where they are, and only selects input values, so the result
// is bit-identical.  Warps 0-1 run N->S over the top half while warps 2-3 run S->N over the bottom half, then they swap
// halves carrying their last row in registers: both chains span the tile, and no cell has two writers in a phase (a
// value read from a cell another warp owns may be old or new; both are upper bounds).
// The tile's change flags and kmin are set for every cell the sweeps lower, as the block loop would have set them: a
// tile edge lowered here and not touched again must still wake the neighbour that already read its lifted value in
// this round.  (W->E / E->W row scans as warp scans of composed clamps were measured too: they cost more than they saved.)
constexpr bool DRAIN_SWEEPS = TX == 64 && TY == 64 && FILL_THREADS == 128;

template <bool TOPO4>
__device__ __forceinline__ void fill_drain_sweeps(float *sW, const float *sZ, int y0, int H, int *sFlags, int *sKey) {
  const unsigned FULL = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int x = 32 * (wrp & 1) + lane;
  const bool down = wrp < 2;
  const int dy = down ? 1 : -1;
  const bool ecol = x < 4 || x >= TX - 4;
  unsigned long long rows = 0;                // tile rows where this thread lowered its column's cell
  float kmin = __int_as_float(0x7f800000);   // lowest level it put on a cell of an edge block
  int y = down ? 0 : TY - 1;
  float p = sW[(y - dy + 1) * SP + PADL + x];  // the apron row
#pragma unroll 1
  for (int half = 0; half < 2; half++) {
#pragma unroll 8
    for (int s = 0; s < TY / 2; s++, y += dy) {
      const float zz = sZ[y * TX + x];
      float *cell = &sW[(y + 1) * SP + PADL + x];
      const float w = *cell;
      float m = p;
      if (!TOPO4) {
        float pl = __shfl_up_sync(FULL, p, 1), pr = __shfl_down_sync(FULL, p, 1);
        const float *prow = &sW[(y - dy + 1) * SP + PADL + x];
        if (lane == 0) pl = prow[-1];
        if (lane == 31) pr = prow[1];
        m = min3f(pl, p, pr);
      }
      const float nw = fminf(w, fmaxf(zz, m));
      p = w;
      if (nw < w) {
        *cell = nw;
        p = nw;
        rows |= 1ull << y;
        if (ecol || y < 4 || y >= TY - 4) kmin = fminf(kmin, nw);
      }
    }
    __syncthreads();  // the other half's writers are done before it is swept
  }
  int f = 0;
#pragma unroll
  for (int by = 0; by < BYN; by++)
    if ((rows >> (4 * by)) & 0xFull) f |= 1 << (12 + by);
  if (rows & 1ull) f |= SIDE_N;
  if (rows >> (TY - 1)) f |= SIDE_S;
  if (x == 0 && rows) f |= SIDE_W | (rows & 1ull ? SIDE_NW : 0) | (rows >> (TY - 1) ? SIDE_SW : 0);
  if (x == TX - 1 && rows) f |= SIDE_E | (rows & 1ull ? SIDE_NE : 0) | (rows >> (TY - 1) ? SIDE_SE : 0);
  const int j1 = 1 - y0, j2 = (H - 2) - y0;  // raster rows 1 and H - 2
  if (j1 >= 0 && j1 < TY && ((rows >> j1) & 1ull)) f |= 1 << 9;
  if (j2 >= 0 && j2 < TY && ((rows >> j2) & 1ull)) f |= 1 << 10;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f |= __shfl_xor_sync(FULL, f, o);
    kmin = fminf(kmin, __shfl_xor_sync(FULL, kmin, o));
  }
  if (lane == 0 && f) {
    atomicOr(sFlags, f);
    if (f & 0xFF) atomicMin(sKey, f2ord(kmin));
  }
  // (the second half's __syncthreads above already published the swept window to the block loop)
}

// End of a fill visit (sW / sZ: the relaxed window; fl: the tile's change flags, key: the lowest new edge level): store
// the tile's edge words, then wake the neighbours across the changed sides and corners that the new edge can lower.
// One warp per edge line; lane 1 of warp s takes corner s (NW, NE, SW, SE).
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
template <bool TOPO4>
__device__ __noinline__ void fill_wake_neighbours(const FillArgs &a, const float *sW, const float *sZ, int t, int fl, int key,
                                                  RoundCtl *next, int *list_next) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int tyT = t / a.tilesX, txT = t - tyT * a.tilesX;
  const bool n_ok = tyT > 0, s_ok = tyT < a.tilesY - 1, w_ok = txT > 0, e_ok = txT < a.tilesX - 1;
  const int sv = a.round + 1;
  for (int s = threadIdx.x >> 5; s < 4; s += NWARP) {
    const EdgeLine e = edge_line(s);
    unsigned long long word = 0;
    for (int i0 = 0; i0 < e.len; i0 += 32) {
      const int i = i0 + lane;
      const bool above = i < e.len && !(sW[e.o + i * e.st] == sZ[e.zo + i * e.zs]);
      word |= (unsigned long long)__ballot_sync(FULL, above) << i0;
    }
    if (lane == 0) __stcg(&a.edge_above[(size_t)t * 4 + s], word);
    if (!((fl >> 12) & 0xFFFF)) continue;  // nothing changed (warp-uniform)
    if (!TOPO4 && lane == 1 && (fl & (SIDE_NW << s))) {
      // corner s: this tile's corner cell against the diagonal neighbour's, the first or last bit of that neighbour's
      // row next to this tile
      const bool north = s < 2, west = (s & 1) == 0;
      if ((north ? n_ok : s_ok) && (west ? w_ok : e_ok)) {
        const int nb = t + (north ? -a.tilesX : a.tilesX) + (west ? -1 : 1);
        const int own = (north ? SP : TY * SP) + PADL + (west ? 0 : TX - 1);
        const int across = own + (north ? -SP : SP) + (west ? -1 : 1);
        const unsigned long long nword = __ldcg(&a.edge_above[(size_t)nb * 4 + (north ? 1 : 0)]);
        if (((nword >> (west ? TX - 1 : 0)) & 1ull) && sW[own] < sW[across])
          enqueue_tile(a, next, list_next, nb, sv, SIDE_NW << (3 - s), key);
        else if (a.profile)
          atomicAdd(&a.dev->wakes_dropped, 1ull);
      }
    }
    if (!((fl >> s) & 1) || !(s == 0 ? n_ok : s == 1 ? s_ok : s == 2 ? w_ok : e_ok)) continue;  // (warp-uniform)
    const int nb = s == 0 ? t - a.tilesX : s == 1 ? t + a.tilesX : s == 2 ? t - 1 : t + 1;
    const unsigned long long nword = __ldcg(&a.edge_above[(size_t)nb * 4 + (s ^ 1)]);  // its line next to this tile
    bool need = false;
    for (int i = lane; i < e.len; i += 32) {
      if (!((nword >> i) & 1ull)) continue;
      float m = sW[e.o + i * e.st];
      if (!TOPO4) {
        if (i > 0) m = fminf(m, sW[e.o + (i - 1) * e.st]);
        if (i < e.len - 1) m = fminf(m, sW[e.o + (i + 1) * e.st]);
      }
      need |= m < sW[e.o + i * e.st + e.da];
    }
    if (__ballot_sync(FULL, need)) {
      if (lane == 0) enqueue_tile(a, next, list_next, nb, sv, 1 << (s ^ 1), key);
    } else if (lane == 0 && a.profile) {
      atomicAdd(&a.dev->wakes_dropped, 1ull);
    }
  }
}

// STEP = 0: depression filling,     new = min(W, max(Z, min8 W))
// STEP = 1: geodesic distance,      new = min(W, max(Z, 1 + min8 W))   with Z = 0 on cells the flood
//           may enter and +inf elsewhere (used for the flat-resolution gradients, csrc/flats.cu)
// STEP = 2: epsilon fill,           new = min(W, max(Z, next_up(min8 W)))   (FillDepressions(epsilon=True); DESIGN.md
//           3.1).  A fill in everything but the neighbour term: pinned cells, the wake test and the edge flags are the
//           fill's (next_up(e) < W implies e < W, so the fill's wake test wakes a superset of the tiles that can drop).
// TOPO4: the 4-neighbour (D4) stencil of FillDepressions<Topology::D4>; corner aprons are then never read
// STAGE: round 1 of a staged lifted start (a.coarse): W is built from the coarse surface, not loaded, every row is
//        written back, and the tile's Z is saved to a.zcopy through mapZout (a template parameter so that the later
//        rounds keep their registers)
template <int STEP, bool TOPO4 = false, bool STAGE = false>
__global__ void __launch_bounds__(FILL_THREADS, FILL_MIN_CTAS)
    fill_sweep_kernel(const __grid_constant__ CUtensorMap mapW, const __grid_constant__ CUtensorMap mapZ,
                      const __grid_constant__ CUtensorMap mapZout, const __grid_constant__ FillArgs a) {
  // a lifted start bounds the plain fill from above, not the epsilon fill (which lies higher)
  static_assert(!(STAGE && STEP != 0), "the staged lifted round is the plain fill's");
  __shared__ __align__(128) float sW[SROWS * SP];
  __shared__ __align__(128) float sZ[TY * TX];
  __shared__ __align__(8) unsigned long long mbar;
  __shared__ unsigned char sMark[MKP * (BYN + 2)];  // next-pass marks; spare rim so neighbour marks need no bounds checks
  // compacted dirty-block lists, double buffered.  Every warp compacts a fixed share of the blocks
  // into its own segment (ballot + popc, no atomics); a pass walks the concatenation of the segments.
  __shared__ unsigned char sList[2][NWARP][SEG];
  __shared__ __align__(16) int sCnt[2][NWARP];
  __shared__ int sTile;
  __shared__ int sFlags;
  __shared__ int sKey;
  __shared__ int sProf[2];
  __shared__ int sNbDone;  // staged round: neighbours (bit (dy + 1) * 3 + dx + 1) whose cells are in W already

  const int tid = threadIdx.x;
  const int r = a.round;
  RoundCtl *cur = &a.dev->ctl[r % 3];
  RoundCtl *next = &a.dev->ctl[(r + 1) % 3];
  const int *list_cur = (r & 1) ? a.list1 : a.list0;
  int *list_next = (r & 1) ? a.list0 : a.list1;
  const int ntiles = a.tilesX * a.tilesY;
  if (a.use_proc) {  // the admit kernel already split this round's worklist
    cur = &a.dev->proc[r % 3];
    list_cur = a.plist;
  }
  const int n = cur->count;

  if (blockIdx.x == 0 && tid == 0) {
    RoundCtl *z = &a.dev->ctl[(r + 2) % 3];
    z->count = 0;
    z->take = 0;
    RoundCtl *zp = &a.dev->proc[(r + 1) % 3];
    zp->count = 0;
    zp->take = 0;
    if (n > 0) {
      atomicAdd(&a.dev->visits, (unsigned long long)n);
      a.dev->live_rounds++;
    }
  }
  if (n == 0) return;

  if (tid == 0) {
    mbar_init(&mbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  uint32_t phase = 0;
  const int max_iters = a.max_iters;

  for (;;) {
    if (tid == 0) sTile = atomicAdd(&cur->take, 1);
    for (int k = tid; k < MKP * (BYN + 2); k += FILL_THREADS) sMark[k] = 0;
    __syncthreads();  // publishes sTile (and the mbarrier init); all warps are done with smem
    const int li = sTile;
    if (li >= n) break;
    const int t = list_cur[li];
    const int tyT = t / a.tilesX, txT = t - tyT * a.tilesX;
    const int x0 = txT * TX, y0 = tyT * TY;  // raster coords of the tile's first cell

    // ---- stage W (+apron) and Z ----
    constexpr bool stage = STAGE;
    if (tid == 0) {
      sFlags = 0;
      sKey = ORD_POS_INF;
      sProf[0] = sProf[1] = 0;
      if (stage) {
        // neighbours visited earlier in this round have written their cells, and a load of the window would see them
        int nb = 0;
        for (int dy = -1; dy <= 1; dy++)
          for (int dx = -1; dx <= 1; dx++) {
            const int ty = tyT + dy, tx = txT + dx;
            if ((dx | dy) && ty >= 0 && ty < a.tilesY && tx >= 0 && tx < a.tilesX &&
                *reinterpret_cast<volatile int *>(&a.staged[ty * a.tilesX + tx]))
              nb |= 1 << ((dy + 1) * 3 + dx + 1);
          }
        __threadfence();  // their W stores are read after their flags
        sNbDone = nb;
      }
    }
    if (a.use_tma) {
      if (tid == 0) {
        fence_proxy_async();  // order earlier generic-proxy smem accesses before the async writes
        if (STAGE) bulk_wait_read();  // the previous tile's Z store has read sZ
        mbar_arrive_expect_tx(&mbar, (stage ? 0u : W_TILE_BYTES) + Z_TILE_BYTES);
        // the window: cells x0-4..x0+67, y0-1..y0+64 (in place, those outside the raster arrive as zeros: see below)
        if (!stage) tma_load_2d(sW, &mapW, x0 - PADL + a.wox, y0 - 1 + a.woy, &mbar);
        tma_load_2d(sZ, &mapZ, x0 + a.zox, y0 + a.zoy, &mbar);  // the 64x64 interior
      }
    } else {
      // (W % 4 == 0 in place: a float4 lies wholly inside or wholly outside the raster)
      const float inf = __int_as_float(0x7f800000);
      if (!stage) {
        for (int k = tid; k < SROWS * (SP / 4); k += FILL_THREADS) {
          const int rr = k / (SP / 4), cc = k - rr * (SP / 4);
          const int y = y0 + rr - 1, x = x0 + 4 * cc - PADL;  // raster cell of the group's first float
          reinterpret_cast<float4 *>(sW)[k] =
              a.inplace && (y < 0 || y >= a.H || x < 0 || x >= a.W)
                  ? make_float4(inf, inf, inf, inf)
                  : __ldcg(reinterpret_cast<const float4 *>(a.Wp + (size_t)(y + a.woy) * a.pitch + x + a.wox));
        }
      }
      for (int k = tid; k < TY * (TX / 4); k += FILL_THREADS) {
        const int rr = k / (TX / 4), cc = k - rr * (TX / 4);
        reinterpret_cast<float4 *>(sZ)[k] =
            a.inplace && (y0 + rr >= a.H || x0 + 4 * cc >= a.W)
                ? make_float4(inf, inf, inf, inf)
                : __ldg(reinterpret_cast<const float4 *>(a.Z + (size_t)(y0 + a.zoy + rr) * a.zpitch + x0 + a.zox) + cc);
      }
    }
    // ---- initial dirty list from the apron sides that changed (overlaps the TMA flight) ----
    int sides = a.sides[(r & 1) * ntiles + t];
    __syncthreads();  // everyone has read `sides` before it is cleared (and sees sNbDone)
    if (tid == 0) {
      a.sides[(r & 1) * ntiles + t] = 0;
      a.keys[(r & 1) * ntiles + t] = ORD_POS_INF;
    }
    if (stage) {
      // The start W0 of fill_init_kernel<true>, built here instead of loaded: Z on the raster border, +inf outside the
      // raster, elsewhere the coarse level of the cell's pool x pool block.  Apron cells of a neighbour that is done
      // with this round come from W (the caller's raster, where that neighbour has stored its cells).  The raster's
      // border cells are read from Z, i.e. the same raster, which a neighbour may be writing right now: coherent loads,
      // and a border cell holds the same bits either way (W = Z there).
      const float inf = __int_as_float(0x7f800000);
      const int nbdone = sNbDone;
      // each thread builds one group of 4 columns in every RSTEP-th row, so the coarse column is found once per tile
      // and the coarse row advances by a fixed quotient and remainder: no division per group
      constexpr int C4N = SP / 4, RSTEP = FILL_THREADS / C4N;
      static_assert(RSTEP >= 1, "a CTA covers one row of the window");
      if (tid < RSTEP * C4N) {
        const int c4 = 4 * (tid % C4N);
        int rr = tid / C4N;
        const int dx = c4 < PADL ? -1 : (c4 >= PADL + TX ? 1 : 0);
        const int xb = x0 + c4 - PADL;  // raster column of the first of the 4 cells (a multiple of 4)
        const int cx = xb >= 0 ? xb / a.pool : 0, rx = xb - cx * a.pool;  // its coarse column and offset in it
        const int yy = y0 + rr - 1 + a.yoff;  // >= -1
        int cy = (yy + a.pool) / a.pool - 1, ry = yy - cy * a.pool;  // floor division
        const int dq = RSTEP / a.pool, dr = RSTEP - dq * a.pool;
        for (; rr < SROWS; rr += RSTEP) {
          const int dy = rr == 0 ? -1 : (rr == SROWS - 1 ? 1 : 0);
          float4 v4;
          // Only the neighbour's cells inside the raster are read: beside the last tile row its rows, and above or below
          // a partial last tile column its columns, may lie outside (the groups of 4 lie wholly on one side: W % 4 == 0).
          // Those take the branch below, which makes them +inf as the padded layout's padding would be.
          if (((nbdone >> ((dy + 1) * 3 + dx + 1)) & 1) && y0 + rr - 1 < a.H && xb < a.W) {
            v4 = __ldcg(reinterpret_cast<const float4 *>(a.Wp + (size_t)(y0 + rr - 1 + a.woy) * a.pitch + xb + a.wox));
          } else {
            const int y = y0 + rr - 1;
            float v[4] = {inf, inf, inf, inf};
            if (y >= 0 && y < a.H) {
              const float *crow = a.coarse + (size_t)cy * a.Wc;
              const float *zrow = a.Z + (size_t)(y + a.zoy) * a.zpitch + a.zox;
              const bool brow = y == 0 || y == a.H - 1;
              // with pool % 4 == 0 the 4 cells share one coarse block
              const float c0 = (a.pool & 3) == 0 && xb >= 0 && xb < a.W ? __ldg(crow + cx) : inf;
              int cc = cx, rc = rx;
#pragma unroll
              for (int j = 0; j < 4; j++) {
                const int x = xb + j;
                if (j > 0 && ++rc == a.pool) {
                  rc = 0;
                  cc++;
                }
                if (x >= 0 && x < a.W)
                  v[j] = brow || x == 0 || x == a.W - 1 ? __ldcg(zrow + x) : (a.pool & 3) == 0 ? c0 : __ldg(crow + cc);
              }
            }
            v4 = make_float4(v[0], v[1], v[2], v[3]);
          }
          *reinterpret_cast<float4 *>(&sW[rr * SP + c4]) = v4;
          cy += dq;
          ry += dr;
          if (ry >= a.pool) {
            ry -= a.pool;
            cy++;
          }
        }
      }
    }
#include "fill_relax_body.inc"

    // ---- write back + activate neighbours ----
    if (f) {
      atomicOr(&sFlags, f);
      if (f & 0xFF) atomicMin(&sKey, f2ord(kmin));
    }
    __syncthreads();
    const int fl = sFlags;
    const int rowch = (fl >> 12) & 0xFFFF;
    // a staged round writes every row: it is what initialises the tile's cells in W
    const int rowout = stage ? (1 << BYN) - 1 : rowch;
    if (rowout) {
      // coalesced float4 write-back of the block rows (4 cell rows x 64) that hold a change; in place, of their cells
      // inside the raster
      for (int k = tid; k < TY * (TX / 4); k += FILL_THREADS) {
        const int rr = k / (TX / 4), cc = k % (TX / 4);
        const int y = y0 + rr, x = x0 + 4 * cc;
        if ((rowout & (1 << (rr >> 2))) && !(a.inplace && (y >= a.H || x >= a.W))) {
          const float4 val = *reinterpret_cast<const float4 *>(&sW[(rr + 1) * SP + PADL + 4 * cc]);
          __stcg(reinterpret_cast<float4 *>(a.Wp + (size_t)(y + a.woy) * a.pitch + x + a.wox), val);
          // (without TMA the staged round saves its Z here)
          if (STAGE && !a.use_tma)
            __stcg(reinterpret_cast<float4 *>(a.zcopy + (size_t)y * a.W + x),
                   *reinterpret_cast<const float4 *>(&sZ[rr * TX + 4 * cc]));
        }
      }
    }
    if (stage) {
      __syncthreads();  // every cell of the tile is stored ...
      if (tid == 0) {
        __threadfence();  // ... and visible to the GPU before the flag
        atomicExch(&a.staged[t], 1);
      }
    }
    if (STEP != 1 && WAKE_WORDS && a.edge_above) {
      // (not inlined: the relaxation above keeps its registers)
      fill_wake_neighbours<TOPO4>(a, sW, sZ, t, fl, sKey, next, list_next);
      if (rowch && tid == 0) {
        if (fl & (3 << 9)) atomicOr(&a.dev->edge_changed, (fl >> 9) & 3);
        if (a.dirty) a.dirty[t] = 1;
      }
    } else if (rowch) {
      if (tid < 8) {
        // one thread per neighbour: the enqueue atomics (or + exch + add) overlap instead of
        // queueing behind each other on a single thread
        const int sv = r + 1;
        const bool n_ok = tyT > 0, s_ok = tyT < a.tilesY - 1, w_ok = txT > 0, e_ok = txT < a.tilesX - 1;
        int nb = -1, bits = 0;
        switch (tid) {
          case 0: if ((fl & SIDE_N) && n_ok) { nb = t - a.tilesX; bits = SIDE_S; } break;
          case 1: if ((fl & SIDE_S) && s_ok) { nb = t + a.tilesX; bits = SIDE_N; } break;
          case 2: if ((fl & SIDE_W) && w_ok) { nb = t - 1; bits = SIDE_E; } break;
          case 3: if ((fl & SIDE_E) && e_ok) { nb = t + 1; bits = SIDE_W; } break;
          case 4: if ((fl & SIDE_NW) && n_ok && w_ok) { nb = t - a.tilesX - 1; bits = SIDE_SE; } break;
          case 5: if ((fl & SIDE_NE) && n_ok && e_ok) { nb = t - a.tilesX + 1; bits = SIDE_SW; } break;
          case 6: if ((fl & SIDE_SW) && s_ok && w_ok) { nb = t + a.tilesX - 1; bits = SIDE_NE; } break;
          default: if ((fl & SIDE_SE) && s_ok && e_ok) { nb = t + a.tilesX + 1; bits = SIDE_NW; } break;
        }
        if (nb >= 0) enqueue_tile(a, next, list_next, nb, sv, bits, sKey);
        if (tid == 0 && (fl & (3 << 9))) atomicOr(&a.dev->edge_changed, (fl >> 9) & 3);
        if (tid == 0 && a.dirty) a.dirty[t] = 1;
      }
    }
    if (tid == 0) {
      if (again) enqueue_tile(a, next, list_next, t, r + 1, SIDE_FULL, f2ord(-__int_as_float(0x7f800000)));
      atomicAdd(&a.dev->iters, (unsigned long long)iters);
      if (a.profile) {
        if (!rowch) atomicAdd(&a.dev->idle_visits, 1ull);
        atomicAdd(&a.dev->block_updates, (unsigned long long)sProf[0]);
        atomicAdd(&a.dev->warp_updates, (unsigned long long)sProf[1]);
        const int hb = iters <= 1 ? 0 : iters <= 2 ? 1 : iters <= 4 ? 2 : iters <= 8 ? 3 : iters <= 16 ? 4 : iters <= 32 ? 5 : iters <= 64 ? 6 : 7;
        atomicAdd(&a.dev->iter_hist[hb], 1ull);
      }
    }
  }
  if (STAGE && a.use_tma && tid == 0) bulk_wait_all();  // the Z stores are done before the CTA's shared memory goes
}

// ---- level-ordered mode: split the round's worklist into admitted / postponed tiles ----------
// Tiles whose lowest incoming water level is above the round's level are carried over to the next
// round untouched (their side masks and keys move to the other parity); flooding then proceeds
// roughly in order of rising water level, as the serial priority flood does, which avoids
// flooding a tile with a high level that a lower one will overwrite later.
__global__ void __launch_bounds__(256) fill_admit_kernel(const FillArgs a) {
  const int r = a.round;
  const RoundCtl *cur = &a.dev->ctl[r % 3];
  RoundCtl *next = &a.dev->ctl[(r + 1) % 3];
  RoundCtl *proc = &a.dev->proc[r % 3];
  const int *list_cur = (r & 1) ? a.list1 : a.list0;
  int *list_next = (r & 1) ? a.list0 : a.list1;
  const int n = cur->count;
  const int ntiles = a.tilesX * a.tilesY;
  const float level = a.level;
  int nd = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int t = list_cur[i];
    const int kord = a.keys[(r & 1) * ntiles + t];
    if (ord2f(kord) <= level) {
      a.plist[atomicAdd(&proc->count, 1)] = t;
    } else {
      int bits = a.sides[(r & 1) * ntiles + t];
      if (bits == 0) bits = SIDE_FULL;
      a.sides[(r & 1) * ntiles + t] = 0;
      a.keys[(r & 1) * ntiles + t] = ORD_POS_INF;
      enqueue_tile(a, next, list_next, t, r + 1, bits, kord);
      nd++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) nd += __shfl_xor_sync(0xffffffffu, nd, o);
  if ((threadIdx.x & 31) == 0 && nd) atomicAdd(&a.dev->ndefer[r % 3], nd);
}

// host-chosen seeds (perimeter tiles at the start, tiles next to a replaced ghost row later)
__global__ void __launch_bounds__(256) fill_seed_kernel(const FillArgs a, const int *__restrict__ tiles, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = a.round;
  // enqueue_tile() targets round `stampval`: here the round about to be launched
  RoundCtl *cur = &a.dev->ctl[r % 3];
  int *list_cur = (r & 1) ? a.list1 : a.list0;
  enqueue_tile(a, cur, list_cur, tiles[i], r, SIDE_FULL, f2ord(-__int_as_float(0x7f800000)));
}

// tiles flagged on the device (prolongation, restriction into a coarse level): same as fill_seed_kernel without the
// trip through the host
__global__ void __launch_bounds__(256) fill_seed_flags_kernel(const FillArgs a, const int *__restrict__ flag, int ntiles,
                                                               int *count) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles || !flag[t]) return;
  const int r = a.round;
  RoundCtl *cur = &a.dev->ctl[r % 3];
  int *list_cur = (r & 1) ? a.list1 : a.list0;
  enqueue_tile(a, cur, list_cur, t, r, SIDE_FULL, f2ord(-__int_as_float(0x7f800000)));
  if (count) atomicAdd(count, 1);
}

// row-band fill: ghost row y of the padded arrays takes the neighbouring band's edge row where that is lower (ghost cells
// are boundary conditions: Z = W), and the tiles whose cells or aprons changed are flagged
__global__ void __launch_bounds__(256) fill_ghost_update_kernel(float *Wp, float *Zp, int pitch, int W, int H, int y,
                                                                 const float *__restrict__ row, int *tile_flag, int tilesX,
                                                                 int *lowered) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  const size_t o = (size_t)(y + 1) * pitch + x + PADL;
  const float v = row[x];
  if (v < Wp[o]) {
    Wp[o] = v;
    Zp[o] = v;
    *lowered = 1;
    const int ya = y > 0 ? y - 1 : 0, yb = y < H - 1 ? y + 1 : H - 1, xa = x > 0 ? x - 1 : 0, xb = x < W - 1 ? x + 1 : W - 1;
    const int ty0 = ya / TY, ty1 = yb / TY, tx0 = xa / TX, tx1 = xb / TX;
    tile_flag[ty0 * tilesX + tx0] = 1;
    if (tx1 != tx0) tile_flag[ty0 * tilesX + tx1] = 1;
    if (ty1 != ty0) {
      tile_flag[ty1 * tilesX + tx0] = 1;
      if (tx1 != tx0) tile_flag[ty1 * tilesX + tx1] = 1;
    }
  }
}

// a ghost row of the band's raster starts at its lifted level: the water level of its k x k block in the coarse fill
__global__ void __launch_bounds__(256) fill_lift_row_kernel(float *row, int W, const float *__restrict__ coarse_row, int k) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x < W) row[x] = coarse_row[x / k];
}

// ---- layout kernels ----------------------------------------------------------------------
// compact dem (H x W) -> Z and W in a `pitch` x `rows` layout whose cell (x, y) sits at (x + ox, y + oy): the padded
// pair (PADL, 1), or in place (0, 0; Wo may be `dem` itself, each thread reads its cells before it writes them).  Border
// cells (all four sides of the raster handed in) are boundary conditions: W = Z = dem there; interior W = +inf; padding
// Z = W = +inf.
// LIFT (fill_multigrid): interior cells start at the water level of their pool x pool block in the filled max-pooled
// raster `coarse` (an upper bound of the answer, see fill_depressions_dev) instead of +inf.
// Cells equal to `pin` are boundary conditions too (the epsilon fill's NoData; NaN pins nothing).
template <bool LIFT>
__global__ void fill_init_kernel(const float *dem, float *__restrict__ Zo, float *Wo, int W, int H, int pitch, int rows,
                                 int ox, int oy, FillDev *dev, const float *__restrict__ coarse, int Wc, int pool, int yoff,
                                 float pin) {
  const int px4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;  // layout column (multiple of 4)
  const float inf = __int_as_float(0x7f800000);
  float lo = inf, hi = -inf;
  for (int py = blockIdx.y; py < rows && px4 < pitch; py += gridDim.y) {
    float zv[4], wv[4];
    const int y = py - oy;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int x = px4 + k - ox;
      float zz = inf, ww = inf;
      if (x >= 0 && x < W && y >= 0 && y < H) {
        zz = dem[(size_t)y * W + x];
        const bool border = (x == 0) | (y == 0) | (x == W - 1) | (y == H - 1) | (zz == pin);
        ww = border ? zz : (LIFT ? __ldg(coarse + (size_t)((y + yoff) / pool) * Wc + x / pool) : inf);
        if (zz < inf && zz > -inf) {
          lo = fminf(lo, zz);
          hi = fmaxf(hi, zz);
        }
      }
      zv[k] = zz;
      wv[k] = ww;
    }
    const size_t o = (size_t)py * pitch + px4;
    *reinterpret_cast<float4 *>(Zo + o) = make_float4(zv[0], zv[1], zv[2], zv[3]);
    *reinterpret_cast<float4 *>(Wo + o) = make_float4(wv[0], wv[1], wv[2], wv[3]);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __shared__ float slo[4], shi[4];  // blockDim.x == 128
  if ((threadIdx.x & 31) == 0) {
    slo[threadIdx.x >> 5] = lo;
    shi[threadIdx.x >> 5] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    lo = fminf(fminf(slo[0], slo[1]), fminf(slo[2], slo[3]));
    hi = fmaxf(fmaxf(shi[0], shi[1]), fmaxf(shi[2], shi[3]));
    if (lo <= hi) {
      atomicMin(&dev->zmin_ord, f2ord(lo));
      atomicMax(&dev->zmax_ord, f2ord(hi));
    }
  }
}

// sampled histogram of the input elevations (every `row_stride`-th row of `ncols` x `nrows` floats, row pitch `zpitch`;
// +inf padding is skipped) for the level schedule
constexpr int HIST_BINS = 1024;
__global__ void __launch_bounds__(256) fill_hist_kernel(const float *__restrict__ Z, int zpitch, int ncols, int nrows,
                                                         int row_stride, float zmin, float inv_range, unsigned int *hist) {
  __shared__ unsigned int sh[HIST_BINS];
  for (int k = threadIdx.x; k < HIST_BINS; k += blockDim.x) sh[k] = 0;
  __syncthreads();
  const int row = blockIdx.x * row_stride;
  if (row < nrows) {
    for (int x = threadIdx.x; x < ncols; x += blockDim.x) {
      const float zv = Z[(size_t)row * zpitch + x];
      if (zv < __int_as_float(0x7f800000) && zv > -__int_as_float(0x7f800000)) {
        int b = (int)((zv - zmin) * inv_range * HIST_BINS);
        b = b < 0 ? 0 : (b >= HIST_BINS ? HIST_BINS - 1 : b);
        atomicAdd(&sh[b], 1u);
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < HIST_BINS; k += blockDim.x)
    if (sh[k]) atomicAdd(&hist[k], sh[k]);
}

// distance mode: padded Z = 0 where `open[i]` has bit `open_bit` (cells the flood may enter), +inf
// elsewhere; padded W = winit (compact float array: +inf, or the seed distance)
__global__ void __launch_bounds__(128) dist_pad_init_kernel(const uint8_t *__restrict__ open, int open_bit,
                                                             const float *__restrict__ winit, float *__restrict__ Zp,
                                                             float *__restrict__ Wp, int W, int H, int pitch, int rows,
                                                             int ghost_top, int ghost_bottom, int *tile_flag, int tilesX) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= pitch) return;
  const float inf = __int_as_float(0x7f800000);
  for (int py = blockIdx.y; py < rows; py += gridDim.y) {
    const int x = px - PADL, y = py - 1;
    float zz = inf, ww = inf;
    if (x >= 0 && x < W && y >= 0 && y < H) {
      const size_t i = (size_t)y * W + x;
      // ghost rows of a row band start closed (+inf): they only ever hold what the neighbour sends
      if (!((ghost_top && y == 0) || (ghost_bottom && y == H - 1))) {
        if (open[i] & open_bit) zz = 0.0f;
        ww = winit[i];
        if (ww < inf) {
          // only tiles that can see a seed (inside, or in their apron) have anything to do in the first round
          const int ya = y > 0 ? y - 1 : 0, yb = y < H - 1 ? y + 1 : H - 1, xa = x > 0 ? x - 1 : 0, xb = x < W - 1 ? x + 1 : W - 1;
          const int ty0 = ya / TY, ty1 = yb / TY, tx0 = xa / TX, tx1 = xb / TX;
          tile_flag[ty0 * tilesX + tx0] = 1;
          if (tx1 != tx0) tile_flag[ty0 * tilesX + tx1] = 1;
          if (ty1 != ty0) {
            tile_flag[ty1 * tilesX + tx0] = 1;
            if (tx1 != tx0) tile_flag[ty1 * tilesX + tx1] = 1;
          }
        }
      }
    }
    Zp[(size_t)py * pitch + px] = zz;
    Wp[(size_t)py * pitch + px] = ww;
  }
}

__global__ void fill_i32_kernel(int *p, int v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// k x k max-pooling of rows [yoff, yoff + H) of a raster into the coarse rows they touch (ragged last row / column
// of blocks included).  `combine`: max with what `dst` already holds (a band covers part of a block row).
__global__ void __launch_bounds__(256) fill_maxpool_kernel(const float *__restrict__ src, int W, int H, int yoff, float *dst, int Wc,
                                                            int Hc, int k, int combine) {
  const int bx = blockIdx.x * blockDim.x + threadIdx.x;
  if (bx >= Wc) return;
  const int by_lo = yoff / k, by_hi = (yoff + H - 1) / k;
  for (int by = by_lo + blockIdx.y; by <= by_hi && by < Hc; by += gridDim.y) {
    float m = -__int_as_float(0x7f800000);
    const bool vec = (k & 3) == 0 && (W & 3) == 0 && bx * k + k <= W && ((uintptr_t)src & 15) == 0;
    for (int j = 0; j < k; j++) {
      const int y = by * k + j - yoff;  // local row
      if (y < 0) continue;
      if (y >= H) break;
      if (vec) {
        const float4 *row = reinterpret_cast<const float4 *>(src + (size_t)y * W + bx * k);
        for (int i = 0; i < k / 4; i++) {
          const float4 q = __ldg(row + i);
          m = fmaxf(fmaxf(m, fmaxf(q.x, q.y)), fmaxf(q.z, q.w));
        }
      } else {
        for (int i = 0; i < k; i++) {
          const int x = bx * k + i;
          if (x < W) m = fmaxf(m, __ldg(src + (size_t)y * W + x));
        }
      }
    }
    float *o = dst + (size_t)by * Wc + bx;
    *o = combine ? fmaxf(*o, m) : m;
  }
}

// V-cycle (fill_vcycle): restriction -- the coarse surface drops to the block maximum of the current fine surface
// wherever that is lower (both are upper bounds of the answer for every cell of the block) ...
// The fine surface's cell (x, y) is at Wp[(y + woy) * pitch + x + wox] (see FillState::Wb).  The coarse surface is the
// water-level array of the coarse level's own solver (cell (bx, by) at Wc[(by + coy) * cpitch + bx + cox]); coarse tiles
// that hold a lowered cell -- and their neighbours when the cell sits on a tile edge -- are flagged for that solver's next
// run.  `dirty` (may be null; used when k divides the tile shape): only blocks inside fine tiles that were written since
// the last restriction are looked at.
__global__ void __launch_bounds__(256) fill_restrict_kernel(const float *__restrict__ Wp, int pitch, int wox, int woy, int W,
                                                             int H, float *Wc, int cpitch, int cox, int coy, int Wcw, int Hc,
                                                             int k, const int *__restrict__ dirty, int tilesX,
                                                             int *ctile_flag, int ctilesX) {
  const int bx = blockIdx.x * blockDim.x + threadIdx.x;
  if (bx >= Wcw) return;
  for (int by = blockIdx.y; by < Hc; by += gridDim.y) {
    if (dirty && !dirty[((by * k) / TY) * tilesX + (bx * k) / TX]) continue;
    float m = -__int_as_float(0x7f800000);
    // whole block inside the raster: 16-byte loads (pitch and wox are multiples of 4 in both layouts)
    if ((k & 3) == 0 && bx * k + k <= W && by * k + k <= H) {
      for (int j = 0; j < k; j++) {
        const float4 *row = reinterpret_cast<const float4 *>(Wp + (size_t)(by * k + j + woy) * pitch + bx * k + wox);
        for (int i = 0; i < k / 4; i++) {
          const float4 q = __ldcg(row + i);
          m = fmaxf(fmaxf(m, fmaxf(q.x, q.y)), fmaxf(q.z, q.w));
        }
      }
    } else {
      for (int j = 0; j < k; j++) {
        const int y = by * k + j;
        if (y >= H) break;
        for (int i = 0; i < k; i++) {
          const int x = bx * k + i;
          if (x < W) m = fmaxf(m, __ldcg(Wp + (size_t)(y + woy) * pitch + x + wox));
        }
      }
    }
    float *o = Wc + (size_t)(by + coy) * cpitch + bx + cox;
    if (m < *o && bx > 0 && by > 0 && bx < Wcw - 1 && by < Hc - 1) {  // border blocks stay pinned at their elevation
      *o = m;
      const int ty0 = (by - 1) / TY, ty1 = (by + 1) / TY, tx0 = (bx - 1) / TX, tx1 = (bx + 1) / TX;
      ctile_flag[ty0 * ctilesX + tx0] = 1;
      if (tx1 != tx0) ctile_flag[ty0 * ctilesX + tx1] = 1;
      if (ty1 != ty0) {
        ctile_flag[ty1 * ctilesX + tx0] = 1;
        if (tx1 != tx0) ctile_flag[ty1 * ctilesX + tx1] = 1;
      }
    }
  }
}

// band variant of the restriction: block maxima of rows [y_lo, y_hi) of a band whose row 0 is global row `yoff`,
// max-combined into the full coarse array `out` (pre-filled with -inf; merged across bands by a MAX all-reduce)
// `dirty` (may be null; used when k divides the tile shape and the band starts on a block boundary): blocks inside fine
// tiles that no sweep has written since the last call report +inf, i.e. "leave the coarse level as it is".
__global__ void __launch_bounds__(256) fill_blockmax_kernel(const float *__restrict__ Wp, int pitch, int wox, int woy, int W,
                                                             int y_lo, int y_hi,
                                                             int yoff, float *out, int Wcw, int Hc, int k,
                                                             const int *__restrict__ dirty, int tilesX) {
  const int bx = blockIdx.x * blockDim.x + threadIdx.x;
  if (bx >= Wcw) return;
  const int by_lo = (yoff + y_lo) / k, by_hi = (yoff + y_hi - 1) / k;
  for (int by = by_lo + blockIdx.y; by <= by_hi && by < Hc; by += gridDim.y) {
    if (dirty) {
      // local rows of the block, clipped to the owned rows; with a ghost row on top they can straddle two tile rows
      int l0 = by * k - yoff, l1 = l0 + k - 1;
      l0 = l0 < y_lo ? y_lo : l0;
      l1 = l1 >= y_hi ? y_hi - 1 : l1;
      const int tx = (bx * k) / TX;
      if (!dirty[(l0 / TY) * tilesX + tx] && !dirty[(l1 / TY) * tilesX + tx]) {
        out[(size_t)by * Wcw + bx] = __int_as_float(0x7f800000);
        continue;
      }
    }
    float m = -__int_as_float(0x7f800000);
    for (int j = 0; j < k; j++) {
      const int y = by * k + j - yoff;  // local row
      if (y < y_lo) continue;
      if (y >= y_hi) break;
      for (int i = 0; i < k; i++) {
        const int x = bx * k + i;
        if (x < W) m = fmaxf(m, __ldcg(Wp + (size_t)(y + woy) * pitch + x + wox));
      }
    }
    float *o = out + (size_t)by * Wcw + bx;
    *o = fmaxf(*o, m);
  }
}

// ... and prolongation: every interior fine cell drops to its block's (re-relaxed) coarse level where that is lower;
// the tiles that hold such a cell -- and the neighbouring tiles whose apron it is part of -- are flagged so that the
// sweep looks at them again.  The fine surface's cell (x, y) is at Wp[(y + woy) * pitch + x + wox], the coarse one's at
// Wc[(by + coff_y) * cpitch + bx + coff_x] (a compact array or a solver in place: offsets 0; a padded solver: 1 and
// PADL).  One block per fine tile; `cdirty` (may be null): tiles whose blocks all lie in coarse tiles that the coarse
// relaxation did not write are skipped.
__global__ void __launch_bounds__(256) fill_prolong_kernel(float *Wp, int pitch, int wox, int woy, int W, int H,
                                                            const float *__restrict__ Wc,
                                                            int cpitch, int coff_x, int coff_y, int k, int *tile_flag,
                                                            int tilesX, int yoff, const int *__restrict__ cdirty,
                                                            int ctilesX) {
  const int t = blockIdx.x;
  const int tyT = t / tilesX, txT = t - tyT * tilesX;
  const int x0 = txT * TX, y0 = tyT * TY;
  if (cdirty) {
    // coarse cells of this tile: columns x0/k .. (x0+TX-1)/k, rows (y0+yoff)/k .. ; at most 2 x 2 coarse tiles
    const int cx0 = (x0 / k) / TX, cx1 = ((x0 + TX - 1) / k) / TX;
    const int cy0 = ((y0 + yoff) / k) / TY, cy1 = ((y0 + TY - 1 + yoff) / k) / TY;
    bool any = false;
    for (int cy = cy0; cy <= cy1; cy++)
      for (int cx = cx0; cx <= cx1; cx++) any |= cdirty[cy * ctilesX + cx] != 0;
    if (!any) return;
  }
  bool lowered = false, lo_n = false, lo_s = false, lo_w = false, lo_e = false;
  for (int g = threadIdx.x; g < TX * TY / 4; g += blockDim.x) {  // 4 cells per thread and step (16-byte accesses)
    const int ly = g / (TX / 4), lx4 = (g - ly * (TX / 4)) * 4;
    const int y = y0 + ly;
    // (in place W % 4 == 0: the 4 cells lie wholly inside or wholly outside the raster)
    if (y < 1 || y >= H - 1 || x0 + lx4 >= W) continue;
    float4 *wp4 = reinterpret_cast<float4 *>(Wp + (size_t)(y + woy) * pitch + x0 + lx4 + wox);
    const float4 w4 = *wp4;
    float wv[4] = {w4.x, w4.y, w4.z, w4.w};
    const float *crow = Wc + (size_t)((y + yoff) / k + coff_y) * cpitch + coff_x;
    bool any = false;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int lx = lx4 + j, x = x0 + lx;
      if (x < 1 || x >= W - 1) continue;
      const float l = __ldg(crow + x / k);
      if (l < wv[j]) {
        wv[j] = l;
        any = true;
        lo_w |= lx == 0;
        lo_e |= lx == TX - 1;
      }
    }
    if (any) {
      *wp4 = make_float4(wv[0], wv[1], wv[2], wv[3]);
      lowered = true;
      lo_n |= ly == 0;
      lo_s |= ly == TY - 1;
    }
  }
  // a lowered cell on a tile edge is also part of the neighbouring tiles' aprons: wake every tile that reads it
  if (lowered) {
    const int tilesY = (H + TY - 1) / TY;
    tile_flag[t] = 1;
    const bool n_ok = tyT > 0, s_ok = tyT < tilesY - 1, w_ok = txT > 0, e_ok = txT < tilesX - 1;
    if (lo_n && n_ok) tile_flag[t - tilesX] = 1;
    if (lo_s && s_ok) tile_flag[t + tilesX] = 1;
    if (lo_w && w_ok) tile_flag[t - 1] = 1;
    if (lo_e && e_ok) tile_flag[t + 1] = 1;
    if (lo_n && lo_w && n_ok && w_ok) tile_flag[t - tilesX - 1] = 1;
    if (lo_n && lo_e && n_ok && e_ok) tile_flag[t - tilesX + 1] = 1;
    if (lo_s && lo_w && s_ok && w_ok) tile_flag[t + tilesX - 1] = 1;
    if (lo_s && lo_e && s_ok && e_ok) tile_flag[t + tilesX + 1] = 1;
  }
}

// W (cell (x, y) at Wp[(y + woy) * pitch + x + wox]) -> the caller's compact raster.  W % 4 == 0 version: 16-byte loads
// and stores (rows start 16-byte aligned at column wox)
__global__ void __launch_bounds__(256) fill_finish_x4_kernel(const float *__restrict__ Wp, float *__restrict__ out, int W,
                                                              int H, int pitch, int wox, int woy) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const float4 v = __ldcs(reinterpret_cast<const float4 *>(Wp + (size_t)(y + woy) * pitch + x4 + wox));
    __stcs(reinterpret_cast<float4 *>(out + (size_t)y * W + x4), v);
  }
}

__global__ void fill_finish_kernel(const float *__restrict__ Wp, float *__restrict__ out, int W, int H,
                                   int pitch, int wox, int woy) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= W) return;
  for (int y = blockIdx.y; y < H; y += gridDim.y) out[(size_t)y * W + x] = Wp[(size_t)(y + woy) * pitch + x + wox];
}

// ---- host side ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    RDB_CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) fail("cuTensorMapEncodeTiled not available from the driver");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

CUtensorMap make_map(float *base, int pitch, int rows, int boxw, int boxh) {
  CUtensorMap m;
  const cuuint64_t gdim[2] = {(cuuint64_t)pitch, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)pitch * 4};
  const cuuint32_t box[2] = {(cuuint32_t)boxw, (cuuint32_t)boxh};
  const cuuint32_t estr[2] = {1, 1};
  CUresult rc = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) fail("cuTensorMapEncodeTiled failed with CUresult %d", (int)rc);
  return m;
}

}  // namespace

struct FillState {
  int W = 0, H = 0, pitch = 0, rows = 0, tilesX = 0, tilesY = 0;
  DevBuf<float> Zp, Wp;
  DevBuf<int> list0, list1, plist, stamp, sides, keys;
  DevBuf<int> dirty, tflag;  // V-cycle bookkeeping: tiles written since the last look / tiles to wake (both per tile)
  DevBuf<int> staged;        // staged lifted start: tiles the first round has written (per tile)
  DevBuf<unsigned long long> edge_above;  // fill: 4 words per tile for the wake test (FillArgs::edge_above)
  float zmin = 0.f, zmax = 0.f;
  bool first_run = true;
  bool ordered = false;
  int step_mode = 0;  // 0: fill, 1: geodesic distance, 2: epsilon fill (fill_sweep_kernel<STEP>)
  bool topo4 = false;  // D4 fill (4-neighbour stencil)
  float pin = __builtin_nanf("");  // cells equal to it are pinned like the raster's border (epsilon fill: NoData)
  std::vector<float> levels;
  DevBuf<FillDev> dev;
  CUtensorMap mapW, mapZ;
  int round = 0;
  int grid = 0;
  int64_t rounds_run = 0;   // sweep launches
  int64_t live_rounds = 0;  // ... that found a non-empty worklist (the dependent rounds of the flood)
  int64_t visits_seen = 0;  // tile visits so far (as of the last read-back)
  bool still_active = false;
  int64_t sched_round = 0;

  // Where W lives: cell (x, y) at Wb[(y + woy) * wpitch + x + wox].  Padded layout: Wp (pitch, PADL, 1), with Z in Zp.
  // In place: the caller's raster (W, 0, 0), with Z in the compact copy Zc.
  float *Wb = nullptr;
  int wpitch = 0, wox = 0, woy = 0;
  bool inplace = false;
  DevBuf<float> Zc;
  // staged lifted start: the first sweep round builds W from this coarse surface, reads Z from the caller's raster and
  // saves it to Zc (see fill_sweep_kernel)
  const float *stage_coarse = nullptr;
  int stage_wc = 0, stage_k = 1, stage_yoff = 0;
  CUtensorMap mapZstage;  // the caller's raster as Z (staged round)

  void use_padded_layout(size_t np) {
    inplace = false;
    Zc.reset();
    Zp.alloc(np);
    Wp.alloc(np);
    Wb = Wp.p;
    wpitch = pitch;
    wox = PADL;
    woy = 1;
  }

  // in_place: the caller hands its raster over for the whole solve (no row updates): W is relaxed in it, Z is kept in a
  // compact copy.  Taken when TMA can address the raster: width a multiple of 4, 16-byte aligned (fill_external_z = 0
  // turns it off).  With a lifted start the first round then builds its W from the coarse surface and saves Z as it goes
  // (no pass over the raster beforehand); otherwise the padded layout holds a copy of both.
  void begin(const float *d_dem, int w, int h, const float *d_coarse = nullptr, int coarse_w = 0, int coarse_k = 0,
             int coarse_yoff = 0, bool in_place = false) {
    Ctx &c = ctx();
    W = w;
    H = h;
    tilesX = (w + TX - 1) / TX;
    tilesY = (h + TY - 1) / TY;
    pitch = tilesX * TX + 2 * PADL;
    rows = tilesY * TY + 2;
    const size_t np = (size_t)pitch * rows;
    if (in_place && c.params.fill_external_z != 0 && (w & 3) == 0 && ((uintptr_t)d_dem & 15) == 0) {
      inplace = true;
      Zp.reset();
      Wp.reset();
      Zc.alloc((size_t)w * h);
      Wb = const_cast<float *>(d_dem);  // (in_place: the caller's raster is writable)
      wpitch = w;
      wox = woy = 0;
    } else {
      use_padded_layout(np);
    }
    stage_coarse = inplace && d_coarse ? d_coarse : nullptr;
    stage_wc = coarse_w;
    stage_k = coarse_k;
    stage_yoff = coarse_yoff;
    const size_t nt = (size_t)tilesX * tilesY;
    list0.alloc(nt);
    list1.alloc(nt);
    plist.alloc(nt);
    stamp.alloc(nt);
    sides.alloc(2 * nt);
    keys.alloc(2 * nt);
    dev.alloc(1);
    RDB_CK(cudaMemsetAsync(stamp.p, 0, nt * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(sides.p, 0, 2 * nt * sizeof(int), c.stream));
    if (stage_coarse) {
      staged.alloc(nt);
      RDB_CK(cudaMemsetAsync(staged.p, 0, nt * sizeof(int), c.stream));
    }
    // every cell may be above its Z until its tile's first visit says otherwise (whatever the start: +inf, lifted in
    // place or padded, staged, a band's, fill_relax_from's)
    edge_above.alloc(4 * nt);
    RDB_CK(cudaMemsetAsync(edge_above.p, 0xff, 4 * nt * sizeof(unsigned long long), c.stream));
    {
      FillDev h0;
      memset(&h0, 0, sizeof(h0));
      h0.zmin_ord = ORD_POS_INF;
      h0.zmax_ord = f2ord(-__builtin_inff());
      memcpy(c.pinned, &h0, sizeof(h0));
      RDB_CK(cudaMemcpyAsync(dev.p, c.pinned, sizeof(FillDev), cudaMemcpyHostToDevice, c.stream));
      // keys start at +inf (0x7f800000 repeated is not a byte pattern: fill with a tiny kernel-free trick:
      // ORD_POS_INF = 0x7f800000 -> use cudaMemsetD32-equivalent via cuMemset is driver API; a 1-line kernel is simpler)
    }
    {
      const int n2 = (int)(2 * nt);
      fill_i32_kernel<<<(n2 + 255) / 256, 256, 0, c.stream>>>(keys.p, ORD_POS_INF, n2);
      count_launch();
      dim3 blk(128), grd((pitch / 4 + 127) / 128, rows < 2048 ? rows : 2048);
      if (stage_coarse) {
        // nothing to do: the first round writes every tile's cells (zmin / zmax serve the level schedule, which a lifted
        // start does not use)
      } else if (inplace) {
        dim3 grdc((W / 4 + 127) / 128, H < 2048 ? H : 2048);
        fill_init_kernel<false><<<grdc, blk, 0, c.stream>>>(d_dem, Zc.p, Wb, W, H, W, H, 0, 0, dev.p, nullptr, 0, 1, 0, pin);
        count_launch();
      } else if (d_coarse) {
        fill_init_kernel<true><<<grd, blk, 0, c.stream>>>(d_dem, Zp.p, Wp.p, W, H, pitch, rows, PADL, 1, dev.p, d_coarse,
                                                         coarse_w, coarse_k, coarse_yoff, pin);
        count_launch();
      } else {
        fill_init_kernel<false><<<grd, blk, 0, c.stream>>>(d_dem, Zp.p, Wp.p, W, H, pitch, rows, PADL, 1, dev.p, nullptr, 0, 1,
                                                          0, pin);
        count_launch();
      }
      RDB_CK(cudaGetLastError());
      zmin = zmax = 0.f;
      if (!d_coarse) {
        FillDev *hd = (FillDev *)c.pinned;
        RDB_CK(cudaMemcpyAsync(hd, dev.p, sizeof(FillDev), cudaMemcpyDeviceToHost, c.stream));
        RDB_CK(cudaStreamSynchronize(c.stream));
        zmin = ord2f(hd->zmin_ord);
        zmax = ord2f(hd->zmax_ord);
        if (!(zmin <= zmax)) zmin = zmax = 0.f;
      }
      // a lifted start (fill_multigrid) is already close to the answer everywhere: no level schedule
      ordered = c.params.fill_ordered != 0 && zmax > zmin && !d_coarse;
      levels.clear();
      if (ordered) {
        // Level schedule: round k admits tiles whose incoming water level is below the k/R quantile of
        // the input elevations, so about the same number of cells becomes floodable every round.
        int64_t R = c.params.fill_order_rounds;
        if (R <= 0) R = (int64_t)(0.8 * (tilesX > tilesY ? tilesX : tilesY));
        if (R < 8) {
          ordered = false;
        } else {
          DevBuf<unsigned int> hist(HIST_BINS);
          RDB_CK(cudaMemsetAsync(hist.p, 0, HIST_BINS * sizeof(unsigned int), c.stream));
          const int stride = rows > 4096 ? 16 : (rows > 512 ? 4 : 1);
          const int nb = (rows - 2 + stride - 1) / stride;
          // (padded rows 1, 1 + stride, ... are raster rows 0, stride, ...)
          if (inplace)  // (the caller's raster holds W by now)
            fill_hist_kernel<<<nb, 256, 0, c.stream>>>(Zc.p, W, W, H, stride, zmin, 1.0f / (zmax - zmin), hist.p);
          else
            fill_hist_kernel<<<nb, 256, 0, c.stream>>>(Zp.p + pitch, pitch, pitch, rows - 1, stride, zmin, 1.0f / (zmax - zmin),
                                                       hist.p);
          RDB_CK(cudaGetLastError());
          count_launch();
          unsigned int *hh = (unsigned int *)c.pinned;
          RDB_CK(cudaMemcpyAsync(hh, hist.p, HIST_BINS * sizeof(unsigned int), cudaMemcpyDeviceToHost, c.stream));
          RDB_CK(cudaStreamSynchronize(c.stream));
          double total = 0;
          for (int k = 0; k < HIST_BINS; k++) total += hh[k];
          levels.resize((size_t)R);
          double cum = 0;
          int bin = 0;
          for (int64_t k = 0; k < R; k++) {
            const double want = total * (double)(k + 1) / (double)R;
            while (bin < HIST_BINS - 1 && cum + hh[bin] < want) cum += hh[bin++];
            levels[(size_t)k] = zmin + (zmax - zmin) * (float)(bin + 1) / (float)HIST_BINS;
          }
        }
      }
    }
    if (inplace) {
      // (TMA fills the box cells beyond the raster's edges with zeros; the sweep overwrites them with +inf)
      mapW = make_map(Wb, W, H, SP, SROWS);
      mapZ = make_map(Zc.p, W, H, TX, TY);
      if (stage_coarse) mapZstage = make_map(Wb, W, H, TX, TY);
    } else {
      mapW = make_map(Wp.p, pitch, rows, SP, SROWS);
      mapZ = make_map(Zp.p, pitch, rows, TX, TY);
    }
    int per_sm = 0;
    RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
        &per_sm, step_mode == 2 ? (const void *)fill_sweep_kernel<2> : (const void *)fill_sweep_kernel<0>, FILL_THREADS, 0));
    if (per_sm < 1) per_sm = 1;
    grid = c.num_sms * per_sm;
    round = 1;  // stamps start at 0, so round numbers (used as stamp values) start at 1
    // initial worklist: every tile on the perimeter of the tile grid (the only tiles whose
    // cells can see a finite neighbour at the start).  The epsilon fill pins NoData cells anywhere, and a cell whose
    // every neighbour is pinned is lowered by no changed neighbour: every tile's first visit relaxes all of its blocks.
    std::vector<int> init;
    for (int ty = 0; ty < tilesY; ty++)
      for (int tx = 0; tx < tilesX; tx++)
        if (d_coarse || step_mode == 2 || ty == 0 || tx == 0 || ty == tilesY - 1 || tx == tilesX - 1)
          init.push_back(ty * tilesX + tx);
    seed_worklist(init);
  }

  // Geodesic-distance mode: `open` marks the cells the flood may enter (bit `open_bit`), `winit`
  // holds +inf or the seed distance of every cell.  The first round visits the tiles that hold or touch a seed.
  void begin_dist(const uint8_t *d_open, int open_bit, const float *d_winit, int w, int h, int ghost_top = 0,
                  int ghost_bottom = 0) {
    Ctx &c = ctx();
    step_mode = 1;
    W = w;
    H = h;
    tilesX = (w + TX - 1) / TX;
    tilesY = (h + TY - 1) / TY;
    pitch = tilesX * TX + 2 * PADL;
    rows = tilesY * TY + 2;
    use_padded_layout((size_t)pitch * rows);
    const size_t nt = (size_t)tilesX * tilesY;
    list0.alloc(nt);
    list1.alloc(nt);
    plist.alloc(nt);
    stamp.alloc(nt);
    sides.alloc(2 * nt);
    keys.alloc(2 * nt);
    dev.alloc(1);
    RDB_CK(cudaMemsetAsync(stamp.p, 0, nt * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(sides.p, 0, 2 * nt * sizeof(int), c.stream));
    RDB_CK(cudaMemsetAsync(dev.p, 0, sizeof(FillDev), c.stream));
    const int n2 = (int)(2 * nt);
    fill_i32_kernel<<<(n2 + 255) / 256, 256, 0, c.stream>>>(keys.p, ORD_POS_INF, n2);
    dim3 blk(128), grd((pitch + 127) / 128, rows < 2048 ? rows : 2048);
    clear_flags();
    dist_pad_init_kernel<<<grd, blk, 0, c.stream>>>(d_open, open_bit, d_winit, Zp.p, Wp.p, W, H, pitch, rows, ghost_top,
                                                    ghost_bottom, tflag.p, tilesX);
    RDB_CK(cudaGetLastError());
    count_launch(2);
    ordered = false;
    mapW = make_map(Wp.p, pitch, rows, SP, SROWS);
    mapZ = make_map(Zp.p, pitch, rows, TX, TY);
    int per_sm = 0;
    RDB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fill_sweep_kernel<1>, FILL_THREADS, 0));
    if (per_sm < 1) per_sm = 1;
    grid = c.num_sms * per_sm;
    round = 1;
    seed_from_flags();  // the tiles that hold or touch a seed
  }

  // add `tiles` to the worklist of the next round to be launched (always eligible: key = -inf,
  // relax every block).  Tiles already waiting in that list are not duplicated (round stamp).
  void seed_worklist(const std::vector<int> &tiles) {
    Ctx &c = ctx();
    if (tiles.empty()) return;
    DevBuf<int> d(tiles.size());
    RDB_CK(cudaMemcpyAsync(d.p, tiles.data(), tiles.size() * sizeof(int), cudaMemcpyHostToDevice, c.stream));
    FillArgs a = make_args();
    a.round = round;
    fill_seed_kernel<<<(unsigned)((tiles.size() + 255) / 256), 256, 0, c.stream>>>(a, d.p, (int)tiles.size());
    RDB_CK(cudaGetLastError());
    count_launch();
    RDB_CK(cudaStreamSynchronize(c.stream));  // host vector / scratch go out of scope
  }

  FillArgs make_args() {
    Ctx &c = ctx();
    FillArgs a;
    memset(&a, 0, sizeof(a));
    if (inplace) {
      a.Z = Zc.p;
      a.zpitch = W;
      a.inplace = 1;
    } else {
      a.Z = Zp.p;
      a.zpitch = pitch;
      a.zox = PADL;
      a.zoy = 1;
    }
    a.Wc = stage_wc;
    a.pool = stage_k;
    a.yoff = stage_yoff;
    a.staged = staged.p;
    a.Wp = Wb;
    a.pitch = wpitch;
    a.wox = wox;
    a.woy = woy;
    a.W = W;
    a.H = H;
    a.tilesX = tilesX;
    a.tilesY = tilesY;
    a.list0 = list0.p;
    a.list1 = list1.p;
    a.stamp = stamp.p;
    a.sides = sides.p;
    a.keys = keys.p;
    a.plist = plist.p;
    a.dev = dev.p;
    a.max_iters = (int)c.params.fill_max_iters;
    a.use_tma = (int)c.params.fill_use_tma;
    a.profile = (int)c.params.fill_profile;
    a.level = __builtin_inff();
    a.dirty = dirty.p;  // null unless track_dirty() was called
    // (the distance mode wakes every neighbour across a changed side, as the fill does with fill_wake_filter = 0; the
    // epsilon fill takes the fill's test, see fill_sweep_kernel)
    a.edge_above = step_mode != 1 && c.params.fill_wake_filter != 0 ? edge_above.p : nullptr;
    return a;
  }

  // One batch of `per_sync` sweep rounds plus the read-back of the control block, queued on the context's current
  // stream / pinned scratch (two solvers can be driven side by side on two streams: see geodesic_distance_pair_dev).
  bool timed = true;      // false: do not touch the context's timing events (solver driven on a side stream)
  int batch_edge = 0;     // edge_changed bits read back by the last collect()
  void launch_batch(int per_sync) {
    Ctx &c = ctx();
    FillArgs a = make_args();
    if (timed) RDB_CK(cudaEventRecord(c.evk0, c.stream));
    for (int k = 0; k < per_sync; k++) {
      a.round = round;
      // level-ordered admission while the schedule lasts; afterwards every active tile is processed
      if (ordered && sched_round < (int64_t)levels.size()) {
        a.level = levels[(size_t)sched_round];
        a.use_proc = 1;
        fill_admit_kernel<<<c.num_sms * 2, 256, 0, c.stream>>>(a);
        c.stats.kernel_launches++;
      } else {
        a.level = __builtin_inff();
        a.use_proc = 0;
      }
      sched_round++;
      // round 1 of a staged lifted start visits every tile (seeded in begin) and builds W instead of loading it; Z is
      // still the caller's raster then, and every tile saves it to Zc (mapZ) before it writes its W
      a.coarse = round == 1 ? stage_coarse : nullptr;
      a.Z = a.coarse ? Wb : (inplace ? Zc.p : Zp.p);
      a.zcopy = a.coarse ? Zc.p : nullptr;
      const CUtensorMap &mz = a.coarse ? mapZstage : mapZ;
      if (step_mode == 1) fill_sweep_kernel<1><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else if (step_mode == 2 && topo4) fill_sweep_kernel<2, true><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else if (step_mode == 2) fill_sweep_kernel<2><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else if (a.coarse && topo4) fill_sweep_kernel<0, true, true><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else if (a.coarse) fill_sweep_kernel<0, false, true><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else if (topo4) fill_sweep_kernel<0, true><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      else fill_sweep_kernel<0><<<grid, FILL_THREADS, 0, c.stream>>>(mapW, mz, mapZ, a);
      round++;
    }
    if (timed) RDB_CK(cudaEventRecord(c.evk1, c.stream));
    RDB_CK(cudaGetLastError());
    RDB_CK(cudaMemcpyAsync(c.pinned, dev.p, sizeof(FillDev), cudaMemcpyDeviceToHost, c.stream));
    c.stats.kernel_launches += per_sync;
    rounds_run += per_sync;
    if (round > (1 << 30)) fail("fill: round counter overflow");
  }
  // waits for the batch; returns whether tiles are still active
  bool collect() {
    Ctx &c = ctx();
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (timed) {
      float t = 0;
      RDB_CK(cudaEventElapsedTime(&t, c.evk0, c.evk1));
      c.stats.ms_main_kernel += t;  // device time of the sweep launches only (read-back excluded)
    }
    const FillDev *hd = (const FillDev *)c.pinned;
    still_active = hd->ctl[round % 3].count != 0;
    if (!still_active) first_run = false;
    live_rounds = (int64_t)hd->live_rounds;
    visits_seen = (int64_t)hd->visits;
    iters_seen = (int64_t)hd->iters;
    batch_edge = hd->edge_changed;
    return still_active;
  }
  int64_t iters_seen = 0;

  // max_rounds > 0: stop after about that many rounds even if tiles are still active (bit 2 of the
  // result then says so); the caller exchanges halos and calls run again
  int run(int64_t max_rounds = 0) {
    Ctx &c = ctx();
    int64_t rounds_this_call = 0;
    int per_sync = (int)(c.params.fill_rounds_per_sync > 0 ? c.params.fill_rounds_per_sync : 16);
    if (max_rounds > 0 && max_rounds < per_sync) per_sync = (int)max_rounds;  // a short leash (V-cycles) is honoured exactly
    RDB_CK(cudaMemsetAsync(&dev.p->edge_changed, 0, sizeof(int), c.stream));
    for (;;) {
      launch_batch(per_sync);
      collect();
      rounds_this_call += per_sync;
      if (!still_active) break;
      if (max_rounds > 0 && rounds_this_call >= max_rounds) break;
    }
    const FillDev *hd = (const FillDev *)c.pinned;
    c.stats.fill_rounds = live_rounds;
    c.stats.fill_tile_visits = visits_seen;
    c.stats.fill_tile_iters = iters_seen;
    c.stats.fill_tile_cells = TX * TY;
    if (c.params.fill_profile) {
      fprintf(stderr, "[fill profile] deferred=%llu visits=%llu iters=%llu block_updates=%llu (%.1f%% of 256/iter) warp_updates=%llu (%.1f%% of 8/iter) idle_visits=%llu wakes_dropped=%llu hist(1,2,3-4,5-8,9-16,17-32,33-64,65+)=",
              hd->deferred, hd->visits, hd->iters, hd->block_updates, 100.0 * hd->block_updates / (256.0 * hd->iters + 1),
              hd->warp_updates, 100.0 * hd->warp_updates / (8.0 * hd->iters + 1), hd->idle_visits, hd->wakes_dropped);
      for (int k = 0; k < 8; k++) fprintf(stderr, "%llu ", hd->iter_hist[k]);
      fprintf(stderr, "\n");
      // what this run added, so that the lines of all the solvers of a call (coarse levels, V-cycle corrections) sum
      fprintf(stderr, "[fill wake] visits=%llu idle_visits=%llu wakes_dropped=%llu\n", hd->visits - prof_seen[0],
              hd->idle_visits - prof_seen[1], hd->wakes_dropped - prof_seen[2]);
      prof_seen[0] = hd->visits;
      prof_seen[1] = hd->idle_visits;
      prof_seen[2] = hd->wakes_dropped;
    }
    return batch_edge | (still_active ? 4 : 0);
  }
  unsigned long long prof_seen[3] = {0, 0, 0};  // fill_profile: visits, idle visits, dropped wakes reported so far

  // V-cycle plumbing (fill_vcycle): see fill_depressions_level
  void track_dirty() {  // from now on the sweep notes which tiles it wrote
    Ctx &c = ctx();
    const size_t nt = (size_t)tilesX * tilesY;
    dirty.alloc(nt);
    RDB_CK(cudaMemsetAsync(dirty.p, 0, nt * sizeof(int), c.stream));
  }
  void clear_dirty() {
    if (dirty.p) RDB_CK(cudaMemsetAsync(dirty.p, 0, (size_t)tilesX * tilesY * sizeof(int), ctx().stream));
  }
  // queue the tiles flagged in tflag for the next run (no host round trip); d_count (optional) receives how many
  void seed_from_flags(int *d_count = nullptr) {
    Ctx &c = ctx();
    const int nt = tilesX * tilesY;
    FillArgs a = make_args();
    a.round = round;
    fill_seed_flags_kernel<<<(nt + 255) / 256, 256, 0, c.stream>>>(a, tflag.p, nt, d_count);
    RDB_CK(cudaGetLastError());
    count_launch();
  }
  void clear_flags() {
    const size_t nt = (size_t)tilesX * tilesY;
    if (!tflag.p) tflag.alloc(nt);
    RDB_CK(cudaMemsetAsync(tflag.p, 0, nt * sizeof(int), ctx().stream));
  }
  // restriction of THIS (fine) level's surface into the coarse level's solver `cs` (its water levels drop to the
  // k x k block maxima where those are lower; the coarse tiles touched are queued for cs's next run)
  void restrict_into(FillState &cs, int k) {
    Ctx &c = ctx();
    cs.clear_flags();
    const bool selective = dirty.p && TX % k == 0 && TY % k == 0;
    dim3 blk(256), grd((unsigned)((cs.W + 255) / 256), (unsigned)(cs.H < 4096 ? cs.H : 4096));
    fill_restrict_kernel<<<grd, blk, 0, c.stream>>>(Wb, wpitch, wox, woy, W, H, cs.Wb, cs.wpitch, cs.wox, cs.woy, cs.W, cs.H,
                                                    k, selective ? dirty.p : nullptr, tilesX, cs.tflag.p, cs.tilesX);
    RDB_CK(cudaGetLastError());
    count_launch();
    cs.seed_from_flags();
    clear_dirty();
  }
  // selective = true: only blocks in tiles written since the last call are evaluated (the others report +inf = "no news")
  // and the dirty flags are cleared; needs track_dirty()
  void blockmax_into(float *d_out, int wc, int hc, int k, int yoff, int y_lo, int y_hi, bool selective = false) {
    Ctx &c = ctx();
    dim3 blk(256), grd((unsigned)((wc + 255) / 256), (unsigned)((y_hi - y_lo) / k + 2 < 4096 ? (y_hi - y_lo) / k + 2 : 4096));
    const bool sel = selective && dirty.p && TX % k == 0;  // (columns of a block then lie in one tile column)
    fill_blockmax_kernel<<<grd, blk, 0, c.stream>>>(Wb, wpitch, wox, woy, W, y_lo, y_hi, yoff, d_out, wc, hc, k,
                                                    sel ? dirty.p : nullptr, tilesX);
    RDB_CK(cudaGetLastError());
    count_launch();
    if (sel) clear_dirty();
  }
  // prolongation from a coarse surface stored with row pitch `cpitch` and first cell at (coff_x, coff_y); `cdirty`
  // (optional, with its tile-grid width): coarse tiles written by the coarse relaxation -- everything else is skipped.
  // d_count (optional): device counter that receives the number of tiles queued.
  void prolong_from(const float *d_wc, int cpitch, int coff_x, int coff_y, int k, int yoff = 0, const int *cdirty = nullptr,
                    int ctilesX = 0, int *d_count = nullptr) {
    Ctx &c = ctx();
    clear_flags();
    const int nt = tilesX * tilesY;
    fill_prolong_kernel<<<nt, 256, 0, c.stream>>>(Wb, wpitch, wox, woy, W, H, d_wc, cpitch, coff_x, coff_y, k, tflag.p, tilesX,
                                                  yoff, cdirty, ctilesX);
    RDB_CK(cudaGetLastError());
    count_launch();
    seed_from_flags(d_count);
  }
  void prolong_from_level(FillState &cs, int k, int yoff = 0, int *d_count = nullptr) {
    prolong_from(cs.Wb, cs.wpitch, cs.wox, cs.woy, k, yoff, cs.dirty.p, cs.tilesX, d_count);
    cs.clear_dirty();
  }
  // a neighbouring band's edge row arrives: ghost row y (0 or H-1) drops to it where it is lower; the tiles that read
  // the lowered cells are queued, *d_lowered (device int) is set when anything moved
  void ghost_update(int y, const float *d_row, int *d_lowered) {
    Ctx &c = ctx();
    clear_flags();
    fill_ghost_update_kernel<<<(W + 255) / 256, 256, 0, c.stream>>>(Wp.p, Zp.p, pitch, W, H, y, d_row, tflag.p, tilesX, d_lowered);
    RDB_CK(cudaGetLastError());
    count_launch();
    seed_from_flags();
  }

  void read_row(int y, float *d_row) {
    if (y < 0 || y >= H) fail("fill_read_row: row %d out of range", y);
    RDB_CK(cudaMemcpyAsync(d_row, Wb + (size_t)(y + woy) * wpitch + wox, (size_t)W * 4,
                           cudaMemcpyDeviceToDevice, ctx().stream));
  }

  // (row-band states only: they keep the padded layout)
  void update_row(int y, const float *d_row) {
    if (y != 0 && y != H - 1) fail("fill_update_row: only boundary rows (0, height-1) can be replaced");
    Ctx &c = ctx();
    const size_t o = (size_t)(y + 1) * pitch + PADL;
    RDB_CK(cudaMemcpyAsync(Wp.p + o, d_row, (size_t)W * 4, cudaMemcpyDeviceToDevice, c.stream));
    RDB_CK(cudaMemcpyAsync(Zp.p + o, d_row, (size_t)W * 4, cudaMemcpyDeviceToDevice, c.stream));
    pending_rows.push_back(y);
  }
  std::vector<int> pending_rows;

  void activate_pending() {
    if (pending_rows.empty()) return;
    std::vector<char> mark((size_t)tilesX * tilesY, 0);
    std::vector<int> tiles;
    for (int y : pending_rows) {
      // the replaced row sits in tile row y/TY, but it is also the apron of the tile row next to it
      // when it is the first/last row of its tile: wake every tile row that can read it
      for (int yy = y - 1; yy <= y + 1; yy++) {
        if (yy < 0 || yy >= H) continue;
        const int tyT = yy / TY;
        for (int tx = 0; tx < tilesX; tx++) {
          const int t = tyT * tilesX + tx;
          if (!mark[t]) {
            mark[t] = 1;
            tiles.push_back(t);
          }
        }
      }
    }
    pending_rows.clear();
    seed_worklist(tiles);
  }

  void finish(float *d_out) {
    Ctx &c = ctx();
    if (d_out == Wb) return;  // in place: the answer is where it belongs already
    if ((W & 3) == 0 && ((uintptr_t)d_out & 15) == 0) {
      dim3 blk(256), grd((W / 4 + 255) / 256, H < 4096 ? H : 4096);
      fill_finish_x4_kernel<<<grd, blk, 0, c.stream>>>(Wb, d_out, W, H, wpitch, wox, woy);
    } else {
      dim3 blk(256), grd((W + 255) / 256, H < 32768 ? H : 32768);
      fill_finish_kernel<<<grd, blk, 0, c.stream>>>(Wb, d_out, W, H, wpitch, wox, woy);
    }
    RDB_CK(cudaGetLastError());
    count_launch();
  }
};

// Geodesic (8-connected, unit step) distance from the seeds in `d_w_inout` (+inf = not a seed)
// through the cells whose `d_open` byte has `open_bit` set; other cells keep +inf unless seeded.
// Same tile machinery as the fill (the operator only differs by the "+1"); exact for distances
// below 2^24.  Result overwrites d_w_inout.
void geodesic_distance_dev(const uint8_t *d_open, int open_bit, float *d_w_inout, int w, int h) {
  Ctx &c = ctx();
  FillState st;
  const rdb200_stats saved = c.stats;
  st.begin_dist(d_open, open_bit, d_w_inout, w, h);
  st.run();
  st.finish(d_w_inout);
  RDB_CK(cudaStreamSynchronize(c.stream));
  // keep the caller's accounting: only add what this solve cost
  const int64_t launches = c.stats.kernel_launches;
  const int64_t rounds = c.stats.fill_rounds;
  c.stats = saved;
  c.stats.kernel_launches = launches;
  c.stats.flat_bfs_levels += rounds;
}

// Two independent distance solves (the away and the towards gradient of the flat resolution) side by side: each is a
// chain of short dependent rounds with few active tiles, i.e. latency-bound, so their rounds are issued on two streams
// and the SMs run whatever CTAs of either solve have work.  Results overwrite d_wa / d_wb.
void geodesic_distance_pair_dev(const uint8_t *d_open, int open_bit, float *d_wa, float *d_wb, int w, int h) {
  Ctx &c = ctx();
  if (!c.aux_stream[0]) {
    RDB_CK(cudaStreamCreateWithFlags(&c.aux_stream[0], cudaStreamNonBlocking));
    RDB_CK(cudaStreamCreateWithFlags(&c.aux_stream[1], cudaStreamNonBlocking));
    RDB_CK(cudaEventCreateWithFlags(&c.aux_event[0], cudaEventDisableTiming));
    RDB_CK(cudaEventCreateWithFlags(&c.aux_event[1], cudaEventDisableTiming));
    RDB_CK(cudaEventCreateWithFlags(&c.aux_event[2], cudaEventDisableTiming));
  }
  const rdb200_stats saved = c.stats;
  cudaStream_t main_stream = c.stream;
  void *main_pinned = c.pinned;
  // the side streams start after everything queued on the main stream so far
  RDB_CK(cudaEventRecord(c.aux_event[2], main_stream));
  FillState st[2];
  float *wbuf[2] = {d_wa, d_wb};
  auto lane = [&](int k, auto &&fn) {  // run fn with lane k's stream and its own slot of the pinned scratch
    c.stream = c.aux_stream[k];
    c.pinned = (char *)main_pinned + 8192 * (k + 1);
    try {
      fn(st[k]);
    } catch (...) {
      c.stream = main_stream;
      c.pinned = main_pinned;
      throw;
    }
    c.stream = main_stream;
    c.pinned = main_pinned;
  };
  static_assert(sizeof(FillDev) <= 8192, "pinned slot");
  try {
    for (int k = 0; k < 2; k++) {
      RDB_CK(cudaStreamWaitEvent(c.aux_stream[k], c.aux_event[2], 0));
      lane(k, [&](FillState &s) {
        s.timed = false;
        s.begin_dist(d_open, open_bit, wbuf[k], w, h);
        // a sweep launch fills every CTA slot of the GPU; two of them only run side by side when each takes half
        s.grid = s.grid > 1 ? s.grid / 2 : 1;
      });
    }
    const int per_sync = (int)(c.params.fill_rounds_per_sync > 0 ? c.params.fill_rounds_per_sync : 16);
    bool live[2] = {true, true};
    while (live[0] || live[1]) {
      for (int k = 0; k < 2; k++)
        if (live[k]) lane(k, [&](FillState &s) { s.launch_batch(per_sync); });
      for (int k = 0; k < 2; k++)
        if (live[k]) lane(k, [&](FillState &s) { live[k] = s.collect(); });
    }
    for (int k = 0; k < 2; k++) {
      lane(k, [&](FillState &s) { s.finish(wbuf[k]); });
      RDB_CK(cudaEventRecord(c.aux_event[k], c.aux_stream[k]));
      RDB_CK(cudaStreamWaitEvent(main_stream, c.aux_event[k], 0));
    }
  } catch (...) {
    cudaStreamSynchronize(c.aux_stream[0]);
    cudaStreamSynchronize(c.aux_stream[1]);
    throw;
  }
  RDB_CK(cudaStreamSynchronize(c.aux_stream[0]));  // the solvers' buffers are released when `st` goes out of scope
  RDB_CK(cudaStreamSynchronize(c.aux_stream[1]));
  const int64_t launches = c.stats.kernel_launches;
  c.stats = saved;
  c.stats.kernel_launches = launches;
  c.stats.flat_bfs_levels += st[0].live_rounds + st[1].live_rounds;
}

// fill_multigrid = k (off by default; prepared for round 2): the flood does not have to start from +inf.  ANY
// surface W0 >= W* with W0 = Z on the border relaxes to exactly W* (DESIGN.md 3.1), and a good one is cheap: max-pool
// the raster over k x k blocks, fill THAT (recursively), and give every cell its block's coarse water level.  It is an
// upper bound because the cells of a block are connected below the block's maximum and 8-adjacent blocks contain
// 8-adjacent cells, so every coarse path lifts to a fine path that is nowhere higher; border blocks contain a border
// cell.  On the CPU model of the schedule this cuts the dependent rounds 3.5x and the tile visits by 20-40 %.
static void fill_depressions_level(float *d_dem, int w, int h, int depth, bool topo4 = false) {
  Ctx &c = ctx();
  const int k = (int)c.params.fill_multigrid;
  const int min_side = (int)(c.params.fill_multigrid_min > 0 ? c.params.fill_multigrid_min : 1024);
  FillState st;
  st.topo4 = topo4;
  if (k >= 2 && depth < 8 && w >= min_side && h >= min_side && w / k >= 3 && h / k >= 3) {
    const int wc = (w + k - 1) / k, hc = (h + k - 1) / k;
    DevBuf<float> coarse((size_t)wc * hc);
    dim3 blk(256), grd((unsigned)((wc + 255) / 256), (unsigned)(hc < 4096 ? hc : 4096));
    fill_maxpool_kernel<<<grd, blk, 0, c.stream>>>(d_dem, w, h, 0, coarse.p, wc, hc, k, 0);
    RDB_CK(cudaGetLastError());
    count_launch();
    const int every = (int)c.params.fill_vcycle;  // > 0: coarse-grid correction after that many fine rounds
    DevBuf<float> zc;
    if (every > 0) {  // the coarse elevations are needed again for the corrections
      zc.alloc((size_t)wc * hc);
      RDB_CK(cudaMemcpyAsync(zc.p, coarse.p, (size_t)wc * hc * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
    }
    const rdb200_stats before = c.stats;
    fill_depressions_level(coarse.p, wc, hc, depth + 1, topo4);
    rdb200_stats extra = c.stats;  // work done on the coarse levels, accounted on top of this level's
    extra.fill_rounds -= before.fill_rounds;
    extra.fill_tile_visits -= before.fill_tile_visits;
    extra.fill_tile_iters -= before.fill_tile_iters;
    // (both solvers run in place where they can: st relaxes W in d_dem, cst in zc, which nothing else reads; `coarse`
    // stays as it is until both are done: their first rounds build their start from it)
    st.begin(d_dem, w, h, coarse.p, wc, k, 0, true);
    if (every <= 0) {
      st.run();
    } else {
      // V-cycles.  The lifted start leaves every lake a little too high (max-pooling raises its pass), and lowering a
      // lake is a sweep across it, one tile per round.  So after `every` fine rounds the coarse surface is lowered to
      // the block maxima of the fine one (restriction), relaxed again -- the same sweep, k times fewer tiles across --
      // and handed back (prolongation: fine = min(fine, lifted)).  Restriction and coarse relaxation keep every coarse
      // value an upper bound of the answer for all cells of its block, so the fine surface stays an upper bound and
      // still relaxes to exactly W*.
      // The coarse level keeps ONE solver for all corrections (cst): restriction lowers its surface in place
      // and queues the coarse tiles it touched, its relaxation notes the tiles it writes, and the prolongation only
      // looks at the fine tiles below those -- a correction costs what it changes, not three passes over the raster.
      FillState cst;
      cst.topo4 = topo4;
      cst.begin(zc.p, wc, hc, coarse.p, wc, 1, 0, true);  // start: the coarse fill itself (already a fixed point)
      cst.run();                                  // (drains the initial all-tiles worklist; nothing moves)
      cst.track_dirty();
      st.track_dirty();
      int64_t coarse_visits0 = c.stats.fill_tile_visits, coarse_iters0 = c.stats.fill_tile_iters;
      const bool trace = c.params.fill_trace != 0;  // per-cycle timeline on stderr (adds stream syncs)
      auto now_ms = [&]() {
        RDB_CK(cudaStreamSynchronize(c.stream));
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
      };
      for (int cycle = 0;; cycle++) {
        const double t0 = trace ? now_ms() : 0;
        const int64_t v0 = st.visits_seen, r0 = st.live_rounds;
        const bool active = (st.run(every) & 4) != 0;
        const double t1 = trace ? now_ms() : 0;
        if (trace)
          fprintf(stderr, "[fill trace] depth %d cycle %d: fine run %.3f ms (%lld live rounds, %lld visits)%s\n", depth, cycle,
                  t1 - t0, (long long)(st.live_rounds - r0), (long long)(st.visits_seen - v0), active ? "" : " -> converged");
        if (!active) break;
        if (cycle >= 1000) {  // safety net: plain relaxation to the end
          st.run();
          break;
        }
        st.restrict_into(cst, k);
        const double t2 = trace ? now_ms() : 0;
        const int64_t cv0 = cst.visits_seen, cr0 = cst.live_rounds;
        cst.run();
        const double t3 = trace ? now_ms() : 0;
        st.prolong_from_level(cst, k);
        if (trace) {
          const double t4 = now_ms();
          fprintf(stderr, "[fill trace] depth %d cycle %d: restrict %.3f ms, coarse run %.3f ms (%lld live rounds, %lld visits), "
                          "prolong %.3f ms\n", depth, cycle, t2 - t1, t3 - t2, (long long)(cst.live_rounds - cr0),
                  (long long)(cst.visits_seen - cv0), t4 - t3);
        }
      }
      cst.run(1);  // refresh the coarse solver's counters in c.stats (FillState::run reports absolute values)
      extra.fill_rounds += cst.live_rounds;
      extra.fill_tile_visits += c.stats.fill_tile_visits;
      extra.fill_tile_iters += c.stats.fill_tile_iters;
      (void)coarse_visits0;
      (void)coarse_iters0;
      st.run(1);  // and the fine solver's (no tile is active: an empty launch)
    }
    st.finish(d_dem);
    RDB_CK(cudaStreamSynchronize(c.stream));
    c.stats.fill_rounds = st.live_rounds + extra.fill_rounds;
    c.stats.fill_tile_visits += extra.fill_tile_visits;
    c.stats.fill_tile_iters += extra.fill_tile_iters;
    return;
  }
  if (w <= 2 || h <= 2) return;  // every cell is a border cell: nothing can change
  st.begin(d_dem, w, h, nullptr, 0, 0, 0, true);
  st.run();
  st.finish(d_dem);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

// fill with a given start: `d_w` holds an upper bound of the answer (e.g. a restricted coarse surface) and receives it
void fill_relax_from_dev(const float *d_dem, float *d_w, int w, int h) {
  Ctx &c = ctx();
  c.stats.cells = (int64_t)w * h;
  if (w <= 2 || h <= 2) {
    RDB_CK(cudaMemcpyAsync(d_w, d_dem, (size_t)w * h * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    return;
  }
  FillState st;
  st.begin(d_dem, w, h, d_w, w, 1);
  st.run();
  st.finish(d_w);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

void fill_maxpool_rows(const float *d_src, int w, int h, int yoff, float *d_coarse, int wc, int hc, int k, dim3 grd, dim3 blk) {
  fill_maxpool_kernel<<<grd, blk, 0, ctx().stream>>>(d_src, w, h, yoff, d_coarse, wc, hc, k, 1);
  RDB_CK(cudaGetLastError());
  count_launch();
}

// =================================================================================================
// Row-band (multi-GPU) fill, driven from C++ over a rdb200_comm (NCCL, or the caller's callbacks in the CPU tests).
// Every rank holds ghost_top + owned + ghost_bottom rows of the raster in `d_local` (in / out; the ghost rows leave
// holding the neighbours' filled edge rows).  The multigrid start is what makes the bands nearly independent:
//   1. every rank max-pools its owned rows; a MAX all-reduce gives every rank the whole k x k pooled raster (1/k^2 of the
//      cells), which every rank fills itself (redundant but small) -- the coarse surface, lifted, is an upper bound of
//      the answer for every band and its ghost rows;
//   2. cycles of: R sweep rounds on the band | edge rows to the neighbours (a ghost row only ever drops) | V-cycle
//      correction: block maxima of the bands (MAX all-reduce) lower the coarse surface, the coarse relaxation runs on every
//      rank, the band takes the lowered blocks back | one 4-int MAX all-reduce decides whether anything moved anywhere.
// The fixed point is the single-GPU one (any admissible schedule ends at W*, DESIGN.md 3.1): when no tile is active, no
// ghost row dropped and no correction lowered a cell on any rank, every band is at its local fixed point with ghost rows
// equal to the neighbours' edge rows.
// topo4: FillDepressions<D4>.  Every solver the driver creates -- the band's, the replicated coarse fill's and the V-cycle
// coarse solver's -- takes the 4-neighbour stencil: the lifted start is an upper bound of the D4 answer only if the coarse
// surface is the D4 fill too (blocks that touch at a corner hold no D4-adjacent cells, so a D8 coarse fill would drain a
// block through that corner and start the band below the answer, which relaxation cannot repair).  The rest does not
// depend on the stencil: a ghost row takes the neighbour's edge row where it is lower (min; the tiles it wakes are the
// D8 readers, a superset of the D4 ones), a lifted ghost row is its blocks' coarse levels, block maxima and
// prolongation (min(fine, lifted)) are cell-wise over k x k blocks, and the termination vote counts events, not cells.
void mgpu_fill_band(const rdb200_comm *comm, float *d_local, int w, int hloc, int gt, int gb, int row0, int H, int *xrounds,
                    bool topo4) {
  Ctx &c = ctx();
  const int world = comm_world(comm);
  gt = gt ? 1 : 0;
  gb = gb ? 1 : 0;
  if (w < 3 || hloc - gt - gb < 1 || hloc < 3) fail("mgpu_fill: band too small (%d x %d)", w, hloc);
  if (row0 < 0 || row0 + hloc > H) fail("mgpu_fill: rows [%d, %d) are outside the raster (%d rows)", row0, row0 + hloc, H);
  // pooling factor of the band's coarse level: every rank fills and re-relaxes that raster itself, a cost that does not
  // shrink with the number of GPUs, so with many bands a coarser one pays (fill_band_multigrid; 0: fill_multigrid for
  // up to two bands, twice that beyond)
  int k = (int)c.params.fill_band_multigrid;
  if (k <= 0) {
    k = (int)c.params.fill_multigrid;
    if (k >= 2 && world > 2 && TX % (2 * k) == 0) k *= 2;
  }
  const int min_side = (int)(c.params.fill_multigrid_min > 0 ? c.params.fill_multigrid_min : 1024);
  const bool mg = k >= 2 && w >= min_side && H >= min_side && w / k >= 3 && H / k >= 3 && c.params.fill_multigrid >= 2;
  const int R = (int)(c.params.fill_vcycle > 0 ? c.params.fill_vcycle : 8);
  const float inf = __builtin_inff();
  DevBuf<float> rows(4 * (size_t)w);  // send up, send down, receive up, receive down
  DevBuf<int> flags(4);               // tiles active | a ghost row dropped | coarse surface lowered | band cells lowered
  float *send_up = rows.p, *send_dn = rows.p + w, *recv_up = rows.p + 2 * (size_t)w, *recv_dn = rows.p + 3 * (size_t)w;
  FillState st, cst;
  DevBuf<float> zc, wcoarse, bm;
  int wc = 0, hc = 0;
  auto fill_f32 = [&](float *p, size_t n, float v) {
    int bits;
    memcpy(&bits, &v, 4);
    fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(reinterpret_cast<int *>(p), bits, (int)n);
    RDB_CK(cudaGetLastError());
  };
  const bool trace0 = c.params.fill_trace != 0;
  double t0_prev = 0;
  auto lap0 = [&](const char *what) {
    if (!trace0) return;
    RDB_CK(cudaStreamSynchronize(c.stream));
    const double t = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    if (what) fprintf(stderr, "[mgpu fill trace] rank %d begin: %-32s %8.3f ms\n", comm_rank(comm), what, t - t0_prev);
    t0_prev = t;
  };
  lap0(nullptr);
  if (mg) {
    wc = (w + k - 1) / k;
    hc = (H + k - 1) / k;
    const size_t nc = (size_t)wc * hc;
    zc.alloc(nc);
    wcoarse.alloc(nc);
    bm.alloc(nc);
    fill_f32(zc.p, nc, -inf);
    {
      const int hown = hloc - gt - gb;
      dim3 blk(256), grd((unsigned)((wc + 255) / 256), (unsigned)(hown / k + 2 < 4096 ? hown / k + 2 : 4096));
      fill_maxpool_rows(d_local + (size_t)gt * w, w, hown, row0 + gt, zc.p, wc, hc, k, grd, blk);
    }
    lap0("max-pool own rows");
    comm_allreduce(comm, zc.p, nc, RDB200_MAX_F32);
    lap0("all-reduce pooled raster");
    RDB_CK(cudaMemcpyAsync(wcoarse.p, zc.p, nc * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
    fill_depressions_level(wcoarse.p, wc, hc, 1, topo4);  // every rank fills the small raster itself
    lap0("coarse fill (replicated)");
    for (int side = 0; side < 2; side++) {
      if (!(side == 0 ? gt : gb)) continue;
      const int y = side == 0 ? 0 : hloc - 1;
      fill_lift_row_kernel<<<(w + 255) / 256, 256, 0, c.stream>>>(d_local + (size_t)y * w, w, wcoarse.p + (size_t)((row0 + y) / k) * wc, k);
    }
    RDB_CK(cudaGetLastError());
    st.topo4 = topo4;
    st.begin(d_local, w, hloc, wcoarse.p, wc, k, row0);
    lap0("band start (lifted)");
    cst.topo4 = topo4;
    cst.begin(zc.p, wc, hc, wcoarse.p, wc, 1);
    cst.run();
    cst.track_dirty();
    st.track_dirty();
    lap0("coarse solver setup");
  } else {
    if (gt) fill_f32(d_local, (size_t)w, inf);
    if (gb) fill_f32(d_local + (size_t)(hloc - 1) * w, (size_t)w, inf);
    st.topo4 = topo4;
    st.begin(d_local, w, hloc);
  }
  int cycles = 0;
  bool vcycle_on = true;
  int *hflags = (int *)c.pinned + 1024;  // (FillState::run reads its control block back into the front of the scratch)
  const bool trace = c.params.fill_trace != 0;  // per-phase timeline on stderr (adds stream syncs)
  double t_prev = 0;
  auto lap = [&](const char *what) {
    if (!trace) return;
    RDB_CK(cudaStreamSynchronize(c.stream));
    const double t = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    if (what) fprintf(stderr, "[mgpu fill trace] rank %d cycle %d: %-28s %8.3f ms\n", comm_rank(comm), cycles, what, t - t_prev);
    t_prev = t;
  };
  lap(nullptr);
  for (;; cycles++) {
    if (cycles > 100000) fail("mgpu_fill: no convergence");
    const bool active = (st.run(world > 1 || mg ? R : 0) & 4) != 0;
    lap("band sweeps");
    RDB_CK(cudaMemsetAsync(flags.p, 0, 4 * sizeof(int), c.stream));
    if (world > 1) {
      if (gt) st.read_row(1, send_up);
      if (gb) st.read_row(hloc - 2, send_dn);
      comm_exchange(comm, send_up, recv_up, send_dn, recv_dn, (size_t)w * sizeof(float));
      if (gt) st.ghost_update(0, recv_up, flags.p + 1);
      if (gb) st.ghost_update(hloc - 1, recv_dn, flags.p + 1);
      lap("halo exchange");
    }
    // the coarse-grid correction is dropped for good once a cycle's correction moved next to nothing on any rank: what is left
    // are local repairs next to the seams, and the correction's fixed cost (the all-reduce of the pooled raster and the
    // coarse relaxation on every rank) would be paid for nothing
    if (mg && vcycle_on) {
      fill_f32(bm.p, (size_t)wc * hc, -inf);
      st.blockmax_into(bm.p, wc, hc, k, row0, gt, hloc - gb, true);
      lap("block maxima");
      comm_allreduce(comm, bm.p, (size_t)wc * hc, RDB200_MAX_F32);
      lap("all-reduce coarse");
      cst.prolong_from(bm.p, wc, 0, 0, 1, 0, nullptr, 0, flags.p + 2);  // the coarse surface drops to the block maxima
      cst.run();
      lap("coarse relaxation");
      st.prolong_from_level(cst, k, row0, flags.p + 3);
      lap("prolongation");
    }
    if (active) fill_i32_kernel<<<1, 1, 0, c.stream>>>(flags.p, 1, 1);
    comm_allreduce(comm, flags.p, 4, RDB200_MAX_I32);
    RDB_CK(cudaMemcpyAsync(hflags, flags.p, 4 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    lap("termination vote");
    if (!(hflags[0] | hflags[1] | hflags[2] | hflags[3])) break;
    // (tiles flagged by the correction on the busiest rank; a band has tilesX * tilesY of them)
    const int few = st.tilesX * st.tilesY / 64 > 32 ? st.tilesX * st.tilesY / 64 : 32;
    if (trace) fprintf(stderr, "[mgpu fill trace] rank %d cycle %d: flags active=%d ghost=%d coarse=%d fine=%d (cut-off %d)\n",
                       comm_rank(comm), cycles, hflags[0], hflags[1], hflags[2], hflags[3], few);
    if (hflags[2] + hflags[3] < few) vcycle_on = false;
  }
  st.run(1);  // refresh the counters (no tile is active: an empty launch)
  const int64_t visits = st.visits_seen, iters = st.iters_seen, rounds = st.live_rounds;
  st.finish(d_local);
  RDB_CK(cudaStreamSynchronize(c.stream));
  lap("finish");
  c.stats.fill_rounds = rounds + (mg ? cst.live_rounds : 0);
  c.stats.fill_tile_visits = visits;
  c.stats.fill_tile_iters = iters;
  c.stats.fill_tile_cells = TX * TY;
  if (xrounds) *xrounds = cycles + 1;
}

void fill_depressions_dev(float *d_dem, int w, int h, bool topo4) {
  Ctx &c = ctx();
  c.stats.cells = (int64_t)w * h;
  if (w <= 2 || h <= 2) return;  // every cell is a border cell: nothing can change
  fill_depressions_level(d_dem, w, h, 0, topo4);
}

// FillDepressions(epsilon=True): the greatest fixed point of W(c) = max(Z(c), min over the neighbours n of
// next_up(W(n))), with W = Z on the raster border and on the cells equal to `nodata` (DESIGN.md section 0, f3).  The
// engine relaxes it in place from +inf (fill_sweep_kernel<2>).  The multigrid start of fill_depressions_level is not
// taken: its coarse surface is an upper bound of the plain fill, which lies below this answer.
void fill_depressions_epsilon_dev(float *d_dem, int w, int h, bool topo4, float nodata) {
  Ctx &c = ctx();
  c.stats.cells = (int64_t)w * h;
  if (w <= 2 || h <= 2) return;  // every cell is a border cell: nothing can change
  FillState st;
  st.step_mode = 2;
  st.topo4 = topo4;
  st.pin = nodata;
  st.begin(d_dem, w, h, nullptr, 0, 0, 0, true);
  st.run();
  st.finish(d_dem);
  RDB_CK(cudaStreamSynchronize(c.stream));
}

}  // namespace rdb

// ---- C ABI: row-band protocol ------------------------------------------------------------
struct rdb200_fill_state {
  rdb::FillState st;
};

namespace rdb {
// row-band geodesic distance: same protocol object as the band fill (run / read_row / update_row / finish)
rdb200_fill_state *new_band_distance_state(const uint8_t *d_open, int open_bit, const float *d_winit, int w, int h,
                                           int ghost_top, int ghost_bottom) {
  auto *s = new rdb200_fill_state();
  try {
    s->st.begin_dist(d_open, open_bit, d_winit, w, h, ghost_top, ghost_bottom);
  } catch (...) {
    delete s;
    throw;
  }
  return s;
}
void finish_band_distance_state(rdb200_fill_state *s, float *d_out) {
  s->st.finish(d_out);
  RDB_CK(cudaStreamSynchronize(ctx().stream));
  delete s;
}

// The band relaxation of mgpu_fill_band without its multigrid start and coarse corrections, for a state that already
// holds its start (the flat-resolution gradients' distance states): cycles of R sweep rounds (0: to the band's local
// fixed point) | edge rows to the neighbours, ghost rows drop to them where lower | one 2-int MAX all-reduce of {tiles
// still active, a ghost row dropped}.  Every value is a decreasing upper bound, so when neither happened on any rank
// the bands hold the single-GPU fixed point.  Returns the number of cycles.
int mgpu_relax_band(const rdb200_comm *comm, rdb200_fill_state *state, int gt, int gb, int R) {
  Ctx &c = ctx();
  FillState &st = state->st;
  const int world = comm_world(comm), w = st.W, h = st.H;
  DevBuf<float> rows(4 * (size_t)w);  // send up, send down, receive up, receive down
  DevBuf<int> flags(2);               // tiles active | a ghost row dropped
  float *send_up = rows.p, *send_dn = rows.p + w, *recv_up = rows.p + 2 * (size_t)w, *recv_dn = rows.p + 3 * (size_t)w;
  int *hflags = (int *)c.pinned + 1024;  // (FillState::run reads its control block back into the front of the scratch)
  for (int cycles = 1;; cycles++) {
    if (cycles > 100000) fail("mgpu_relax_band: no convergence");
    const bool active = (st.run(world > 1 ? R : 0) & 4) != 0;
    if (world == 1) {
      if (active) continue;
      RDB_CK(cudaStreamSynchronize(c.stream));
      return cycles;
    }
    RDB_CK(cudaMemsetAsync(flags.p, 0, 2 * sizeof(int), c.stream));
    if (gt) st.read_row(1, send_up);
    if (gb) st.read_row(h - 2, send_dn);
    comm_exchange(comm, send_up, recv_up, send_dn, recv_dn, (size_t)w * sizeof(float));
    if (gt) st.ghost_update(0, recv_up, flags.p + 1);
    if (gb) st.ghost_update(h - 1, recv_dn, flags.p + 1);
    if (active) fill_i32_kernel<<<1, 1, 0, c.stream>>>(flags.p, 1, 1);
    comm_allreduce(comm, flags.p, 2, RDB200_MAX_I32);
    RDB_CK(cudaMemcpyAsync(hflags, flags.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (!(hflags[0] | hflags[1])) return cycles;
  }
}
}  // namespace rdb

extern "C" {

int rdb200_dev_fill_begin(rdb200_fill_state **state, const float *d_dem, int32_t width, int32_t height) {
  return rdb::capi_call([&] {
    rdb::ensure_init();
    if (!state) rdb::fail("fill_begin: null state pointer");
    if (width < 3 || height < 3) rdb::fail("fill_begin: band must be at least 3x3");
    auto s = std::make_unique<rdb200_fill_state>();
    s->st.begin(d_dem, width, height);
    *state = s.release();
  });
}

int rdb200_dev_fill_begin_lifted(rdb200_fill_state **state, const float *d_dem, int32_t width, int32_t height,
                                 const float *d_coarse, int32_t coarse_width, int32_t pool, int32_t row_offset) {
  return rdb::capi_call([&] {
    rdb::ensure_init();
    if (!state) rdb::fail("fill_begin_lifted: null state pointer");
    if (width < 3 || height < 3) rdb::fail("fill_begin_lifted: band must be at least 3x3");
    if (!d_coarse || pool < 2 || coarse_width < (width + pool - 1) / pool || row_offset < 0)
      rdb::fail("fill_begin_lifted: bad coarse raster (pool %d, coarse_width %d, row_offset %d)", pool, coarse_width, row_offset);
    auto s = std::make_unique<rdb200_fill_state>();
    s->st.begin(d_dem, width, height, d_coarse, coarse_width, pool, row_offset);
    *state = s.release();
  });
}

int rdb200_dev_maxpool_rows_f32(const float *d_src, int32_t width, int32_t height, int32_t row_offset, int32_t pool,
                                float *d_coarse, int32_t coarse_width, int32_t coarse_height) {
  return rdb::capi_call([&] {
    rdb::ensure_init();
    if (width < 1 || height < 1 || pool < 2 || row_offset < 0 || coarse_width < (width + pool - 1) / pool ||
        coarse_height < (row_offset + height + pool - 1) / pool)
      rdb::fail("maxpool_rows: bad geometry");
    rdb::Ctx &c = rdb::ctx();
    dim3 blk(256), grd((unsigned)((coarse_width + 255) / 256), (unsigned)(height / pool + 2 < 4096 ? height / pool + 2 : 4096));
    rdb::fill_maxpool_rows(d_src, width, height, row_offset, d_coarse, coarse_width, coarse_height, pool, grd, blk);
    RDB_CK(cudaStreamSynchronize(c.stream));
  });
}

int rdb200_dev_fill_relax_from_f32(const float *d_dem, float *d_w_inout, int32_t width, int32_t height) {
  return rdb::capi_call([&] {
    rdb::ensure_init();
    if (width < 1 || height < 1) rdb::fail("fill_relax_from: raster dimensions must be positive");
    rdb::fill_relax_from_dev(d_dem, d_w_inout, width, height);
  });
}

int rdb200_dev_fill_blockmax(rdb200_fill_state *state, float *d_blockmax, int32_t coarse_width, int32_t coarse_height, int32_t pool,
                             int32_t row_offset, int32_t skip_top, int32_t skip_bottom) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_blockmax: null state");
    rdb::FillState &st = state->st;
    if (pool < 2 || row_offset < 0 || skip_top < 0 || skip_bottom < 0 || skip_top + skip_bottom >= st.H ||
        coarse_width < (st.W + pool - 1) / pool || coarse_height < (row_offset + st.H - skip_bottom + pool - 1) / pool)
      rdb::fail("fill_blockmax: bad geometry");
    st.blockmax_into(d_blockmax, coarse_width, coarse_height, pool, row_offset, skip_top, st.H - skip_bottom);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_fill_prolong(rdb200_fill_state *state, const float *d_coarse, int32_t coarse_width, int32_t pool, int32_t row_offset,
                            int32_t *tiles_lowered) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_prolong: null state");
    if (!d_coarse || pool < 2 || row_offset < 0) rdb::fail("fill_prolong: bad arguments");
    rdb::Ctx &c = rdb::ctx();
    rdb::DevBuf<int> cnt(1);
    RDB_CK(cudaMemsetAsync(cnt.p, 0, sizeof(int), c.stream));
    state->st.prolong_from(d_coarse, coarse_width, 0, 0, pool, row_offset, nullptr, 0, cnt.p);
    int *h = (int *)c.pinned;
    RDB_CK(cudaMemcpyAsync(h, cnt.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    RDB_CK(cudaStreamSynchronize(c.stream));
    if (tiles_lowered) *tiles_lowered = *h;
  });
}

int rdb200_dev_fill_run(rdb200_fill_state *state, int32_t *changed_rows) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_run: null state");
    state->st.activate_pending();
    const int ch = state->st.run(rdb::ctx().params.fill_band_rounds);
    if (changed_rows) *changed_rows = ch;
  });
}

int rdb200_dev_fill_read_row(rdb200_fill_state *state, int32_t y, float *d_row) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_read_row: null state");
    state->st.read_row(y, d_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_fill_update_row(rdb200_fill_state *state, int32_t y, const float *d_row) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_update_row: null state");
    state->st.update_row(y, d_row);
    RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
  });
}

int rdb200_dev_fill_finish(rdb200_fill_state *state, float *d_out) {
  return rdb::capi_call([&] {
    if (!state) rdb::fail("fill_finish: null state");
    if (d_out) {
      state->st.finish(d_out);
      RDB_CK(cudaStreamSynchronize(rdb::ctx().stream));
    }
    delete state;
  });
}

}  // extern "C"
