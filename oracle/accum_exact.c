/* TEST INFRASTRUCTURE ONLY -- flow accumulation from given proportions in extended precision, with a per-cell error
 * budget for the library's engines (oracle/accum_exact.py is the front end).
 *
 *     A(c) = w(c) + sum over donors d -> c of p(d, c) * A(d)
 *
 * over the proportions the library itself returns (FlowProportions), in topological order, in `long double` (64-bit
 * significand on x86-64).  The graph is the one every engine walks: interior cells only donate, a share p <= 0 is no
 * flow, flow into a NoData cell (slot 0 == -2) is dropped and NoData cells end as -1.
 *
 * Budgets (|engine - A| <= B, cell by cell):
 *   mode 0 -- double engines (any summation order, atomics included): a cell's value is the double sum of its weight and
 *     k double products p * a(d), each of those rounded once, then k additions in some order.  With u = 2^-53 and
 *     eta = 2^-1074 (the absolute error of a rounding into the subnormal range):
 *         B(c) = sum p B(d) + (k + 1) u s (|w(c)| + sum p (|A(d)| + B(d))) + (k + 1) eta,   s = 1.01
 *   mode 1 -- the packed fixed-point D-infinity walk (unit weights, 24 fractional bits): a donor with two positive shares
 *     sends each rounded to the nearest 2^-24 (error <= 2^-25, plus the double rounding of the product p * a(d)); a sole
 *     share is sent exactly; the final conversion to double rounds once:
 *         B(c) = sum p B(d) + sum over rounded shares (2^-25 + 2 u p |A(d)|) + u |A(c)|
 * Mode 1 also replays the packed walk itself: integer sums do not depend on their order, so its result is a function of
 * the proportions alone and the replay gives its bits (`packed`, `packed_fma` with the product and the half rounded once,
 * as a fused multiply-add does).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const int dx[9] = {0, -1, -1, 0, 1, 1, 1, 0, -1};
static const int dy[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};

#define NO_DATA_GEN (-2.0f)

static uint64_t share_fx(float p, uint64_t acc, int fused) {
  const double ad = (double)acc;
  return (uint64_t)(fused ? fma((double)p, ad, 0.5) : (double)p * ad + 0.5);
}

/* Returns the number of data cells that were never completed (0 for any acyclic graph), or -1 on allocation failure.
 * weights: NULL means unit weights.  got: NULL, or an engine's result; then err = |got - A| (long double, rounded up to
 * double only at the end).  rounded: shares rounded into each cell (mode 1) / shares received (mode 0). */
int ae_accumulate(const float *props, const double *weights, int w, int h, int mode, const double *got, double *ref,
                  double *budget, double *err, double *packed, double *packed_fma, int32_t *shares) {
  const size_t n = (size_t)w * h;
  long double *A = calloc(n, sizeof(long double)), *B = calloc(n, sizeof(long double));
  long double *Sabs = calloc(n, sizeof(long double)), *R = calloc(n, sizeof(long double));
  uint64_t *fx = mode == 1 ? calloc(2 * n, sizeof(uint64_t)) : NULL;
  int32_t *deps = calloc(n, sizeof(int32_t)), *k = calloc(n, sizeof(int32_t));
  int *queue = malloc(n * sizeof(int));
  if (!A || !B || !Sabs || !R || (mode == 1 && !fx) || !deps || !k || !queue) return -1;
  const long double u = ldexpl(1.0L, -53), eta = ldexpl(1.0L, -1074), half_unit = ldexpl(1.0L, -25);
  for (size_t i = 0; i < n; i++) {
    A[i] = weights ? (long double)weights[i] : 1.0L;
    if (fx) fx[i] = fx[n + i] = (uint64_t)1 << 24;
  }
  for (int y = 1; y < h - 1; y++)
    for (int x = 1; x < w - 1; x++) {
      const size_t c = (size_t)y * w + x;
      if (props[9 * c] == NO_DATA_GEN) continue;
      for (int m = 1; m <= 8; m++)
        if (props[9 * c + m] > 0) deps[c + (ptrdiff_t)dy[m] * w + dx[m]]++;
    }
  size_t qh = 0, qt = 0, data = 0;
  for (size_t i = 0; i < n; i++)
    if (props[9 * i] != NO_DATA_GEN) {
      data++;
      if (deps[i] == 0) queue[qt++] = (int)i;
    }
  while (qh < qt) {
    const size_t c = (size_t)queue[qh++];
    /* the cell is complete: close its budget */
    const long double wc = weights ? fabsl((long double)weights[c]) : 1.0L;
    if (mode == 0)
      B[c] += (long double)(k[c] + 1) * u * 1.01L * (wc + Sabs[c]) + (long double)(k[c] + 1) * eta;
    else
      B[c] += R[c] + u * fabsl(A[c]);
    const int y = (int)(c / w), x = (int)(c - (size_t)y * w);
    if (x == 0 || y == 0 || x == w - 1 || y == h - 1) continue;
    int npos = 0;
    for (int m = 1; m <= 8; m++) npos += props[9 * c + m] > 0;
    for (int m = 1; m <= 8; m++) {
      const float p = props[9 * c + m];
      if (!(p > 0)) continue;
      const size_t r = c + (ptrdiff_t)dy[m] * w + dx[m];
      if (props[9 * r] == NO_DATA_GEN) continue;
      {
        const long double pl = (long double)p;
        A[r] += pl * A[c];
        B[r] += pl * B[c];
        Sabs[r] += pl * (fabsl(A[c]) + B[c]);
        k[r]++;
        if (fx) {
          if (npos > 1) {
            R[r] += half_unit + 2 * u * pl * (fabsl(A[c]) + B[c]);
            fx[r] += share_fx(p, fx[c], 0);
            fx[n + r] += share_fx(p, fx[n + c], 1);
            if (shares) shares[r]++;
          } else {
            fx[r] += fx[c];
            fx[n + r] += fx[n + c];
          }
        } else if (shares) {
          shares[r]++;
        }
      }
      if (--deps[r] == 0) queue[qt++] = (int)r;
    }
  }
  for (size_t i = 0; i < n; i++) {
    const int nd = props[9 * i] == NO_DATA_GEN;
    ref[i] = nd ? -1.0 : (double)A[i];
    budget[i] = nd ? 0.0 : (double)(B[i] * (1.0L + ldexpl(1.0L, -50)));  /* rounded up past the double conversion */
    if (got) err[i] = nd ? (got[i] == -1.0 ? 0.0 : INFINITY) : (double)fabsl((long double)got[i] - A[i]);
    if (fx) {
      packed[i] = nd ? -1.0 : (double)fx[i] * (1.0 / 16777216.0);
      packed_fma[i] = nd ? -1.0 : (double)fx[n + i] * (1.0 / 16777216.0);
    }
  }
  free(A); free(B); free(Sabs); free(R); free(fx); free(deps); free(k); free(queue);
  return (int)(data - qt);
}
