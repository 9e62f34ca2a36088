/* TEST INFRASTRUCTURE ONLY -- plain-C restatement of the epsilon fill the GPU computes for FillDepressions(epsilon=True)
 * (richdem_b200/csrc/fill.cu, fill_sweep_kernel<2>; DESIGN.md section 0, f3).  Built by oracle/epsilon_fill.py into
 * oracle/libepsilon_fill_oracle.so, without -ffast-math and without flush-to-zero: the answer lives in the last ulp, and
 * subnormals are part of it (up(0) = denorm_min).
 *
 * With up(x) = nextafterf(x, +inf), the result W is the unique solution of
 *   W(c) = Z(c)                                          on the raster's border and where Z(c) == nodata,
 *   W(c) = max(Z(c), min over the neighbours n of up(W(n)))   elsewhere (8 neighbours for D8, 4 for D4).
 * It is computed by a Dijkstra flood in which entering a cell from a closed one costs max(Z, up(cost so far)): that cost
 * never decreases along a path, so the cells close in non-decreasing W.  The open set is a binary heap ordered by
 * (value, index), so the run does not depend on how ties fall; the result would not either. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
  float v;
  int64_t i;
} item;

static int before(item a, item b) { return a.v < b.v || (a.v == b.v && a.i < b.i); }

typedef struct {
  item *a;
  size_t n, cap;
} heap;

static int push(heap *h, float v, int64_t i) {
  if (h->n == h->cap) {
    const size_t cap = h->cap ? 2 * h->cap : 1024;
    item *a = (item *)realloc(h->a, cap * sizeof(item));
    if (!a) return -1;
    h->a = a;
    h->cap = cap;
  }
  size_t k = h->n++;
  const item x = {v, i};
  while (k > 0) {
    const size_t p = (k - 1) / 2;
    if (!before(x, h->a[p])) break;
    h->a[k] = h->a[p];
    k = p;
  }
  h->a[k] = x;
  return 0;
}

static item pop(heap *h) {
  const item top = h->a[0];
  const item x = h->a[--h->n];
  size_t k = 0;
  for (;;) {
    size_t c = 2 * k + 1;
    if (c >= h->n) break;
    if (c + 1 < h->n && before(h->a[c + 1], h->a[c])) c++;
    if (!before(h->a[c], x)) break;
    h->a[k] = h->a[c];
    k = c;
  }
  if (h->n) h->a[k] = x;
  return top;
}

/* topo: 0 D8, 1 D4.  dem (w x h, row-major) is replaced by W.  Returns 0, or -1 when memory runs out. */
int orc_epsilon_fill_f32(int topo, float *dem, int w, int h, float nodata) {
  static const int dx8[8] = {-1, 0, 1, 1, 1, 0, -1, -1}, dy8[8] = {-1, -1, -1, 0, 1, 1, 1, 0};
  static const int dx4[4] = {0, 1, 0, -1}, dy4[4] = {-1, 0, 1, 0};
  const int nn = topo ? 4 : 8;
  const int *dx = topo ? dx4 : dx8, *dy = topo ? dy4 : dy8;
  const int64_t n = (int64_t)w * h;
  float *W = (float *)malloc((size_t)n * sizeof(float));
  unsigned char *done = (unsigned char *)calloc((size_t)n, 1);
  heap q = {NULL, 0, 0};
  int rc = W && done ? 0 : -1;
  for (int64_t i = 0; i < n && rc == 0; i++) {
    const int x = (int)(i % w), y = (int)(i / w);
    const int pinned = x == 0 || y == 0 || x == w - 1 || y == h - 1 || dem[i] == nodata;
    W[i] = pinned ? dem[i] : INFINITY;
    if (pinned) rc = push(&q, W[i], i);
  }
  while (rc == 0 && q.n) {
    const item c = pop(&q);
    if (done[c.i]) continue;
    done[c.i] = 1;
    const float up = nextafterf(W[c.i], INFINITY);
    const int x = (int)(c.i % w), y = (int)(c.i / w);
    for (int k = 0; k < nn && rc == 0; k++) {
      const int xx = x + dx[k], yy = y + dy[k];
      if (xx < 0 || yy < 0 || xx >= w || yy >= h) continue;
      const int64_t j = (int64_t)yy * w + xx;
      if (done[j]) continue;
      const float v = dem[j] > up ? dem[j] : up;
      if (v < W[j]) {
        W[j] = v;
        rc = push(&q, v, j);
      }
    }
  }
  if (rc == 0)
    for (int64_t i = 0; i < n; i++) dem[i] = W[i];
  free(W);
  free(done);
  free(q.a);
  return rc;
}
