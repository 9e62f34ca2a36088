/* TEST INFRASTRUCTURE ONLY -- plain-C restatement of pit_mask<topo> and HasDepressions<topo>
 * (reference include/richdem/depressions/Barnes2014.hpp:593-676, :43-104) for the tests and the GPU box, where the
 * reference tree is absent.  Built by oracle/depressions.py into oracle/libdepressions_oracle.so, linked against
 * oracle/liboracle.so for the fill.
 *
 * Both are order-free functions of the Priority-Flood fill L of Z (NoData an ordinary value): the reference pops cells
 * in non-decreasing level, so the level an interior cell is discovered at is L of its lowest-level neighbour, and
 *   mask = 3 where Z == nodata, 1 where Z < L, 0 elsewhere (the cells the reference never writes keep resize()'s 0);
 *   HasDepressions = some cell has Z < L.
 * (See richdem_b200/csrc/depressions.cu for the argument.) */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void orc_fill_depressions_d8_f32(float *dem, int w, int h);
void orc_fill_depressions_d4_f32(float *dem, int w, int h);

/* topo: 0 D8, 1 D4.  mask may be null; returns 1 if some cell lies below the fill. */
int orc_pit_mask_f32(int topo, const float *dem, int w, int h, float nodata, uint8_t *mask) {
  const size_t n = (size_t)w * h;
  float *lvl = (float *)malloc(n * sizeof(float));
  int any = 0;
  memcpy(lvl, dem, n * sizeof(float));
  if (topo) orc_fill_depressions_d4_f32(lvl, w, h);
  else orc_fill_depressions_d8_f32(lvl, w, h);
  for (size_t i = 0; i < n; i++) {
    const int below = dem[i] < lvl[i];
    any |= below;
    if (mask) mask[i] = dem[i] == nodata ? 3 : (uint8_t)below;
  }
  free(lvl);
  return any;
}

int orc_has_depressions_f32(int topo, const float *dem, int w, int h) {
  return orc_pit_mask_f32(topo, dem, w, h, 0.f, NULL);
}
