// Compile/link/run check of the pit_mask / HasDepressions specialisations in include/richdem_b200.hpp against the
// reference headers.  Calls on float rasters resolve to the H100 specialisations; the same templates instantiated for
// double elevations run the reference's CPU code, which serves as the in-process oracle (float values are exact in
// double, and both functions only compare elevations).  Without a GPU every H100 call must throw std::runtime_error.
#include <richdem_b200.hpp>

#include <cstdio>

using namespace richdem;

static unsigned lcg(unsigned &s) { return s = s * 1664525u + 1013904223u; }

int main() {
  const int W = 260, H = 197;
  int thrown = 0, calls = 0, mism = 0;
  auto attempt = [&](const char *name, auto &&fn) {
    calls++;
    try {
      fn();
      std::printf("%-32s ran\n", name);
      return true;
    } catch (const std::runtime_error &e) {
      thrown++;
      std::printf("%-32s runtime_error: %s\n", name, e.what());
      return false;
    }
  };
  auto as_double = [](const Array2D<float> &a) {
    Array2D<double> d(a.width(), a.height(), 0.0);
    for (int y = 0; y < a.height(); y++)
      for (int x = 0; x < a.width(); x++) d(x, y) = a(x, y);
    d.setNoData(a.noData());
    return d;
  };

  // rasters: terrain with strict pits and a NoData block; terraced terrain whose basins have flat floors only; a plane
  // that drains everywhere (no depression); the plane with one enclosed flat basin (a depression without a strict pit)
  Array2D<float> rough(W, H, 0.f), terraced(W, H, 0.f), plane(W, H, 0.f), basin(W, H, 0.f);
  unsigned seed = 777;
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      const float ridge = 40.f * ((x / 37 + y / 29) % 3);
      rough(x, y) = ridge + (float)(lcg(seed) >> 24) * 0.5f;
      terraced(x, y) = 10.f * (float)(((x / 23) * 7 + (y / 19) * 3) % 5);
      plane(x, y) = (float)(x + 2 * y);
      const int dx = x - W / 2, dy = y - H / 2;
      const int r2 = dx * dx + dy * dy;
      basin(x, y) = r2 < 15 * 15 ? 5.f : (r2 < 18 * 18 ? 1000.f : plane(x, y));
    }
  for (int y = 60; y < 90; y++)
    for (int x = 100; x < 170; x++) rough(x, y) = -9999.f;
  for (auto *a : {&rough, &terraced, &plane, &basin}) a->setNoData(-9999.f);

  const char *names[] = {"rough", "terraced", "plane", "basin"};
  Array2D<float> *rasters[] = {&rough, &terraced, &plane, &basin};
  const int expect_has[] = {1, -1, 0, 1};  // -1: whatever the reference says
  for (int k = 0; k < 4; k++) {
    const Array2D<float> &dem = *rasters[k];
    const Array2D<double> demd = as_double(dem);
    for (int topo = 0; topo < 2; topo++) {
      char name[64];
      std::snprintf(name, sizeof(name), "pit_mask<%s> %s", topo ? "D4" : "D8", names[k]);
      Array2D<uint8_t> mask(7, 3, 42), maskd;  // a stale output of another size: resized like the reference does
      if (attempt(name, [&] { topo ? pit_mask<Topology::D4>(dem, mask) : pit_mask<Topology::D8>(dem, mask); })) {
        topo ? pit_mask<Topology::D4>(demd, maskd) : pit_mask<Topology::D8>(demd, maskd);
        long bad = mask.width() != maskd.width() || mask.height() != maskd.height() || mask.noData() != maskd.noData();
        for (int y = 0; !bad && y < H; y++)
          for (int x = 0; x < W; x++) bad += mask(x, y) != maskd(x, y);
        std::printf("  %-30s %s (%ld cells differ)\n", name, bad ? "MISMATCH" : "identical", bad);
        if (bad) mism++;
      }
      std::snprintf(name, sizeof(name), "HasDepressions<%s> %s", topo ? "D4" : "D8", names[k]);
      bool got = false;
      if (attempt(name, [&] { got = topo ? HasDepressions<Topology::D4>(dem) : HasDepressions<Topology::D8>(dem); })) {
        const bool ref = topo ? HasDepressions<Topology::D4>(demd) : HasDepressions<Topology::D8>(demd);
        const bool ok = got == ref && (expect_has[k] < 0 || (int)ref == expect_has[k]);
        std::printf("  %-30s %s (got %d, reference %d)\n", name, ok ? "identical" : "MISMATCH", (int)got, (int)ref);
        if (!ok) mism++;
      }
    }
  }
  std::printf("calls=%d thrown=%d mismatches=%d\n", calls, thrown, mism);
  if (thrown != 0 && thrown != calls) return 2;  // partial failure
  return mism == 0 ? 0 : 1;
}
