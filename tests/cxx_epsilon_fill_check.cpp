// Runs the epsilon-fill specialisations of include/richdem_b200.hpp (opt-in: RICHDEM_B200_EPSILON) on rasters the GPU
// test writes, and writes what they return next to them; tests/test_gpu_epsilon_fill.py compares the outputs with the C
// ABI's.  Every call goes through the reference's own template names, so a specialisation the macro failed to declare
// would run the CPU template instead: the launch count the library reports after each call shows that the GPU ran it.
//
//   cxx_epsilon_fill_check DIR NAME...   reads DIR/NAME.in (int32 width, int32 height, float nodata, width*height floats)
//                                        and writes DIR/NAME.<function>.out (raw cells) and DIR/NAME.launches
#define RICHDEM_B200_EPSILON
#include <richdem_b200.hpp>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

using namespace richdem;

static bool write_raw(const std::string &path, const void *p, size_t bytes) {
  FILE *f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  const bool ok = std::fwrite(p, 1, bytes, f) == bytes;
  std::fclose(f);
  return ok;
}

int main(int argc, char **argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s DIR NAME...\n", argv[0]);
    return 2;
  }
  const std::string dir = argv[1];
  for (int a = 2; a < argc; a++) {
    const std::string base = dir + "/" + argv[a];
    FILE *f = std::fopen((base + ".in").c_str(), "rb");
    if (!f) return 2;
    int32_t wh[2];
    float nodata;
    if (std::fread(wh, 4, 2, f) != 2 || std::fread(&nodata, 4, 1, f) != 1) return 2;
    const int w = wh[0], h = wh[1];
    const size_t n = (size_t)w * h;
    std::vector<float> z(n);
    if (std::fread(z.data(), 4, n, f) != n) return 2;
    std::fclose(f);
    FILE *log = std::fopen((base + ".launches").c_str(), "w");
    if (!log) return 2;
    try {
      auto run = [&](const char *fn, auto &&call) {
        Array2D<float> r(w, h, 0.f);
        std::memcpy(r.data(), z.data(), n * sizeof(float));
        r.setNoData(nodata);
        call(r);
        rdb200_stats s;
        richdem_b200::check(rdb200_get_stats(&s));
        std::fprintf(log, "%s %lld\n", fn, (long long)s.kernel_launches);
        if (!write_raw(base + "." + fn + ".out", r.data(), n * sizeof(float))) throw std::runtime_error("write failed");
      };
      run("PriorityFloodEpsilon_D8", [](Array2D<float> &r) { PriorityFloodEpsilon_Barnes2014<Topology::D8>(r); });
      run("PriorityFloodEpsilon_D4", [](Array2D<float> &r) { PriorityFloodEpsilon_Barnes2014<Topology::D4>(r); });
      run("FillDepressionsEpsilon_D8", [](Array2D<float> &r) { FillDepressionsEpsilon<Topology::D8>(r); });
      run("FillDepressionsEpsilon_D4", [](Array2D<float> &r) { FillDepressionsEpsilon<Topology::D4>(r); });
    } catch (const std::exception &e) {
      std::fprintf(stderr, "%s: %s\n", argv[a], e.what());
      std::fclose(log);
      return 1;
    }
    std::fclose(log);
  }
  return 0;
}
