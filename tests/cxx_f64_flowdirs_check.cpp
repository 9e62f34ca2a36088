// Runs barnes_flat_resolution_d8<double, uint8_t> of include/richdem_b200.hpp (opt-in: RICHDEM_B200_F64) on rasters the
// GPU test writes from tests/golden/f64_flowdirs_flats_ref.npz, and writes what it returns next to them;
// tests/test_gpu_f64_flowdirs_flats.py compares the outputs with the fixtures (the unmodified reference's double template).
// The call goes through the reference's own template name, so a specialisation the macro failed to declare would run the
// CPU template instead: the launch count the library reports after each call shows that the GPU ran it.
//
//   cxx_f64_flowdirs_check DIR NAME...   reads DIR/NAME.in (int32 width, int32 height, double nodata, width*height
//                                        doubles) and writes DIR/NAME.dirs<alter>.out, DIR/NAME.dem<alter>.out and
//                                        DIR/NAME.launches (one line per call)
#define RICHDEM_B200_F64
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
    double nodata;
    if (std::fread(wh, 4, 2, f) != 2 || std::fread(&nodata, 8, 1, f) != 1) return 2;
    const int w = wh[0], h = wh[1];
    const size_t n = (size_t)w * h;
    std::vector<double> z(n);
    if (std::fread(z.data(), 8, n, f) != n) return 2;
    std::fclose(f);
    FILE *log = std::fopen((base + ".launches").c_str(), "w");
    try {
      for (int alter = 0; alter < 2; alter++) {
        Array2D<double> r(w, h, 0.0);
        std::memcpy(r.data(), z.data(), n * sizeof(double));
        r.setNoData(nodata);
        Array2D<uint8_t> d(3, 5, 42);  // a stale output of another size: resized like the reference does
        barnes_flat_resolution_d8(r, d, alter != 0);
        rdb200_stats s;
        richdem_b200::check(rdb200_get_stats(&s));
        std::fprintf(log, "barnes_flat_resolution_d8_%d %lld\n", alter, (long long)s.kernel_launches);
        if (d.width() != w || d.height() != h) return 3;
        write_raw(base + ".dirs" + std::to_string(alter) + ".out", d.data(), n);
        write_raw(base + ".dem" + std::to_string(alter) + ".out", r.data(), n * 8);
      }
    } catch (const std::runtime_error &e) {
      std::fprintf(stderr, "%s: runtime_error: %s\n", argv[a], e.what());
      return 1;
    }
    std::fclose(log);
  }
  return 0;
}
