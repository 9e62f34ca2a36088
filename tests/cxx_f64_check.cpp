// Runs the float64 specialisations of include/richdem_b200.hpp (opt-in: RICHDEM_B200_F64) on rasters the GPU test writes
// from tests/golden/f64_ref.npz, and writes what they return next to them; tests/test_gpu_f64.py compares the outputs with
// the fixtures (the unmodified reference's double templates).  Every call goes through the reference's own template
// names, so a specialisation the macro failed to declare would run the CPU template instead: the launch count the
// library reports after each call shows that the GPU ran it.
//
//   cxx_f64_check DIR NAME...   reads DIR/NAME.in (int32 width, int32 height, double nodata, width*height doubles) and
//                               writes DIR/NAME.<function>.out (raw cells) and DIR/NAME.launches (one line per call)
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
    auto raster = [&] {
      Array2D<double> r(w, h, 0.0);
      std::memcpy(r.data(), z.data(), n * sizeof(double));
      r.setNoData(nodata);
      return r;
    };
    FILE *log = std::fopen((base + ".launches").c_str(), "w");
    auto launches = [&](const char *fn) {
      rdb200_stats s;
      richdem_b200::check(rdb200_get_stats(&s));
      std::fprintf(log, "%s %lld\n", fn, (long long)s.kernel_launches);
    };
    try {
      {
        Array2D<double> r = raster();
        FillDepressions<Topology::D8>(r);
        launches("FillDepressions_D8");
        write_raw(base + ".fill_D8.out", r.data(), n * 8);
      }
      {
        Array2D<double> r = raster();
        FillDepressions<Topology::D4>(r);
        launches("FillDepressions_D4");
        write_raw(base + ".fill_D4.out", r.data(), n * 8);
      }
      {
        Array2D<double> r = raster();
        PriorityFlood_Zhou2016(r);
        launches("PriorityFlood_Zhou2016");
        write_raw(base + ".zhou.out", r.data(), n * 8);
      }
      {
        Array2D<double> r = raster();
        PriorityFlood_Barnes2014<Topology::D4>(r);
        launches("PriorityFlood_Barnes2014_D4");
        write_raw(base + ".barnes_D4.out", r.data(), n * 8);
      }
      const Array2D<double> r = raster();
      for (int topo = 0; topo < 2; topo++) {
        Array2D<uint8_t> m(3, 5, 42);  // a stale output of another size: resized like the reference does
        topo ? pit_mask<Topology::D4>(r, m) : pit_mask<Topology::D8>(r, m);
        launches(topo ? "pit_mask_D4" : "pit_mask_D8");
        if (m.width() != w || m.height() != h || m.noData() != 3) return 3;
        write_raw(base + (topo ? ".mask_D4.out" : ".mask_D8.out"), m.data(), n);
        const int32_t has = topo ? HasDepressions<Topology::D4>(r) : HasDepressions<Topology::D8>(r);
        launches(topo ? "HasDepressions_D4" : "HasDepressions_D8");
        write_raw(base + (topo ? ".has_D4.out" : ".has_D8.out"), &has, 4);
      }
      {
        Array2D<double> q = raster();
        ResolveFlatsEpsilon(q);
        launches("ResolveFlatsEpsilon");
        write_raw(base + ".resolved.out", q.data(), n * 8);
      }
      {
        Array2D<uint8_t> d;
        d8_flow_directions(r, d);
        launches("d8_flow_directions");
        write_raw(base + ".dirs.out", d.data(), n);
      }
      for (int topo = 0; topo < 2; topo++) {
        Array2D<double> acc(w, h, 1.0);
        topo ? FA_D4(r, acc) : FA_D8(r, acc);
        launches(topo ? "FA_D4" : "FA_D8");
        write_raw(base + (topo ? ".fa_D4.out" : ".fa_D8.out"), acc.data(), n * 8);
      }
    } catch (const std::runtime_error &e) {
      std::fprintf(stderr, "%s: runtime_error: %s\n", argv[a], e.what());
      return 1;
    }
    std::fclose(log);
  }
  return 0;
}
