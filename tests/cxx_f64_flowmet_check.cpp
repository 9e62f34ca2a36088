// Runs the float64 flow-metric, accumulation and terrain-attribute specialisations of include/richdem_b200.hpp (opt-in:
// RICHDEM_B200_F64) on rasters the GPU test writes from tests/golden/f64_flowmet_ref.npz, and writes what they return
// next to them; tests/test_gpu_f64_flowmet.py compares the outputs with the fixtures.  Every call goes through the
// reference's own template names on Array2D<double>, so a specialisation the macro failed to declare would run the CPU
// template instead: the launch count the library reports after each call shows that the GPU ran it.
//
//   cxx_f64_flowmet_check DIR NAME...   reads DIR/NAME.in (int32 width, int32 height, double nodata, width*height
//                                       doubles) and writes DIR/NAME.<call>.out (raw cells) and DIR/NAME.launches
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
    Array2D<double> r(w, h, 0.0);
    if (std::fread(r.data(), 8, n, f) != n) return 2;
    std::fclose(f);
    r.setNoData(nodata);
    r.geotransform = {0.0, 2.0, 0.0, 0.0, 0.0, -3.0};  // 2 x 3 cells, as the fixtures' attributes
    FILE *log = std::fopen((base + ".launches").c_str(), "w");
    auto launches = [&](const std::string &fn) {
      rdb200_stats s;
      richdem_b200::check(rdb200_get_stats(&s));
      std::fprintf(log, "%s %lld\n", fn.c_str(), (long long)s.kernel_launches);
    };
    try {
      auto props = [&](const std::string &name, auto call) {
        Array3D<float> p(w, h, 0.0f);
        call(p);
        launches(name);
        write_raw(base + "." + name + ".out", p.getData(), n * 9 * sizeof(float));
      };
      props("FM_D8", [&](Array3D<float> &p) { FM_D8(r, p); });
      props("FM_D4", [&](Array3D<float> &p) { FM_D4(r, p); });
      props("FM_Tarboton", [&](Array3D<float> &p) { FM_Tarboton(r, p); });
      props("FM_Dinfinity", [&](Array3D<float> &p) { FM_Dinfinity(r, p); });
      props("FM_Quinn", [&](Array3D<float> &p) { FM_Quinn(r, p); });
      props("FM_Holmgren_0.5", [&](Array3D<float> &p) { FM_Holmgren(r, p, 0.5); });
      props("FM_Freeman_1.1", [&](Array3D<float> &p) { FM_Freeman(r, p, 1.1); });
      props("FM_Freeman_4.0", [&](Array3D<float> &p) { FM_Freeman(r, p, 4.0); });
      auto accum = [&](const std::string &name, auto call) {
        Array2D<double> acc(w, h, 1.0);
        call(acc);
        launches(name);
        if (acc.noData() != ACCUM_NO_DATA) throw std::runtime_error("accumulation NoData not set");
        write_raw(base + "." + name + ".out", acc.data(), n * 8);
      };
      accum("FA_Tarboton", [&](Array2D<double> &acc) { FA_Tarboton(r, acc); });
      accum("FA_Dinfinity", [&](Array2D<double> &acc) { FA_Dinfinity(r, acc); });
      accum("FA_Quinn", [&](Array2D<double> &acc) { FA_Quinn(r, acc); });
      accum("FA_Holmgren_1.0", [&](Array2D<double> &acc) { FA_Holmgren(r, acc, 1.0); });
      accum("FA_Freeman_1.1", [&](Array2D<double> &acc) { FA_Freeman(r, acc, 1.1); });
      {
        Array2D<double> small(3, 3, 1.0);  // mismatched dimensions are refused, as by the float specialisations
        bool threw = false;
        try {
          FA_Quinn(r, small);
        } catch (const std::runtime_error &) {
          threw = true;
        }
        if (!threw) return 3;
      }
      auto attr = [&](const std::string &name, auto call) {
        Array2D<float> o(3, 5, 7.0f);  // a stale output of another size: resized like the reference does
        o.setNoData(-9999.0f);
        call(o);
        launches(name);
        if (o.width() != w || o.height() != h) throw std::runtime_error("attribute output not resized");
        write_raw(base + "." + name + ".out", o.data(), n * sizeof(float));
      };
      const float zs = 2.5f;
      attr("TA_slope_riserun", [&](Array2D<float> &o) { TA_slope_riserun(r, o, zs); });
      attr("TA_slope_percentage", [&](Array2D<float> &o) { TA_slope_percentage(r, o, zs); });
      attr("TA_slope_degrees", [&](Array2D<float> &o) { TA_slope_degrees(r, o, zs); });
      attr("TA_slope_radians", [&](Array2D<float> &o) { TA_slope_radians(r, o, zs); });
      attr("TA_aspect", [&](Array2D<float> &o) { TA_aspect(r, o, zs); });
      attr("TA_curvature", [&](Array2D<float> &o) { TA_curvature(r, o, zs); });
      attr("TA_planform_curvature", [&](Array2D<float> &o) { TA_planform_curvature(r, o, zs); });
      attr("TA_profile_curvature", [&](Array2D<float> &o) { TA_profile_curvature(r, o, zs); });
    } catch (const std::runtime_error &e) {
      std::fprintf(stderr, "%s: runtime_error: %s\n", argv[a], e.what());
      return 1;
    }
    std::fclose(log);
  }
  return 0;
}
