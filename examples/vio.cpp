// vio — the reference's command-line VIO application (src/app/vio.cpp) on top of xivo_b200:
//   vio <estimator_cfg.json> <image_dir> <imu_dir> <out_state> [max_groups max_features]
// reads an ASL / EuRoC / TUM-VI style sequence (cam0/data.csv with PNG or PGM/PPM frames, imu0/data.csv), feeds it message by
// message to xivo::Estimator and writes "ts Tsb Wsb" after every message, like the reference does (vio.cpp:101-106).  PNG frames
// (file name ending in .png) go through Estimator::VisualMeas(ts, path), decoded on the device like cv::imread(path).
// `--list` stops after loading and prints the merged message list (used by the CPU test of the loader); for a PNG frame it prints
// the file's geometry (xivo_png_info) and size in bytes instead of the pixel checksum.
// Build: g++ -std=c++17 -O2 -I include examples/vio.cpp -o vio -L xivo_b200 -lxivo_b200 -Wl,-rpath,$PWD/xivo_b200
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>

#include "xivo_b200.hpp"
#include "xivo_b200_io.hpp"

static bool is_png(const std::string& p) { return p.size() >= 4 && p.compare(p.size() - 4, 4, ".png") == 0; }

int main(int argc, char** argv) {
  if (argc >= 4 && !std::strcmp(argv[1], "--list")) {
    try {
      xivo::DataLoader loader(argv[2], argv[3]);
      for (int i = 0; i < loader.size(); ++i) {
        auto* m = loader.Get(i);
        if (auto* im = dynamic_cast<xivo::msg::Image*>(m)) {
          if (is_png(im->image_path_)) {
            const auto bytes = xivo::ReadFileBytes(im->image_path_);
            int rows = 0, cols = 0, ch = 0, bits = 0;
            if (xivo_png_info(bytes.data(), bytes.size(), &rows, &cols, &ch, &bits)) throw std::runtime_error(im->image_path_ + ": " + xivo_last_error());
            std::printf("img %lld %dx%dx%d %zu\n", (long long)im->ts_ns, rows, cols, ch, bytes.size());
            continue;
          }
          auto px = xivo::ReadPnm(im->image_path_);
          unsigned long long sum = 0;
          for (uint8_t v : px.data) sum += v;
          std::printf("img %lld %dx%dx%d %llu\n", (long long)im->ts_ns, px.rows, px.cols, px.channels, sum);
        } else if (auto* mu = dynamic_cast<xivo::msg::IMU*>(m)) {
          std::printf("imu %lld %.17g %.17g %.17g %.17g %.17g %.17g\n", (long long)mu->ts_ns, mu->gyro_[0], mu->gyro_[1], mu->gyro_[2], mu->accel_[0],
                      mu->accel_[1], mu->accel_[2]);
        }
      }
      return 0;
    } catch (const std::exception& e) {
      std::fprintf(stderr, "%s\n", e.what());
      return 2;
    }
  }
  if (argc < 5) {
    std::fprintf(stderr, "usage: %s <estimator_cfg.json> <image_dir> <imu_dir> <out_state> [max_groups max_features]\n", argv[0]);
    return 1;
  }
  const int G = argc > 6 ? std::atoi(argv[5]) : 15, F = argc > 6 ? std::atoi(argv[6]) : 30;
  try {
    xivo::DataLoader loader(argv[2], argv[3]);
    auto est = xivo::Estimator::CreateFromFile(argv[1], G, F);
    std::ofstream out(argv[4]);
    if (!out) throw std::runtime_error(std::string("cannot write ") + argv[4]);
    for (int i = 0; i < loader.size(); ++i) {
      auto* m = loader.Get(i);
      if (auto* im = dynamic_cast<xivo::msg::Image*>(m)) {
        if (is_png(im->image_path_)) {
          est->VisualMeas(xivo::timestamp_t(im->ts_ns), im->image_path_);
        } else {
          auto px = xivo::ReadPnm(im->image_path_);
          est->VisualMeas(xivo::timestamp_t(im->ts_ns), xivo::ImageView{px.data.data(), px.rows, px.cols, px.channels});
        }
      } else if (auto* mu = dynamic_cast<xivo::msg::IMU*>(m)) {
        est->InertialMeas(xivo::timestamp_t(mu->ts_ns), {mu->gyro_[0], mu->gyro_[1], mu->gyro_[2]}, {mu->accel_[0], mu->accel_[1], mu->accel_[2]});
      }
      const auto g = est->gsb();
      out << xivo::TrajectoryLine(est->ts().count(), g.data()) << "\n";
    }
    std::printf("processed %d messages, %d in-state features, %d groups\n", loader.size(), est->num_instate_features(), est->num_instate_groups());
    return 0;
  } catch (const xivo::Error& e) {
    std::fprintf(stderr, "xivo::Error %d: %s\n", e.code, e.what());
    return e.code == XIVO_ERR_CUDA ? 42 : 3;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 2;
  }
}
