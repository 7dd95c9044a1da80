// vio — the reference's command-line VIO application (src/app/vio.cpp) on top of xivo_b200:
//   vio <estimator_cfg.json> <image_dir> <imu_dir> <out_state> [max_groups max_features]
// reads an ASL / EuRoC / TUM-VI style sequence (cam0/data.csv with PNG or PGM/PPM frames, imu0/data.csv), feeds it message by
// message to xivo::Estimator and writes "ts Tsb Wsb" after every message, like the reference does (vio.cpp:101-106).  PNG frames
// (file name ending in .png) go through Estimator::VisualMeas(ts, path), decoded on the device like cv::imread(path).
// `--list` stops after loading and prints the merged message list (used by the CPU test of the loader); for a PNG frame it prints
// the file's geometry (xivo_png_info) and size in bytes instead of the pixel checksum.
//   vio --batch <estimator_cfg.json> <list.txt> [max_groups max_features]
// runs every sequence of list.txt in one xivo::Batch handle.  Each line of the list is `image_dir imu_dir out_state [cfg.json]` (empty
// lines and lines starting with '#' are skipped); a line's own config, which must agree with the handle's on the batch-wide settings,
// is applied with ResetSequence before the first message.  Round r gives every sequence its r-th piece (xivo::FeedPieces: its IMU
// messages up to and including its next frame), PNM frames through Batch::Feed and PNG frames through Batch::FeedPng, and after each
// round the trajectory line of every sequence that received a frame is written to its out_state: the lines a solo run writes at
// that sequence's frame messages.  `--batch --plan <list.txt>` stops after loading and prints one line per piece:
// `round sequence n_imu frame_ts` (`-` for a piece without a frame).
//   vio --batch --isolate-failures <estimator_cfg.json> <list.txt> [max_groups max_features]
// confines a failure to its sequence (Batch::IsolateFailures): a sequence that fails is reported on stderr with its image_dir and
// message, its out_state ends at its last frame before the failure, the other sequences run to their end, and the exit status is 4.
// Build: g++ -std=c++17 -O2 -I include examples/vio.cpp -o vio -L xivo_b200 -lxivo_b200 -Wl,-rpath,$PWD/xivo_b200
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "xivo_b200.hpp"
#include "xivo_b200_io.hpp"

static bool is_png(const std::string& p) { return p.size() >= 4 && p.compare(p.size() - 4, 4, ".png") == 0; }

static std::string read_text(const std::string& path) {
  std::ifstream f(path);
  if (!f) throw std::runtime_error("cannot open " + path);
  return std::string((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

struct SeqLine {
  std::string image_dir, imu_dir, out_state, cfg;
};

static std::vector<SeqLine> read_list(const std::string& path) {
  std::ifstream f(path);
  if (!f) throw std::runtime_error("cannot open " + path);
  std::vector<SeqLine> out;
  std::string line;
  while (std::getline(f, line)) {
    std::istringstream ss(line);
    SeqLine l;
    if (!(ss >> l.image_dir) || l.image_dir[0] == '#') continue;
    if (!(ss >> l.imu_dir >> l.out_state)) throw std::runtime_error(path + ": a line needs image_dir imu_dir out_state [cfg.json]: " + line);
    ss >> l.cfg;
    out.push_back(l);
  }
  if (out.empty()) throw std::runtime_error(path + " lists no sequence");
  return out;
}

static int run_batch(int argc, char** argv_in) {
  std::vector<char*> args(argv_in, argv_in + argc);
  const bool isolate = argc >= 3 && !std::strcmp(args[2], "--isolate-failures");
  if (isolate) args.erase(args.begin() + 2);
  argc = (int)args.size();
  char** argv = args.data();
  const bool plan = argc >= 4 && !std::strcmp(argv[2], "--plan");
  if (argc < 4) {
    std::fprintf(stderr, "usage: %s --batch [--isolate-failures] <estimator_cfg.json> <list.txt> [max_groups max_features] | --batch --plan <list.txt>\n", argv[0]);
    return 1;
  }
  const std::vector<SeqLine> list = read_list(argv[3]);
  const int B = (int)list.size();
  std::vector<std::unique_ptr<xivo::DataLoader>> loaders;
  std::vector<std::vector<std::pair<int, int>>> pieces;
  size_t rounds = 0;
  for (const auto& l : list) {
    loaders.emplace_back(new xivo::DataLoader(l.image_dir, l.imu_dir));
    pieces.push_back(xivo::FeedPieces(*loaders.back()));
    rounds = std::max(rounds, pieces.back().size());
  }
  auto frame_of = [&](int s, size_t r) -> const xivo::msg::Image* {  // the frame ending sequence s's piece r, or null
    if (r >= pieces[s].size()) return nullptr;
    return dynamic_cast<const xivo::msg::Image*>(loaders[s]->Get(pieces[s][r].second - 1));
  };
  if (plan) {
    for (size_t r = 0; r < rounds; ++r)
      for (int s = 0; s < B; ++s) {
        if (r >= pieces[s].size()) continue;
        const auto* im = frame_of(s, r);
        const int n_imu = pieces[s][r].second - pieces[s][r].first - (im ? 1 : 0);
        if (im) std::printf("%zu %d %d %lld\n", r, s, n_imu, (long long)im->ts_ns);
        else std::printf("%zu %d %d -\n", r, s, n_imu);
      }
    return 0;
  }
  const int G = argc > 5 ? std::atoi(argv[4]) : 15, F = argc > 5 ? std::atoi(argv[5]) : 30;
  xivo::Batch batch(read_text(argv[2]), B, G, F);
  if (isolate) batch.IsolateFailures(true);
  std::vector<char> failed(B, 0);
  // an isolating handle: report the sequences that failed during a call; their trajectories end here
  auto report = [&](bool ok) {
    if (ok) return;
    for (const auto& kv : batch.Failed())
      if (!failed[kv.first]) {
        failed[kv.first] = 1;
        std::fprintf(stderr, "sequence %d (%s) failed: error %d: %s\n", kv.first, list[kv.first].image_dir.c_str(), kv.second.code, kv.second.msg.c_str());
      }
  };
  std::vector<std::ofstream> out(B);
  for (int s = 0; s < B; ++s) {
    if (!list[s].cfg.empty()) {
      try {
        batch.ResetSequence(s, read_text(list[s].cfg));
      } catch (const xivo::Error& e) {
        throw xivo::Error(e.code, list[s].cfg + ": " + e.what());
      }
    }
    out[s].open(list[s].out_state);
    if (!out[s]) throw std::runtime_error("cannot write " + list[s].out_state);
  }
  for (size_t r = 0; r < rounds; ++r) {
    std::vector<xivo::Batch::Input> pnm(B), png(B);
    std::vector<xivo::PnmImage> pixels(B);
    bool any_pnm = false, any_png = false;
    for (int s = 0; s < B; ++s) {
      if (r >= pieces[s].size()) continue;
      xivo::Batch::Input& in = pnm[s];  // the IMU samples go with the first call of the round
      for (int i = pieces[s][r].first; i < pieces[s][r].second; ++i)
        if (auto* mu = dynamic_cast<const xivo::msg::IMU*>(loaders[s]->Get(i))) {
          in.imu_ts.push_back((uint64_t)mu->ts_ns);
          in.gyro.push_back({mu->gyro_[0], mu->gyro_[1], mu->gyro_[2]});
          in.accel.push_back({mu->accel_[0], mu->accel_[1], mu->accel_[2]});
        }
      const auto* im = frame_of(s, r);
      if (!im) continue;
      if (is_png(im->image_path_)) {
        png[s].has_frame = any_png = true;
        png[s].frame_ts = (uint64_t)im->ts_ns;
        png[s].png = xivo::ReadFileBytes(im->image_path_);
      } else {
        pixels[s] = xivo::ReadPnm(im->image_path_);
        in.has_frame = any_pnm = true;
        in.frame_ts = (uint64_t)im->ts_ns;
        in.image = xivo::ImageView{pixels[s].data.data(), pixels[s].rows, pixels[s].cols, pixels[s].channels};
      }
    }
    if (any_pnm || !any_png) report(batch.Feed(pnm));
    if (any_png) {
      if (!any_pnm)  // the round's only call carries the IMU samples
        for (int s = 0; s < B; ++s) {
          png[s].imu_ts.swap(pnm[s].imu_ts);
          png[s].gyro.swap(pnm[s].gyro);
          png[s].accel.swap(pnm[s].accel);
        }
      report(batch.FeedPng(png));
    }
    for (int s = 0; s < B; ++s)
      if (frame_of(s, r) && !failed[s]) {
        const auto g = batch.gsb(s);
        out[s] << xivo::TrajectoryLine(batch.ts(s).count(), g.data()) << "\n";
      }
  }
  int n_failed = 0;
  for (int s = 0; s < B; ++s) {
    if (failed[s]) {
      std::printf("sequence %d: %d messages, failed\n", s, loaders[s]->size());
      ++n_failed;
      continue;
    }
    std::printf("sequence %d: %d messages, %d in-state features, %d groups\n", s, loaders[s]->size(), batch.num_instate_features(s),
                batch.num_instate_groups(s));
  }
  return n_failed ? 4 : 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !std::strcmp(argv[1], "--batch")) {
    try {
      return run_batch(argc, argv);
    } catch (const xivo::Error& e) {
      std::fprintf(stderr, "xivo::Error %d: %s\n", e.code, e.what());
      return e.code == XIVO_ERR_CUDA ? 42 : 3;
    } catch (const std::exception& e) {
      std::fprintf(stderr, "%s\n", e.what());
      return 2;
    }
  }
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
