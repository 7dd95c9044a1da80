// xivo_b200_io.hpp — header-only C++ I/O around the hot path (SURVEY.md §8f row 4): the ASL/EuRoC/TUM-VI folder loader
// with the reference's DataLoader surface (src/loader.h:12-31, src/loader.cpp:14-60), a binary PGM/PPM reader standing in
// for cv::imread (OpenCV C++ is not a dependency here), and the trajectory line of the `vio` app (src/app/vio.cpp:101-106).
// xivo_b200/dataio.py is the same thing in Python; tests/test_cpp_io.py checks the two against each other.
#ifndef XIVO_B200_IO_HPP_
#define XIVO_B200_IO_HPP_

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <iterator>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace xivo {
namespace msg {
struct Message {
  int64_t ts_ns;
  explicit Message(int64_t t) : ts_ns(t) {}
  virtual ~Message() {}
};
struct Image : Message {
  std::string image_path_;
  Image(int64_t t, std::string p) : Message(t), image_path_(std::move(p)) {}
};
struct IMU : Message {
  double gyro_[3], accel_[3];
  IMU(int64_t t, const double* g, const double* a) : Message(t) {
    for (int i = 0; i < 3; ++i) { gyro_[i] = g[i]; accel_[i] = a[i]; }
  }
};
}  // namespace msg

// whole file as bytes (the PNG frames handed to Estimator::VisualMeas(ts, path) / xivo_decode_png)
inline std::vector<uint8_t> ReadFileBytes(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::runtime_error("cannot open " + path);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

class DataLoader {
 public:
  DataLoader(const std::string& image_dir, const std::string& imu_dir) {
    load_images(image_dir);
    for (const auto& c : rows(imu_dir + "/data.csv")) {
      if (c.size() < 7) throw std::runtime_error("malformed IMU row in " + imu_dir + "/data.csv");
      double v[6];
      for (int i = 0; i < 6; ++i) v[i] = std::stod(c[i + 1]);
      entries_.emplace_back(new msg::IMU(std::stoll(c[0]), v, v + 3));
    }
    sort();
  }
  explicit DataLoader(const std::string& image_dir) {
    load_images(image_dir);
    sort();
  }
  msg::Message* Get(int i) const { return entries_[i].get(); }
  int size() const { return (int)entries_.size(); }

 private:
  std::vector<std::unique_ptr<msg::Message>> entries_;

  static std::vector<std::vector<std::string>> rows(const std::string& csv) {
    std::ifstream is(csv);
    if (!is) throw std::runtime_error("failed to open data.csv @ " + csv);  // reference: LOG(FATAL)
    std::vector<std::vector<std::string>> out;
    std::string line;
    std::getline(is, line);  // header
    while (is >> line) {     // whitespace-separated tokens, like the reference
      if (line.empty() || line.front() == '#') continue;
      std::vector<std::string> c;
      std::stringstream ss(line);
      std::string item;
      while (std::getline(ss, item, ',')) c.push_back(item);
      out.push_back(std::move(c));
    }
    return out;
  }
  void load_images(const std::string& image_dir) {
    for (const auto& c : rows(image_dir + "/data.csv")) {
      if (c.size() < 2) throw std::runtime_error("malformed image row in " + image_dir + "/data.csv");
      entries_.emplace_back(new msg::Image(std::stoll(c[0]), image_dir + "/data/" + c[1]));
    }
  }
  void sort() {  // ascending stamps; stable, so images (listed first) precede IMU samples with the same stamp
    std::stable_sort(entries_.begin(), entries_.end(), [](const auto& a, const auto& b) { return a->ts_ns < b->ts_ns; });
  }
};
// The pieces of a loaded sequence for xivo::Batch::Feed, as [begin, end) message ranges: the IMU messages up to and including the next
// image, and the IMU messages after the last image as a last piece.  Round r of a batch gives every sequence its r-th piece
// (xivo_b200.dataio.feed_rounds is the same rule in Python).
inline std::vector<std::pair<int, int>> FeedPieces(const DataLoader& loader) {
  std::vector<std::pair<int, int>> out;
  int begin = 0;
  for (int i = 0; i < loader.size(); ++i)
    if (dynamic_cast<const msg::Image*>(loader.Get(i))) {
      out.emplace_back(begin, i + 1);
      begin = i + 1;
    }
  if (begin < loader.size()) out.emplace_back(begin, loader.size());
  return out;
}
using TUMVILoader = DataLoader;
using EuRoCLoader = DataLoader;

// Binary PGM (1 channel) / PPM (3 channels, returned in BGR order like cv::imread).
struct PnmImage {
  std::vector<uint8_t> data;
  int rows = 0, cols = 0, channels = 0;
};
inline PnmImage ReadPnm(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::runtime_error("cannot open image " + path);
  std::string magic;
  int vals[3], n = 0;
  f >> magic;
  while (n < 3) {
    f >> std::ws;
    if (f.peek() == '#') { std::string skip; std::getline(f, skip); continue; }
    if (!(f >> vals[n])) throw std::runtime_error("bad PNM header in " + path);
    ++n;
  }
  f.get();  // the single whitespace after maxval
  if ((magic != "P5" && magic != "P6") || vals[2] != 255) throw std::runtime_error("unsupported PNM (need binary P5/P6, maxval 255): " + path);
  PnmImage im;
  im.cols = vals[0]; im.rows = vals[1]; im.channels = magic == "P5" ? 1 : 3;
  im.data.resize((size_t)im.rows * im.cols * im.channels);
  f.read(reinterpret_cast<char*>(im.data.data()), (std::streamsize)im.data.size());
  if ((size_t)f.gcount() != im.data.size()) throw std::runtime_error("truncated PNM " + path);
  if (im.channels == 3)
    for (size_t i = 0; i + 2 < im.data.size(); i += 3) std::swap(im.data[i], im.data[i + 2]);
  return im;
}

// so3().log() of a row-major 3x3 rotation (first 3 columns of a 3x4 pose).
inline void RotationVector(const double* g34, double w[3]) {
  const double R[3][3] = {{g34[0], g34[1], g34[2]}, {g34[4], g34[5], g34[6]}, {g34[8], g34[9], g34[10]}};
  double c = 0.5 * (R[0][0] + R[1][1] + R[2][2] - 1.0);
  c = c > 1 ? 1 : (c < -1 ? -1 : c);
  const double th = std::acos(c);
  const double v[3] = {R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]};
  if (th < 1e-9) { for (int i = 0; i < 3; ++i) w[i] = 0.5 * v[i]; return; }
  if (M_PI - th < 1e-6) {
    int k = 0;
    for (int i = 1; i < 3; ++i) if (R[i][i] > R[k][k]) k = i;
    double ax[3];
    const double akk = 0.5 * (R[k][k] + 1.0);
    for (int i = 0; i < 3; ++i) ax[i] = 0.5 * (R[i][k] + (i == k ? 1.0 : 0.0)) / std::sqrt(akk > 1e-300 ? akk : 1e-300);
    const double dot = ax[0] * v[0] + ax[1] * v[1] + ax[2] * v[2];
    for (int i = 0; i < 3; ++i) w[i] = (dot < 0 ? -th : th) * ax[i];
    return;
  }
  const double s = th / (2.0 * std::sin(th));
  for (int i = 0; i < 3; ++i) w[i] = s * v[i];
}

// One line of the `vio` app's output: "ts_ns Tx Ty Tz Wx Wy Wz".
inline std::string TrajectoryLine(int64_t ts_ns, const double* gsb34) {
  double w[3];
  RotationVector(gsb34, w);
  char buf[256];
  std::snprintf(buf, sizeof(buf), "%lld %.9g %.9g %.9g %.9g %.9g %.9g", (long long)ts_ns, gsb34[3], gsb34[7], gsb34[11], w[0], w[1], w[2]);
  return buf;
}

}  // namespace xivo
#endif
