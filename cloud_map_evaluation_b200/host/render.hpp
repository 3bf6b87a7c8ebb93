// render.hpp — the rendered clouds MapEval saves next to map_results.txt (SURVEY.md §8f N3): points coloured by entropy
// or by nearest-neighbour distance.  Host-side only: the per-point entropies and nearest-neighbour distances come from
// the GPU through me_get_entropies / me_get_nn, the coordinates through me_get_cloud.
//
// Reference: MapEval::ColorPointCloudByMME (map_eval.cpp:686-736), renderDistanceOnPointCloud / computePointCloudDistance
// (:568-606), saveMmeResults (:404-412), saveRegistrationResults (:485-499).  [ext] open3d::visualization::ColorMapJet and
// open3d::io::WritePointCloud (binary PCD, colours packed into one float field) are restated from Open3D 0.15-0.17.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

namespace render {

// [ext] open3d::visualization::ColorMap::Interpolate / ColorMapJet::JetBase / GetColor
inline double interpolate(double value, double y0, double x0, double y1, double x1) {
  if (value < x0) return y0;
  if (value > x1) return y1;
  return (value - x0) * (y1 - y0) / (x1 - x0) + y0;
}
inline double jet_base(double value) {
  if (value <= -0.75) return 0.0;
  if (value <= -0.25) return interpolate(value, 0.0, -0.75, 1.0, -0.25);
  if (value <= 0.25) return 1.0;
  if (value <= 0.75) return interpolate(value, 1.0, 0.25, 0.0, 0.75);
  return 0.0;
}
inline void jet(double value, double rgb[3]) {
  rgb[0] = jet_base(value * 2.0 - 1.5);
  rgb[1] = jet_base(value * 2.0 - 1.0);
  rgb[2] = jet_base(value * 2.0 - 0.5);
}
// [ext] open3d ColorToUint8: round(clamp(c, 0, 1) * 255)
inline uint8_t to_u8(double c) { return (uint8_t)std::round(std::min(1.0, std::max(0.0, c)) * 255.0); }

struct ColoredCloud {
  std::vector<float> xyz;       // the PCD stores single precision
  std::vector<uint8_t> rgb;     // 3 per point
  size_t size() const { return xyz.size() / 3; }
  void push(const double *p, const double c[3]) {
    for (int a = 0; a < 3; ++a) xyz.push_back((float)p[a]);
    for (int a = 0; a < 3; ++a) rgb.push_back(to_u8(c[a]));
  }
};

// ColorPointCloudByMME (map_eval.cpp:686-736): valid points only, |entropy| normalised between the extrema of the
// non-zero entropies, log-mapped with epsilon = 0.1, jet colour.  (The reference keys validity on the shared
// valid_entropy_points vector, which it never clears between the est and GT calls — SURVEY.md §5; here a point is valid
// iff its own entropy is non-zero.)
inline ColoredCloud color_by_entropy(const std::vector<double> &xyz, const std::vector<double> &entropy) {
  ColoredCloud out;
  double mn = INFINITY, mx = -INFINITY;
  for (double e : entropy)
    if (e != 0.0) { mn = std::min(mn, e); mx = std::max(mx, e); }
  if (!(mn <= mx)) return out;
  const double max_abs = std::fabs(mn), min_abs = std::fabs(mx);      // :700-701
  const double epsilon = 1e-1;
  for (size_t i = 0; i < entropy.size(); ++i) {
    if (entropy[i] == 0.0) continue;
    double normalized = (std::fabs(entropy[i]) - min_abs) / (max_abs - min_abs);
    const double mapped = std::log(normalized + epsilon);
    normalized = (mapped - std::log(epsilon)) / (std::log(1.0 + epsilon) - std::log(epsilon));
    double c[3];
    jet(normalized, c);
    out.push(&xyz[3 * i], c);
  }
  return out;
}

// renderDistanceOnPointCloud (map_eval.cpp:586-606) on distances already computed: value clipped at `dis`, jet(value / dis).
// NOTE the reference feeds it the SQUARED nearest-neighbour distance (computePointCloudDistance returns SearchKNN's
// distance2, :579-580) and clips it against the un-squared threshold; reproduced as written.
inline ColoredCloud color_by_distance(const std::vector<double> &xyz, const std::vector<double> &sqdist, double dis) {
  ColoredCloud out;
  for (size_t i = 0; i < sqdist.size(); ++i) {
    double d = sqdist[i];
    if (!(d == d)) d = dis;                       // no neighbour found
    if (d > dis) d = dis;
    double c[3];
    jet(d / dis, c);
    out.push(&xyz[3 * i], c);
  }
  return out;
}

// [ext] open3d::io::WritePointCloudToPCD, binary: FIELDS x y z rgb, rgb = (r << 16 | g << 8 | b) reinterpreted as float
inline bool write_pcd(const std::string &path, const ColoredCloud &c) {
  std::ofstream f(path, std::ios::binary);
  if (!f.is_open()) return false;
  const size_t n = c.size();
  f << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z rgb\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
    << "WIDTH " << n << "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << n << "\nDATA binary\n";
  std::vector<char> buf(n * 16);
  for (size_t i = 0; i < n; ++i) {
    std::memcpy(&buf[i * 16], &c.xyz[3 * i], 12);
    const uint32_t packed = ((uint32_t)c.rgb[3 * i] << 16) | ((uint32_t)c.rgb[3 * i + 1] << 8) | (uint32_t)c.rgb[3 * i + 2];
    std::memcpy(&buf[i * 16 + 12], &packed, 4);
  }
  f.write(buf.data(), (std::streamsize)buf.size());
  return (bool)f;
}

// the same binary layout without colours: FIELDS x y z, float32 (noise_gt_map.pcd, map_eval.cpp:502-507)
inline bool write_pcd_xyz(const std::string &path, const std::vector<double> &xyz) {
  std::ofstream f(path, std::ios::binary);
  if (!f.is_open()) return false;
  const size_t n = xyz.size() / 3;
  f << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n"
    << "WIDTH " << n << "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << n << "\nDATA binary\n";
  std::vector<float> buf(n * 3);
  for (size_t i = 0; i < n * 3; ++i) buf[i] = (float)xyz[i];
  f.write((const char *)buf.data(), (std::streamsize)(buf.size() * sizeof(float)));
  return (bool)f;
}

}  // namespace render
