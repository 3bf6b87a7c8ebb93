// cloud_io.hpp — minimal PCD / PLY point readers for the re-hosted map_eval driver.
//
// The reference loads its clouds with Open3D (io::ReadPointCloudFromPCD / FromPLY with
// ReadPointCloudOption("auto", remove_nan = true, remove_infinite = true, print_progress = true), map_eval.cpp:6-21),
// which is not available here.  Only the x/y/z fields are consumed by the metric path; points with a non-finite
// coordinate are dropped, as that option does.  Coordinates are widened to double — the type of Open3D's
// PointCloud::points_.  Normals (PCD normal_x / normal_y / normal_z, PLY nx / ny / nz) are read on request, as Open3D's
// PointCloud::normals_: point-to-plane ICP (registration_methods: 1) needs them on the ground-truth cloud, generalized ICP
// (2) uses those of either cloud.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace cloud_io {

struct Field { std::string name; int size = 4; char type = 'F'; int count = 1; int offset = 0; };

inline double read_scalar(const unsigned char *p, int size, char type) {
  switch (type) {
    case 'F': if (size == 4) { float v; std::memcpy(&v, p, 4); return v; } { double v; std::memcpy(&v, p, 8); return v; }
    case 'I': if (size == 1) { int8_t v; std::memcpy(&v, p, 1); return v; } if (size == 2) { int16_t v; std::memcpy(&v, p, 2); return v; }
              if (size == 4) { int32_t v; std::memcpy(&v, p, 4); return v; } { int64_t v; std::memcpy(&v, p, 8); return (double)v; }
    default:  if (size == 1) { uint8_t v; std::memcpy(&v, p, 1); return v; } if (size == 2) { uint16_t v; std::memcpy(&v, p, 2); return v; }
              if (size == 4) { uint32_t v; std::memcpy(&v, p, 4); return v; } { uint64_t v; std::memcpy(&v, p, 8); return (double)v; }
  }
}

// LZF decompression (PCD "binary_compressed"); returns false on malformed input
inline bool lzf_decompress(const unsigned char *in, size_t in_len, unsigned char *out, size_t out_len) {
  size_t ip = 0, op = 0;
  while (ip < in_len) {
    unsigned ctrl = in[ip++];
    if (ctrl < 32) {
      ctrl++;
      if (op + ctrl > out_len || ip + ctrl > in_len) return false;
      std::memcpy(out + op, in + ip, ctrl);
      op += ctrl; ip += ctrl;
    } else {
      unsigned len = ctrl >> 5;
      if (len == 7) { if (ip >= in_len) return false; len += in[ip++]; }
      if (ip >= in_len) return false;
      size_t ref_off = ((ctrl & 0x1f) << 8) + in[ip++] + 1;
      len += 2;
      if (ref_off > op || op + len > out_len) return false;
      size_t ref = op - ref_off;
      for (unsigned i = 0; i < len; ++i) out[op++] = out[ref++];
    }
  }
  return op == out_len;
}

inline bool push_if_finite(std::vector<double> &xyz, double x, double y, double z) {
  if (std::isfinite(x) && std::isfinite(y) && std::isfinite(z)) { xyz.push_back(x); xyz.push_back(y); xyz.push_back(z); return true; }
  return false;
}

// returns false if the file cannot be opened / parsed; xyz = N x 3 AoS
// normals (nullable): filled with N x 3 normals when the file carries them, left empty otherwise
inline bool read_pcd(const std::string &path, std::vector<double> &xyz, std::string *err = nullptr, std::vector<double> *normals = nullptr) {
  std::ifstream in(path, std::ios::binary);
  if (!in.is_open()) { if (err) *err = "cannot open " + path; return false; }
  std::vector<Field> fields;
  long long points = -1, width = 0, height = 1;
  std::string data_kind, line;
  while (std::getline(in, line)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    if (line.empty() || line[0] == '#') continue;
    std::istringstream ls(line);
    std::string tag;
    ls >> tag;
    if (tag == "FIELDS") { std::string f; while (ls >> f) { Field fd; fd.name = f; fields.push_back(fd); } }
    else if (tag == "SIZE") { for (auto &f : fields) ls >> f.size; }
    else if (tag == "TYPE") { for (auto &f : fields) ls >> f.type; }
    else if (tag == "COUNT") { for (auto &f : fields) ls >> f.count; }
    else if (tag == "WIDTH") ls >> width;
    else if (tag == "HEIGHT") ls >> height;
    else if (tag == "POINTS") ls >> points;
    else if (tag == "DATA") { ls >> data_kind; break; }
  }
  if (points < 0) points = width * height;
  int step = 0, ix = -1, iy = -1, iz = -1, nx = -1, ny = -1, nz = -1;
  for (size_t i = 0; i < fields.size(); ++i) {
    fields[i].offset = step;
    step += fields[i].size * fields[i].count;
    if (fields[i].name == "x") ix = (int)i;
    if (fields[i].name == "y") iy = (int)i;
    if (fields[i].name == "z") iz = (int)i;
    if (fields[i].name == "normal_x") nx = (int)i;
    if (fields[i].name == "normal_y") ny = (int)i;
    if (fields[i].name == "normal_z") nz = (int)i;
  }
  const bool want_n = normals && nx >= 0 && ny >= 0 && nz >= 0;
  if (normals) normals->clear();
  if (ix < 0 || iy < 0 || iz < 0 || data_kind.empty()) { if (err) *err = "PCD header without x/y/z fields or DATA line: " + path; return false; }
  xyz.clear();
  xyz.reserve((size_t)points * 3);
  if (data_kind == "ascii") {
    std::vector<double> vals;
    while (std::getline(in, line)) {
      std::istringstream ls(line);
      vals.clear();
      std::string tok;
      while (ls >> tok) { try { vals.push_back(std::stod(tok)); } catch (...) { vals.push_back(std::nan("")); } }
      if (vals.empty()) continue;
      // field index -> value index (COUNT may exceed 1 for non-xyz fields)
      auto value_of = [&](int f) { int k = 0; for (int i = 0; i < f; ++i) k += fields[i].count; return k < (int)vals.size() ? vals[k] : std::nan(""); };
      if (push_if_finite(xyz, value_of(ix), value_of(iy), value_of(iz)) && want_n) {
        normals->push_back(value_of(nx)); normals->push_back(value_of(ny)); normals->push_back(value_of(nz));
      }
    }
  } else if (data_kind == "binary") {
    std::vector<unsigned char> buf((size_t)points * step);
    in.read((char *)buf.data(), (std::streamsize)buf.size());
    if ((size_t)in.gcount() != buf.size()) { if (err) *err = "truncated binary PCD: " + path; return false; }
    for (long long i = 0; i < points; ++i) {
      const unsigned char *p = buf.data() + (size_t)i * step;
      auto at = [&](int f) { return read_scalar(p + fields[f].offset, fields[f].size, fields[f].type); };
      if (push_if_finite(xyz, at(ix), at(iy), at(iz)) && want_n) { normals->push_back(at(nx)); normals->push_back(at(ny)); normals->push_back(at(nz)); }
    }
  } else if (data_kind == "binary_compressed") {
    uint32_t comp = 0, uncomp = 0;
    in.read((char *)&comp, 4);
    in.read((char *)&uncomp, 4);
    std::vector<unsigned char> cbuf(comp), buf(uncomp);
    in.read((char *)cbuf.data(), comp);
    if ((size_t)in.gcount() != comp || uncomp != (uint64_t)points * step || !lzf_decompress(cbuf.data(), comp, buf.data(), uncomp)) {
      if (err) *err = "malformed binary_compressed PCD: " + path;
      return false;
    }
    // struct-of-arrays: all values of field 0, then field 1, ...
    std::vector<size_t> base(fields.size());
    size_t off = 0;
    for (size_t f = 0; f < fields.size(); ++f) { base[f] = off; off += (size_t)fields[f].size * fields[f].count * points; }
    for (long long i = 0; i < points; ++i) {
      auto at = [&](int f) { return read_scalar(buf.data() + base[f] + (size_t)i * fields[f].size * fields[f].count, fields[f].size, fields[f].type); };
      if (push_if_finite(xyz, at(ix), at(iy), at(iz)) && want_n) { normals->push_back(at(nx)); normals->push_back(at(ny)); normals->push_back(at(nz)); }
    }
  } else {
    if (err) *err = "unsupported PCD DATA kind '" + data_kind + "': " + path;
    return false;
  }
  return true;
}

inline bool read_ply(const std::string &path, std::vector<double> &xyz, std::string *err = nullptr, std::vector<double> *normals = nullptr) {
  std::ifstream in(path, std::ios::binary);
  if (!in.is_open()) { if (err) *err = "cannot open " + path; return false; }
  std::string line, format;
  long long nvert = -1;
  bool in_vertex = false, vertex_first = true, seen_element = false;
  struct Prop { std::string type, name; };
  std::vector<Prop> props;
  std::getline(in, line);
  if (line.rfind("ply", 0) != 0) { if (err) *err = "not a PLY file: " + path; return false; }
  while (std::getline(in, line)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    std::istringstream ls(line);
    std::string tag;
    ls >> tag;
    if (tag == "format") ls >> format;
    else if (tag == "element") {
      std::string name; long long n;
      ls >> name >> n;
      in_vertex = (name == "vertex");
      if (in_vertex) { nvert = n; vertex_first = !seen_element; }
      seen_element = true;
    } else if (tag == "property" && in_vertex) {
      Prop p; ls >> p.type;
      if (p.type == "list") { if (err) *err = "PLY list property on vertices is not supported: " + path; return false; }
      ls >> p.name;
      props.push_back(p);
    } else if (tag == "end_header") break;
  }
  if (nvert < 0 || !vertex_first) { if (err) *err = "PLY without a leading vertex element: " + path; return false; }
  auto size_of = [](const std::string &t) {
    if (t == "char" || t == "uchar" || t == "int8" || t == "uint8") return 1;
    if (t == "short" || t == "ushort" || t == "int16" || t == "uint16") return 2;
    if (t == "double" || t == "float64") return 8;
    return 4;
  };
  auto kind_of = [](const std::string &t) { return (t == "float" || t == "double" || t == "float32" || t == "float64") ? 'F' : (t[0] == 'u' ? 'U' : 'I'); };
  int step = 0, ox = -1, oy = -1, oz = -1, px = -1, py = -1, pz = -1, on[3] = {-1, -1, -1}, pn[3] = {-1, -1, -1};
  for (size_t i = 0; i < props.size(); ++i) {
    if (props[i].name == "x") { ox = step; px = (int)i; }
    if (props[i].name == "y") { oy = step; py = (int)i; }
    if (props[i].name == "z") { oz = step; pz = (int)i; }
    if (props[i].name == "nx") { on[0] = step; pn[0] = (int)i; }
    if (props[i].name == "ny") { on[1] = step; pn[1] = (int)i; }
    if (props[i].name == "nz") { on[2] = step; pn[2] = (int)i; }
    step += size_of(props[i].type);
  }
  const bool want_n = normals && pn[0] >= 0 && pn[1] >= 0 && pn[2] >= 0;
  if (normals) normals->clear();
  if (px < 0 || py < 0 || pz < 0) { if (err) *err = "PLY vertex element without x/y/z: " + path; return false; }
  xyz.clear();
  xyz.reserve((size_t)nvert * 3);
  if (format == "ascii") {
    for (long long i = 0; i < nvert && std::getline(in, line); ++i) {
      std::istringstream ls(line);
      std::vector<double> v(props.size(), std::nan(""));
      std::string tok;
      for (size_t k = 0; k < props.size() && (ls >> tok); ++k) {   // stod understands nan / inf, operator>> does not
        try { v[k] = std::stod(tok); } catch (...) { v[k] = std::nan(""); }
      }
      if (push_if_finite(xyz, v[px], v[py], v[pz]) && want_n) for (int a = 0; a < 3; ++a) normals->push_back(v[pn[a]]);
    }
  } else if (format == "binary_little_endian") {
    std::vector<unsigned char> buf((size_t)nvert * step);
    in.read((char *)buf.data(), (std::streamsize)buf.size());
    if ((size_t)in.gcount() != buf.size()) { if (err) *err = "truncated binary PLY: " + path; return false; }
    for (long long i = 0; i < nvert; ++i) {
      const unsigned char *p = buf.data() + (size_t)i * step;
      if (push_if_finite(xyz, read_scalar(p + ox, size_of(props[px].type), kind_of(props[px].type)),
                         read_scalar(p + oy, size_of(props[py].type), kind_of(props[py].type)),
                         read_scalar(p + oz, size_of(props[pz].type), kind_of(props[pz].type))) && want_n)
        for (int a = 0; a < 3; ++a) normals->push_back(read_scalar(p + on[a], size_of(props[pn[a]].type), kind_of(props[pn[a]].type)));
    }
  } else {
    if (err) *err = "unsupported PLY format '" + format + "': " + path;
    return false;
  }
  return true;
}

}  // namespace cloud_io
