// yaml_lite.hpp — the subset of YAML that MapEval's config files use (map_eval/config/*.yaml):
//   key: scalar            # comment
//   key: [a, b, c]         inline sequence
//   key:                   block sequence of inline sequences (initial_matrix)
//     - [1.0, 0.0, 0.0, 0.0]
// yaml-cpp (the reference's parser, map_eval_main.cpp:123) is not available in this environment; this parser keeps
// the loader's observable behaviour: as<T>() of a missing key or of a malformed scalar throws.
#pragma once
#include <cctype>
#include <cstdint>
#include <fstream>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace yaml_lite {

struct Node {
  enum Kind { Null, Scalar, Sequence } kind = Null;
  std::string scalar;
  std::vector<Node> seq;
  std::string key;   // for messages

  explicit operator bool() const { return kind != Null; }
  size_t size() const { return kind == Sequence ? seq.size() : 0; }
  const Node &operator[](size_t i) const {
    if (kind != Sequence) throw std::runtime_error("yaml: operator[] call on a scalar (key '" + key + "')");
    if (i >= seq.size()) throw std::runtime_error("yaml: index out of range (key '" + key + "')");
    return seq[i];
  }
  template <typename T> T as() const;
};

inline std::string trim(const std::string &s) {
  size_t b = 0, e = s.size();
  while (b < e && std::isspace((unsigned char)s[b])) ++b;
  while (e > b && std::isspace((unsigned char)s[e - 1])) --e;
  return s.substr(b, e - b);
}

inline std::string strip_comment(const std::string &line) {
  bool in_s = false, in_d = false;
  for (size_t i = 0; i < line.size(); ++i) {
    char c = line[i];
    if (c == '\'' && !in_d) in_s = !in_s;
    else if (c == '"' && !in_s) in_d = !in_d;
    else if (c == '#' && !in_s && !in_d && (i == 0 || std::isspace((unsigned char)line[i - 1]))) return line.substr(0, i);
  }
  return line;
}

inline std::string unquote(const std::string &s) {
  if (s.size() >= 2 && ((s.front() == '"' && s.back() == '"') || (s.front() == '\'' && s.back() == '\'')))
    return s.substr(1, s.size() - 2);
  return s;
}

inline Node parse_value(const std::string &text, const std::string &key);

inline Node parse_inline_seq(const std::string &text, const std::string &key) {
  Node n;
  n.kind = Node::Sequence;
  n.key = key;
  std::string inner = trim(text.substr(1, text.size() - 2));
  int depth = 0;
  std::string cur;
  for (char c : inner) {
    if (c == '[') ++depth;
    if (c == ']') --depth;
    if (c == ',' && depth == 0) { n.seq.push_back(parse_value(trim(cur), key)); cur.clear(); }
    else cur += c;
  }
  if (!trim(cur).empty()) n.seq.push_back(parse_value(trim(cur), key));
  return n;
}

inline Node parse_value(const std::string &text, const std::string &key) {
  Node n;
  n.key = key;
  if (text.empty() || text == "~" || text == "null") return n;
  if (text.front() == '[' && text.back() == ']') return parse_inline_seq(text, key);
  n.kind = Node::Scalar;
  n.scalar = unquote(text);
  return n;
}

template <> inline std::string Node::as<std::string>() const {
  if (kind != Scalar) throw std::runtime_error("yaml: bad conversion of key '" + key + "' to string");
  return scalar;
}
template <> inline double Node::as<double>() const {
  if (kind != Scalar) throw std::runtime_error("yaml: bad conversion of key '" + key + "' to double");
  size_t pos = 0;
  double v = 0;
  try { v = std::stod(scalar, &pos); } catch (...) { throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to double"); }
  if (pos != scalar.size()) throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to double");
  return v;
}
template <> inline int Node::as<int>() const {
  if (kind != Scalar) throw std::runtime_error("yaml: bad conversion of key '" + key + "' to int");
  size_t pos = 0;
  long v = 0;
  try { v = std::stol(scalar, &pos); } catch (...) { throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to int"); }
  if (pos != scalar.size()) throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to int");
  return (int)v;
}
template <> inline uint64_t Node::as<uint64_t>() const {
  if (kind != Scalar || scalar.empty() || scalar[0] == '-') throw std::runtime_error("yaml: bad conversion of key '" + key + "' to uint64");
  size_t pos = 0;
  unsigned long long v = 0;
  try { v = std::stoull(scalar, &pos); } catch (...) { throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to uint64"); }
  if (pos != scalar.size()) throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to uint64");
  return (uint64_t)v;
}
template <> inline bool Node::as<bool>() const {
  if (kind != Scalar) throw std::runtime_error("yaml: bad conversion of key '" + key + "' to bool");
  std::string s;
  for (char c : scalar) s += (char)std::tolower((unsigned char)c);
  if (s == "true" || s == "yes" || s == "on" || s == "y") return true;     // yaml-cpp's bool spellings
  if (s == "false" || s == "no" || s == "off" || s == "n") return false;
  throw std::runtime_error("yaml: bad conversion of key '" + key + "' ('" + scalar + "') to bool");
}

class Document {
 public:
  static Document LoadFile(const std::string &path) {
    std::ifstream in(path);
    if (!in.is_open()) throw std::runtime_error("yaml: bad file: " + path);
    std::stringstream ss;
    ss << in.rdbuf();
    return Load(ss.str());
  }
  static Document Load(const std::string &text) {
    Document d;
    std::istringstream in(text);
    std::string raw, open_key;
    while (std::getline(in, raw)) {
      std::string line = strip_comment(raw);
      if (trim(line).empty()) continue;
      const bool indented = std::isspace((unsigned char)line[0]);
      std::string t = trim(line);
      if (t[0] == '-' && (indented || !open_key.empty())) {           // block sequence item of the open key
        if (open_key.empty()) throw std::runtime_error("yaml: sequence item without a key: " + t);
        Node &n = d.map_[open_key];
        n.kind = Node::Sequence;
        n.key = open_key;
        n.seq.push_back(parse_value(trim(t.substr(1)), open_key));
        continue;
      }
      size_t colon = std::string::npos;
      bool in_s = false, in_d = false;
      for (size_t i = 0; i < t.size(); ++i) {
        if (t[i] == '\'' && !in_d) in_s = !in_s;
        else if (t[i] == '"' && !in_s) in_d = !in_d;
        else if (t[i] == ':' && !in_s && !in_d && (i + 1 == t.size() || std::isspace((unsigned char)t[i + 1]))) { colon = i; break; }
      }
      if (colon == std::string::npos) throw std::runtime_error("yaml: cannot parse line: " + t);
      std::string key = trim(t.substr(0, colon)), val = trim(t.substr(colon + 1));
      d.map_[key] = parse_value(val, key);
      open_key = val.empty() ? key : std::string();
    }
    return d;
  }
  // yaml-cpp semantics: a missing key yields a node that is false in boolean context and throws on as<T>()
  Node operator[](const std::string &key) const {
    auto it = map_.find(key);
    if (it != map_.end()) return it->second;
    Node n;
    n.key = key;
    return n;
  }

 private:
  std::map<std::string, Node> map_;
};

template <typename T> inline T Node::as() const { static_assert(sizeof(T) == 0, "unsupported as<T>"); return T(); }

}  // namespace yaml_lite
