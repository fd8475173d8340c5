// Forced splits (forcedsplits_filename): the JSON plan file and its flattening into the device table of kernels.cuh ForcedNode.
//
// [UPSTREAM] SerialTreeLearner::ForceSplits reads the file with json11.  It holds one object
//   {"feature": <real feature index>, "threshold": <number>, "left": {...}, "right": {...}}
// nested through "left" and "right"; a child is part of the plan only when it has both "feature" and "threshold", and every other key
// is ignored.  The nodes are applied in breadth-first order from the root, one per split, so node j is the tree's split j while the
// forced phase lasts: it splits the leaf its parent left it (the root's is leaf 0, a left child keeps its parent's leaf, the right child
// of node j gets the new leaf j + 1).  The threshold is mapped to a bin as Dataset::BinThreshold does: the value's bin for a numerical
// feature, the category's bin for a categorical one (0 when the category has no bin of its own, which the device treats as invalid).
//
// Deviations: upstream ignores a file it cannot read or parse and trains without a plan; here that fails, as do a feature that is not an
// integer in [0, F), a feature the dataset does not use (upstream would index inner feature -1) and a threshold that is not a number.
// Part of engine.cu's translation unit.
#pragma once
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <deque>
#include <fstream>
#include <sstream>
#include <system_error>
#include <string>
#include <utility>
#include <vector>

namespace b200gbm {

// A JSON value (RFC 8259), enough to read a plan: objects keep their keys in file order, and a repeated key's last value wins.
struct JsonValue {
  enum Kind { kNull, kBool, kNumber, kString, kArray, kObject } kind = kNull;
  double number = 0.0;
  bool boolean = false;
  std::string str;
  std::vector<JsonValue> items;
  std::vector<std::pair<std::string, JsonValue>> members;
  const JsonValue* Get(const std::string& key) const {
    const JsonValue* v = nullptr;
    for (const auto& m : members) if (m.first == key) v = &m.second;
    return v;
  }
};

// Recursive-descent reader; throws std::runtime_error with the byte offset of the first error.
class JsonReader {
 public:
  static JsonValue Parse(const std::string& text) {
    JsonReader r(text);
    JsonValue v = r.Value(0);
    r.Space();
    if (r.i_ != text.size()) r.Fail("unexpected text after the value");
    return v;
  }

 private:
  static constexpr int kMaxDepth = 512;
  explicit JsonReader(const std::string& t) : t_(t) {}
  [[noreturn]] void Fail(const std::string& what) const { throw std::runtime_error(what + " at byte " + std::to_string(i_)); }
  void Space() { while (i_ < t_.size() && (t_[i_] == ' ' || t_[i_] == '\t' || t_[i_] == '\n' || t_[i_] == '\r')) ++i_; }
  bool Eat(char c) { Space(); if (i_ < t_.size() && t_[i_] == c) { ++i_; return true; } return false; }
  void Expect(char c) { if (!Eat(c)) Fail(std::string("expected '") + c + "'"); }
  JsonValue Value(int depth) {
    if (depth > kMaxDepth) Fail("nesting deeper than " + std::to_string(kMaxDepth));
    Space();
    if (i_ >= t_.size()) Fail("unexpected end of input");
    JsonValue v;
    const char c = t_[i_];
    if (c == '{') {
      ++i_; v.kind = JsonValue::kObject;
      if (Eat('}')) return v;
      do {
        Space();
        if (i_ >= t_.size() || t_[i_] != '"') Fail("expected a string key");
        std::string key = String();
        Expect(':');
        v.members.emplace_back(std::move(key), Value(depth + 1));
      } while (Eat(','));
      Expect('}');
    } else if (c == '[') {
      ++i_; v.kind = JsonValue::kArray;
      if (Eat(']')) return v;
      do v.items.push_back(Value(depth + 1)); while (Eat(','));
      Expect(']');
    } else if (c == '"') {
      v.kind = JsonValue::kString; v.str = String();
    } else if (Word("true")) { v.kind = JsonValue::kBool; v.boolean = true; }
    else if (Word("false")) { v.kind = JsonValue::kBool; }
    else if (Word("null")) { v.kind = JsonValue::kNull; }
    else { v.kind = JsonValue::kNumber; v.number = Number(); }
    return v;
  }
  bool Word(const char* w) {
    const size_t n = std::char_traits<char>::length(w);
    if (t_.compare(i_, n, w) != 0) return false;
    i_ += n;
    return true;
  }
  static bool Digit(char c) { return c >= '0' && c <= '9'; }
  double Number() {      // -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?
    const size_t b = i_;
    if (i_ < t_.size() && t_[i_] == '-') ++i_;
    if (i_ >= t_.size() || !Digit(t_[i_])) Fail("invalid value");
    if (t_[i_] == '0') ++i_; else while (i_ < t_.size() && Digit(t_[i_])) ++i_;
    if (i_ < t_.size() && t_[i_] == '.') {
      ++i_;
      if (i_ >= t_.size() || !Digit(t_[i_])) Fail("invalid number");
      while (i_ < t_.size() && Digit(t_[i_])) ++i_;
    }
    if (i_ < t_.size() && (t_[i_] == 'e' || t_[i_] == 'E')) {
      ++i_;
      if (i_ < t_.size() && (t_[i_] == '+' || t_[i_] == '-')) ++i_;
      if (i_ >= t_.size() || !Digit(t_[i_])) Fail("invalid number");
      while (i_ < t_.size() && Digit(t_[i_])) ++i_;
    }
    double v = 0.0;      // from_chars: the same in every locale (strtod would read "30.5" as 30 under a comma decimal separator)
    const std::from_chars_result r = std::from_chars(t_.data() + b, t_.data() + i_, v);
    if (r.ec == std::errc::result_out_of_range) Fail("number out of range");
    if (r.ec != std::errc() || r.ptr != t_.data() + i_) Fail("invalid number");
    return v;
  }
  static void Utf8(unsigned cp, std::string* out) {
    if (cp < 0x80) { out->push_back(static_cast<char>(cp)); }
    else if (cp < 0x800) { out->push_back(static_cast<char>(0xC0 | (cp >> 6))); out->push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) {
      out->push_back(static_cast<char>(0xE0 | (cp >> 12))); out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F)));
      out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
    } else {
      out->push_back(static_cast<char>(0xF0 | (cp >> 18))); out->push_back(static_cast<char>(0x80 | ((cp >> 12) & 0x3F)));
      out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F))); out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
    }
  }
  unsigned Hex4() {
    if (i_ + 4 > t_.size()) Fail("invalid \\u escape");
    unsigned v = 0;
    for (int k = 0; k < 4; ++k) {
      const char c = t_[i_++];
      v <<= 4;
      if (Digit(c)) v |= static_cast<unsigned>(c - '0');
      else if (c >= 'a' && c <= 'f') v |= static_cast<unsigned>(c - 'a' + 10);
      else if (c >= 'A' && c <= 'F') v |= static_cast<unsigned>(c - 'A' + 10);
      else Fail("invalid \\u escape");
    }
    return v;
  }
  std::string String() {
    ++i_;      // the opening quote
    std::string out;
    for (;;) {
      if (i_ >= t_.size()) Fail("unterminated string");
      const char c = t_[i_++];
      if (c == '"') return out;
      if (static_cast<unsigned char>(c) < 0x20) Fail("control character in a string");
      if (c != '\\') { out.push_back(c); continue; }
      if (i_ >= t_.size()) Fail("unterminated string");
      const char e = t_[i_++];
      switch (e) {
        case '"': case '\\': case '/': out.push_back(e); break;
        case 'b': out.push_back('\b'); break;
        case 'f': out.push_back('\f'); break;
        case 'n': out.push_back('\n'); break;
        case 'r': out.push_back('\r'); break;
        case 't': out.push_back('\t'); break;
        case 'u': {
          unsigned cp = Hex4();
          if (cp >= 0xD800 && cp < 0xDC00 && i_ + 1 < t_.size() && t_[i_] == '\\' && t_[i_ + 1] == 'u') {
            const size_t back = i_;
            i_ += 2;
            const unsigned lo = Hex4();
            if (lo >= 0xDC00 && lo < 0xE000) cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            else i_ = back;
          }
          Utf8(cp, &out);
          break;
        }
        default: Fail("invalid escape");
      }
    }
  }
  const std::string& t_;
  size_t i_ = 0;
};

// The plan of `root` over `train`'s features, breadth-first (see the top of this file).  Throws std::runtime_error on a node of the plan
// whose feature is not an integer in [0, F) or is not used by the dataset, or whose threshold is not a number.
inline std::vector<ForcedNode> FlattenForcedPlan(const JsonValue& root, const Dataset& train) {
  auto in_plan = [](const JsonValue* v) { return v && v->kind == JsonValue::kObject && v->Get("feature") && v->Get("threshold"); };
  if (!in_plan(&root)) throw std::runtime_error("the root must be an object with \"feature\" and \"threshold\"");
  struct Item { const JsonValue* v; int parent, side, leaf; };
  std::vector<ForcedNode> plan;
  std::deque<Item> q{{&root, -1, 0, 0}};
  while (!q.empty()) {
    const Item it = q.front();
    q.pop_front();
    const int j = static_cast<int>(plan.size());
    const JsonValue& f = *it.v->Get("feature");
    const JsonValue& t = *it.v->Get("threshold");
    const std::string where = "node " + std::to_string(j) + " (breadth-first)";
    if (f.kind != JsonValue::kNumber || f.number != std::floor(f.number))
      throw std::runtime_error(where + ": \"feature\" should be an integer feature index");
    if (!(f.number >= 0 && f.number < train.num_total_features))
      throw std::runtime_error(where + ": feature " + Config::Num(f.number) + " is outside [0, " + std::to_string(train.num_total_features) + ")");
    const int real = static_cast<int>(f.number);
    if (train.inner_of[real] < 0)
      throw std::runtime_error(where + ": feature " + std::to_string(real) + " is not used by the dataset (it has a single bin, or was filtered out)");
    if (t.kind != JsonValue::kNumber) throw std::runtime_error(where + ": \"threshold\" should be a number");
    const FeatureBins& fb = train.mappers[real];
    ForcedNode n{train.inner_of[real], static_cast<int>(fb.ValueToBin(t.number)), fb.categorical ? 1 : 0, it.leaf, -1, -1};
    if (it.parent >= 0) (it.side ? plan[it.parent].right : plan[it.parent].left) = j;
    plan.push_back(n);
    const JsonValue* l = it.v->Get("left");
    const JsonValue* r = it.v->Get("right");
    if (in_plan(l)) q.push_back({l, j, 0, it.leaf});
    if (in_plan(r)) q.push_back({r, j, 1, j + 1});
  }
  return plan;
}

// the plan in forcedsplits_filename, read and flattened; empty when the value is empty
inline std::vector<ForcedNode> LoadForcedPlan(const std::string& path, const Dataset& train) {
  if (path.empty()) return {};
  std::ifstream in(path, std::ios::binary);
  if (!in) throw std::runtime_error("cannot read the file");
  std::stringstream ss;
  ss << in.rdbuf();
  if (in.bad()) throw std::runtime_error("cannot read the file");
  return FlattenForcedPlan(JsonReader::Parse(ss.str()), train);
}

// FNV-1a over the flattened plan, cut to 52 bits so that it travels exactly in a double; the ranks all-reduce it to agree on one plan
inline double ForcedPlanDigest(const std::vector<ForcedNode>& plan) {
  uint64_t h = 1469598103934665603ull;
  const unsigned char* p = reinterpret_cast<const unsigned char*>(plan.data());
  for (size_t i = 0; i < plan.size() * sizeof(ForcedNode); ++i) { h ^= p[i]; h *= 1099511628211ull; }
  h ^= plan.size(); h *= 1099511628211ull;
  return static_cast<double>(h >> 12);
}

}  // namespace b200gbm
