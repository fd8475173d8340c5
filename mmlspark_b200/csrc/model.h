// Host-side booster model: tree container, LightGBM model-text v3 writer/reader, row predictor.
//
// Replaces [UPSTREAM lightgbmlib 3.2.110] Tree / GBDT::SaveModelToString / LoadModelFromString and the
// single-row predictor behind LGBM_BoosterPredictForMatSingle.  Reference call sites:
//   saveToString            lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/booster/LightGBMBooster.scala:269-274
//   BoosterHandler(model)   .../booster/LightGBMBooster.scala:41-48
//   score/predictLeaf/SHAP  .../booster/LightGBMBooster.scala:390-423,510-545
// Format: SURVEY.md Appendix B.3.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "bin_mapper.h"

namespace b200gbm {

struct HostTree {
  int num_leaves = 1;
  int num_cat = 0;
  double shrinkage = 1.0;
  std::vector<int> left_child, right_child, split_feature, leaf_count, internal_count, leaf_depth;
  std::vector<int> split_feature_inner;
  std::vector<uint32_t> threshold_in_bin;
  std::vector<double> threshold, leaf_value, leaf_weight, internal_value, internal_weight;
  std::vector<float> split_gain;
  std::vector<int8_t> decision_type;
  // categorical splits ([UPSTREAM] Tree::cat_boundaries_ / cat_threshold_): node's threshold = index i, its bitset over
  // CATEGORY VALUES is cat_threshold[cat_boundaries[i] .. cat_boundaries[i+1])
  std::vector<int> cat_boundaries{0};
  std::vector<uint32_t> cat_threshold;

  static bool InBitset(const uint32_t* bits, int n, int pos) {
    const int w = pos / 32;
    if (pos < 0 || w >= n) return false;
    return (bits[w] >> (pos % 32)) & 1u;
  }
  void AddCategoricalNode(int node, const std::vector<int>& categories) {
    std::vector<uint32_t> bits;
    for (int c : categories) {
      const size_t w = static_cast<size_t>(c) / 32;
      if (bits.size() < w + 1) bits.resize(w + 1, 0u);
      bits[w] |= 1u << (c % 32);
    }
    threshold[node] = num_cat;
    threshold_in_bin[node] = static_cast<uint32_t>(num_cat);
    ++num_cat;
    cat_boundaries.push_back(cat_boundaries.back() + static_cast<int>(bits.size()));
    cat_threshold.insert(cat_threshold.end(), bits.begin(), bits.end());
  }

  void Resize(int nl) {
    num_leaves = nl;
    int ni = std::max(nl - 1, 0);
    left_child.resize(ni); right_child.resize(ni); split_feature.resize(ni); split_feature_inner.resize(ni);
    threshold_in_bin.resize(ni); threshold.resize(ni); split_gain.resize(ni); decision_type.resize(ni);
    internal_value.resize(ni); internal_weight.resize(ni); internal_count.resize(ni);
    leaf_value.resize(nl); leaf_weight.resize(nl); leaf_count.resize(nl); leaf_depth.resize(nl);
  }
  static double RoundTiny(double x) { return std::fabs(x) > kZeroThr ? x : 0.0; }
  void Shrink(double rate) {
    for (int i = 0; i < num_leaves; ++i) leaf_value[i] = RoundTiny(leaf_value[i] * rate);
    for (int i = 0; i < num_leaves - 1; ++i) internal_value[i] = RoundTiny(internal_value[i] * rate);
    shrinkage *= rate;
  }
  void AddBias(double v) {
    for (int i = 0; i < num_leaves; ++i) leaf_value[i] = RoundTiny(leaf_value[i] + v);
    for (int i = 0; i < num_leaves - 1; ++i) internal_value[i] = RoundTiny(internal_value[i] + v);
    shrinkage = 1.0;
  }
  void MakeConstant(double v) { Resize(1); leaf_value[0] = v; shrinkage = 1.0; }

  inline int Decide(double fval, int node) const {
    int mt = (decision_type[node] >> 2) & 3;
    if (decision_type[node] & 1) {       // [UPSTREAM] Tree::CategoricalDecision
      // NaN goes right whatever the missing type: upstream converts it to int first, which on x86 gives INT_MIN (< 0 => right), so
      // its "NaN -> category 0" branch never runs.  Binning agrees: NaN falls in bin 0, which no left set holds.
      if (std::isnan(fval)) return right_child[node];
      const int iv = static_cast<int>(fval);
      if (iv < 0) return right_child[node];
      const int ci = static_cast<int>(threshold[node]);
      return InBitset(cat_threshold.data() + cat_boundaries[ci], cat_boundaries[ci + 1] - cat_boundaries[ci], iv) ? left_child[node] : right_child[node];
    }
    if (std::isnan(fval) && mt != MISSING_NAN) fval = 0.0;
    if ((mt == MISSING_ZERO && std::fabs(fval) <= kZeroThr) || (mt == MISSING_NAN && std::isnan(fval)))
      return (decision_type[node] & 2) ? left_child[node] : right_child[node];
    return fval <= threshold[node] ? left_child[node] : right_child[node];
  }
  int LeafIndex(const double* row) const {
    if (num_leaves <= 1) return 0;
    int node = 0;
    while (node >= 0) node = Decide(row[split_feature[node]], node);
    return ~node;
  }
  double Predict(const double* row) const { return leaf_value[LeafIndex(row)]; }

  // ---- TreeSHAP (Lundberg et al.), the algorithm behind C_API_PREDICT_CONTRIB
  struct PathElem { int feature_index; double zero_fraction, one_fraction, pweight; };
  double NodeCount(int node) const { return node >= 0 ? internal_count[node] : leaf_count[~node]; }
  static void ExtendPath(PathElem* p, int depth, double zf, double of, int fi) {
    p[depth] = {fi, zf, of, depth == 0 ? 1.0 : 0.0};
    for (int i = depth - 1; i >= 0; --i) {
      p[i + 1].pweight += of * p[i].pweight * (i + 1) / static_cast<double>(depth + 1);
      p[i].pweight = zf * p[i].pweight * (depth - i) / static_cast<double>(depth + 1);
    }
  }
  static void UnwindPath(PathElem* p, int depth, int pi) {
    const double of = p[pi].one_fraction, zf = p[pi].zero_fraction;
    double next = p[depth].pweight;
    for (int i = depth - 1; i >= 0; --i) {
      if (of != 0) {
        double tmp = p[i].pweight;
        p[i].pweight = next * (depth + 1) / static_cast<double>((i + 1) * of);
        next = tmp - p[i].pweight * zf * (depth - i) / static_cast<double>(depth + 1);
      } else {
        p[i].pweight = (p[i].pweight * (depth + 1)) / static_cast<double>(zf * (depth - i));
      }
    }
    for (int i = pi; i < depth; ++i) { p[i].feature_index = p[i + 1].feature_index; p[i].zero_fraction = p[i + 1].zero_fraction; p[i].one_fraction = p[i + 1].one_fraction; }
  }
  static double UnwoundSum(const PathElem* p, int depth, int pi) {
    const double of = p[pi].one_fraction, zf = p[pi].zero_fraction;
    double next = p[depth].pweight, total = 0;
    for (int i = depth - 1; i >= 0; --i) {
      if (of != 0) {
        double tmp = next * (depth + 1) / static_cast<double>((i + 1) * of);
        total += tmp;
        next = p[i].pweight - tmp * zf * ((depth - i) / static_cast<double>(depth + 1));
      } else {
        total += (p[i].pweight / zf) / ((depth - i) / static_cast<double>(depth + 1));
      }
    }
    return total;
  }
  void ShapRecurse(const double* row, double* phi, int node, int depth, PathElem* parent_path, double pzf, double pof, int pfi) const {
    PathElem* path = parent_path + depth;
    if (depth > 0) std::memcpy(path, parent_path, sizeof(PathElem) * depth);
    ExtendPath(path, depth, pzf, pof, pfi);
    if (node < 0) {
      for (int i = 1; i <= depth; ++i) {
        double w = UnwoundSum(path, depth, i);
        phi[path[i].feature_index] += w * (path[i].one_fraction - path[i].zero_fraction) * leaf_value[~node];
      }
      return;
    }
    int hot = Decide(row[split_feature[node]], node);
    int cold = hot == left_child[node] ? right_child[node] : left_child[node];
    double w = NodeCount(node);
    double hot_zf = NodeCount(hot) / w, cold_zf = NodeCount(cold) / w;
    double inc_zf = 1, inc_of = 1;
    int pi = 0;
    for (; pi <= depth; ++pi) if (path[pi].feature_index == split_feature[node]) break;
    if (pi != depth + 1) {
      inc_zf = path[pi].zero_fraction; inc_of = path[pi].one_fraction;
      UnwindPath(path, depth, pi);
      depth -= 1;
    }
    ShapRecurse(row, phi, hot, depth + 1, path, hot_zf * inc_zf, inc_of, split_feature[node]);
    ShapRecurse(row, phi, cold, depth + 1, path, cold_zf * inc_zf, 0, split_feature[node]);
  }
  double ExpectedValue() const {
    if (num_leaves == 1) return leaf_value[0];
    double total = internal_count[0], e = 0;
    for (int i = 0; i < num_leaves; ++i) e += (leaf_count[i] / total) * leaf_value[i];
    return e;
  }
  int MaxDepth() const { int d = 0; for (int i = 0; i < num_leaves; ++i) d = std::max(d, leaf_depth[i]); return d; }
  // phi has num_features+1 entries (last = expected value)
  void AddContrib(const double* row, int num_features, double* phi) const {
    phi[num_features] += ExpectedValue();
    if (num_leaves <= 1) return;
    int md = MaxDepth() + 2;
    std::vector<PathElem> buf(static_cast<size_t>(md) * (md + 1) / 2 + md);
    ShapRecurse(row, phi, 0, 0, buf.data(), 1, 1, -1);
  }

  template <typename T>
  static std::string Join(const std::vector<T>& v, int n, const char* fmt) {
    std::string s;
    char buf[64];
    for (int i = 0; i < n; ++i) {
      if (i) s += ' ';
      if (std::is_floating_point<T>::value) snprintf(buf, sizeof(buf), fmt, static_cast<double>(v[i]));
      else snprintf(buf, sizeof(buf), fmt, static_cast<long long>(v[i]));
      s += buf;
    }
    return s;
  }
  std::string ToString() const {
    std::ostringstream s;
    const int nl = num_leaves;
    s << "num_leaves=" << nl << '\n' << "num_cat=" << num_cat << '\n';
    s << "split_feature=" << Join(split_feature, nl - 1, "%lld") << '\n';
    s << "split_gain=" << Join(split_gain, nl - 1, "%g") << '\n';
    s << "threshold=" << Join(threshold, nl - 1, "%.17g") << '\n';
    s << "decision_type=" << Join(decision_type, nl - 1, "%lld") << '\n';
    s << "left_child=" << Join(left_child, nl - 1, "%lld") << '\n';
    s << "right_child=" << Join(right_child, nl - 1, "%lld") << '\n';
    s << "leaf_value=" << Join(leaf_value, nl, "%.17g") << '\n';
    s << "leaf_weight=" << Join(leaf_weight, nl, "%.17g") << '\n';
    s << "leaf_count=" << Join(leaf_count, nl, "%lld") << '\n';
    s << "internal_value=" << Join(internal_value, nl - 1, "%g") << '\n';
    s << "internal_weight=" << Join(internal_weight, nl - 1, "%g") << '\n';
    s << "internal_count=" << Join(internal_count, nl - 1, "%lld") << '\n';
    if (num_cat > 0) {
      s << "cat_boundaries=" << Join(cat_boundaries, num_cat + 1, "%lld") << '\n';
      s << "cat_threshold=" << Join(cat_threshold, static_cast<int>(cat_threshold.size()), "%lld") << '\n';
    }
    s << "is_linear=0\n";
    char buf[64];
    snprintf(buf, sizeof(buf), "%g", shrinkage);
    s << "shrinkage=" << buf << "\n\n";
    return s.str();
  }
  static HostTree FromKV(const std::map<std::string, std::string>& kv) {
    HostTree t;
    auto need = [&](const char* k) -> const std::string& {
      auto it = kv.find(k);
      if (it == kv.end()) throw std::runtime_error(std::string("Tree model string format error, should contain ") + k + " field");
      return it->second;
    };
    int nl = std::atoi(need("num_leaves").c_str());
    t.Resize(nl);
    auto it = kv.find("num_cat");
    t.num_cat = it == kv.end() ? 0 : std::atoi(it->second.c_str());
    auto fill_d = [&](const char* k, std::vector<double>& v, int n, bool req) {
      auto f = kv.find(k);
      if (f == kv.end()) { if (req && n > 0) need(k); return; }
      std::istringstream is(f->second);
      for (int i = 0; i < n; ++i) { std::string x; is >> x; v[i] = std::strtod(x.c_str(), nullptr); }
    };
    auto fill_i = [&](const char* k, auto& v, int n, bool req) {
      auto f = kv.find(k);
      if (f == kv.end()) { if (req && n > 0) need(k); return; }
      std::istringstream is(f->second);
      for (int i = 0; i < n; ++i) { long long x = 0; is >> x; v[i] = static_cast<typename std::decay<decltype(v[0])>::type>(x); }
    };
    fill_d("leaf_value", t.leaf_value, nl, true);
    if (nl > 1) {
      fill_i("split_feature", t.split_feature, nl - 1, true);
      std::vector<double> g(nl - 1, 0.0);
      fill_d("split_gain", g, nl - 1, false);
      for (int i = 0; i < nl - 1; ++i) t.split_gain[i] = static_cast<float>(g[i]);
      fill_d("threshold", t.threshold, nl - 1, true);
      fill_i("decision_type", t.decision_type, nl - 1, false);
      fill_i("left_child", t.left_child, nl - 1, true);
      fill_i("right_child", t.right_child, nl - 1, true);
      fill_d("leaf_weight", t.leaf_weight, nl, false);
      fill_i("leaf_count", t.leaf_count, nl, false);
      fill_d("internal_value", t.internal_value, nl - 1, false);
      fill_d("internal_weight", t.internal_weight, nl - 1, false);
      fill_i("internal_count", t.internal_count, nl - 1, false);
      t.split_feature_inner = t.split_feature;
      if (t.num_cat > 0) {
        t.cat_boundaries.assign(t.num_cat + 1, 0);
        fill_i("cat_boundaries", t.cat_boundaries, t.num_cat + 1, true);
        t.cat_threshold.assign(t.cat_boundaries.back(), 0u);
        fill_i("cat_threshold", t.cat_threshold, t.cat_boundaries.back(), true);
      }
      // recompute leaf depths
      std::vector<std::pair<int, int>> st{{0, 0}};
      while (!st.empty()) {
        auto [node, d] = st.back(); st.pop_back();
        for (int c : {t.left_child[node], t.right_child[node]}) {
          if (c < 0) t.leaf_depth[~c] = d + 1; else st.push_back({c, d + 1});
        }
      }
    }
    it = kv.find("shrinkage");
    t.shrinkage = it == kv.end() ? 1.0 : std::atof(it->second.c_str());
    return t;
  }
};

struct HostModel {
  int num_class = 1;
  int num_tree_per_iteration = 1;
  int label_index = 0;
  int max_feature_idx = 0;
  std::string objective_str;                 // e.g. "binary sigmoid:1"
  bool average_output = false;
  std::vector<std::string> feature_names;
  std::vector<std::string> feature_infos;
  std::vector<int> monotone_constraints;     // the header's monotone_constraints= line, only when non-empty ([UPSTREAM] GBDT::SaveModelToString)
  std::vector<std::unique_ptr<HostTree>> trees;
  std::string loaded_parameters;

  int NumIterations() const { return num_tree_per_iteration ? static_cast<int>(trees.size()) / num_tree_per_iteration : 0; }

  std::vector<double> FeatureImportance(int num_iteration, int type) const {
    int used = static_cast<int>(trees.size());
    if (num_iteration > 0) used = std::min(used, num_iteration * num_tree_per_iteration);
    std::vector<double> imp(max_feature_idx + 1, 0.0);
    for (int t = 0; t < used; ++t)
      for (int i = 0; i < trees[t]->num_leaves - 1; ++i)
        if (trees[t]->split_gain[i] > 0) imp[trees[t]->split_feature[i]] += type == 0 ? 1.0 : trees[t]->split_gain[i];
    return imp;
  }

  std::string ToString(int start_iteration, int num_iteration, int importance_type, const std::string& params_block) const {
    std::ostringstream ss;
    ss << "tree\nversion=v3\n";
    ss << "num_class=" << num_class << '\n' << "num_tree_per_iteration=" << num_tree_per_iteration << '\n';
    ss << "label_index=" << label_index << '\n' << "max_feature_idx=" << max_feature_idx << '\n';
    if (!objective_str.empty()) ss << "objective=" << objective_str << '\n';
    if (average_output) ss << "average_output\n";
    ss << "feature_names=";
    for (size_t i = 0; i < feature_names.size(); ++i) ss << (i ? " " : "") << feature_names[i];
    if (!monotone_constraints.empty()) {
      ss << "\nmonotone_constraints=";
      for (size_t i = 0; i < monotone_constraints.size(); ++i) ss << (i ? " " : "") << monotone_constraints[i];
    }
    ss << "\nfeature_infos=";
    for (size_t i = 0; i < feature_infos.size(); ++i) ss << (i ? " " : "") << feature_infos[i];
    ss << '\n';
    int used = static_cast<int>(trees.size());
    int total_iter = num_tree_per_iteration ? used / num_tree_per_iteration : 0;
    start_iteration = std::min(std::max(start_iteration, 0), total_iter);
    if (num_iteration > 0) used = std::min((start_iteration + num_iteration) * num_tree_per_iteration, used);
    int start_model = start_iteration * num_tree_per_iteration;
    std::vector<std::string> strs;
    for (int i = start_model; i < used; ++i) strs.push_back("Tree=" + std::to_string(i - start_model) + "\n" + trees[i]->ToString() + "\n");
    ss << "tree_sizes=";
    for (size_t i = 0; i < strs.size(); ++i) ss << (i ? " " : "") << strs[i].size();
    ss << "\n\n";
    for (auto& s : strs) ss << s;
    ss << "end of trees\n";
    std::vector<double> imp = FeatureImportance(num_iteration, importance_type);
    std::vector<std::pair<size_t, std::string>> pairs;
    for (size_t i = 0; i < imp.size() && i < feature_names.size(); ++i) {
      size_t v = static_cast<size_t>(imp[i]);
      if (v > 0) pairs.emplace_back(v, feature_names[i]);
    }
    std::stable_sort(pairs.begin(), pairs.end(), [](const auto& a, const auto& b) { return a.first > b.first; });
    ss << "\nfeature_importances:\n";
    for (auto& p : pairs) ss << p.second << "=" << p.first << '\n';
    const std::string& pb = params_block.empty() ? loaded_parameters : params_block;
    if (!pb.empty()) ss << "\nparameters:\n" << pb << "\nend of parameters\n";
    return ss.str();
  }

  static std::unique_ptr<HostModel> FromString(const std::string& text) {
    std::unique_ptr<HostModel> m(new HostModel());
    std::vector<std::string> lines;
    {
      std::istringstream is(text);
      std::string ln;
      while (std::getline(is, ln)) { if (!ln.empty() && ln.back() == '\r') ln.pop_back(); lines.push_back(ln); }
    }
    size_t i = 0;
    std::map<std::string, std::string> head;
    bool saw_tree_header = false;
    for (; i < lines.size(); ++i) {
      const std::string& ln = lines[i];
      if (ln.rfind("Tree=", 0) == 0 || ln == "end of trees") break;
      if (ln == "tree") { saw_tree_header = true; continue; }
      if (ln == "average_output") { m->average_output = true; continue; }
      size_t p = ln.find('=');
      if (p != std::string::npos) head[ln.substr(0, p)] = ln.substr(p + 1);
    }
    (void)saw_tree_header;
    auto need = [&](const char* k) -> std::string {
      auto it = head.find(k);
      if (it == head.end()) throw std::runtime_error(std::string("Model file doesn't specify ") + k);
      return it->second;
    };
    m->num_class = std::atoi(need("num_class").c_str());
    m->num_tree_per_iteration = head.count("num_tree_per_iteration") ? std::atoi(head["num_tree_per_iteration"].c_str()) : m->num_class;
    m->label_index = std::atoi(need("label_index").c_str());
    m->max_feature_idx = std::atoi(need("max_feature_idx").c_str());
    if (head.count("objective")) m->objective_str = head["objective"];
    {
      OutputTransform t;      // an objective whose output transform is unknown must not silently predict raw scores as probabilities
      if (!ObjectiveTransform(m->objective_str, &t)) throw std::runtime_error("Unknown objective type name: " + m->objective_str);
    }
    {
      std::istringstream is(need("feature_names"));
      std::string x;
      while (is >> x) m->feature_names.push_back(x);
      if (static_cast<int>(m->feature_names.size()) != m->max_feature_idx + 1) throw std::runtime_error("Wrong size of feature_names");
    }
    if (head.count("monotone_constraints")) {
      std::istringstream is(head["monotone_constraints"]);
      int x;
      while (is >> x) m->monotone_constraints.push_back(x);
    }
    if (head.count("feature_infos")) {
      std::istringstream is(head["feature_infos"]);
      std::string x;
      while (is >> x) m->feature_infos.push_back(x);
    }
    while (i < lines.size()) {
      if (lines[i].rfind("Tree=", 0) == 0) {
        std::map<std::string, std::string> kv;
        ++i;
        for (; i < lines.size(); ++i) {
          const std::string& ln = lines[i];
          if (ln.rfind("Tree=", 0) == 0 || ln == "end of trees") break;
          size_t p = ln.find('=');
          if (p != std::string::npos) kv[ln.substr(0, p)] = ln.substr(p + 1);
        }
        m->trees.emplace_back(new HostTree(HostTree::FromKV(kv)));
      } else if (lines[i] == "end of trees") {
        ++i;
        break;
      } else {
        ++i;
      }
    }
    for (; i < lines.size(); ++i) {
      if (lines[i] == "parameters:") {
        std::string pb;
        for (++i; i < lines.size() && lines[i] != "end of parameters"; ++i) pb += (pb.empty() ? "" : "\n") + lines[i];
        m->loaded_parameters = pb;
      }
    }
    return m;
  }

  // objective output transform ([UPSTREAM] ObjectiveFunction::ConvertOutput of the objective named in the model header).
  // kind: 0 identity, 1 sigmoid(sig * x), 2 softmax, 3 exp, 4 per-class sigmoid (multiclassova), 5 log1p(exp(x)) (cross_entropy_lambda),
  // 6 sign(x) * x^2 (regression with the `sqrt` flag)
  struct OutputTransform { int kind = 0; double sigmoid = 1.0; };
  static bool ObjectiveTransform(const std::string& o, OutputTransform* t) {
    std::istringstream is(o);
    std::string name, tok;
    is >> name;
    OutputTransform r;
    bool sqrt_flag = false;
    while (is >> tok) {
      if (tok.rfind("sigmoid:", 0) == 0) r.sigmoid = std::atof(tok.c_str() + 8);
      else if (tok == "sqrt") sqrt_flag = true;
    }
    if (name.empty() || name == "custom" || name == "none" || name == "null" || name == "na") r.kind = 0;
    else if (name == "regression" || name == "regression_l1" || name == "huber" || name == "fair" || name == "quantile" || name == "mape" ||
             name == "lambdarank" || name == "rank_xendcg") r.kind = (name == "regression" && sqrt_flag) ? 6 : 0;
    else if (name == "binary") r.kind = 1;
    else if (name == "multiclass") r.kind = 2;
    else if (name == "poisson" || name == "gamma" || name == "tweedie") r.kind = 3;
    else if (name == "multiclassova") r.kind = 4;
    else if (name == "cross_entropy") { r.kind = 1; r.sigmoid = 1.0; }
    else if (name == "cross_entropy_lambda") r.kind = 5;
    else return false;
    *t = r;
    return true;
  }
  // nrow rows of K raw scores, class k of row i at s[i * row_step + k * class_step], turned into outputs in place: the mean over
  // `iterations` for an averaged (rf) model when iterations > 0, then the objective transform unless raw
  void ConvertScores(double* s, int64_t nrow, int64_t row_step, int64_t class_step, int iterations, bool raw) const {
    const int K = num_tree_per_iteration;
    const bool avg = average_output && iterations > 0;
    OutputTransform t;
    if (!raw && !ObjectiveTransform(objective_str, &t)) throw std::runtime_error("Unknown objective type name: " + objective_str);
    for (int64_t i = 0; i < nrow && (avg || !raw); ++i) {
      double* p = s + i * row_step;
      auto v = [&](int k) -> double& { return p[k * class_step]; };
      if (avg) for (int k = 0; k < K; ++k) v(k) /= iterations;
      if (raw) continue;
      switch (t.kind) {
        case 1: v(0) = 1.0 / (1.0 + std::exp(-t.sigmoid * v(0))); break;
        case 2: {
          double mx = v(0);
          for (int k = 1; k < num_class; ++k) mx = std::max(mx, v(k));
          double sum = 0;
          for (int k = 0; k < num_class; ++k) { v(k) = std::exp(v(k) - mx); sum += v(k); }
          for (int k = 0; k < num_class; ++k) v(k) /= sum;
          break;
        }
        case 3: v(0) = std::exp(v(0)); break;
        case 4: for (int k = 0; k < K; ++k) v(k) = 1.0 / (1.0 + std::exp(-t.sigmoid * v(k))); break;
        case 5: v(0) = std::log1p(std::exp(v(0))); break;
        case 6: v(0) = (v(0) >= 0 ? 1.0 : -1.0) * v(0) * v(0); break;
      }
    }
  }
  int64_t NumPredictPerRow(int predict_type, int start_iteration, int num_iteration) const {      // outputs per row of predict_type
    int t0, t1;
    IterRange(start_iteration, num_iteration, &t0, &t1);
    return predict_type == 2 ? t1 - t0 : predict_type == 3 ? static_cast<int64_t>(num_tree_per_iteration) * (max_feature_idx + 2) : num_tree_per_iteration;
  }
  void IterRange(int start_iteration, int num_iteration, int* t0, int* t1) const {
    int total = NumIterations();
    start_iteration = std::min(std::max(start_iteration, 0), total);
    int end = num_iteration > 0 ? std::min(start_iteration + num_iteration, total) : total;
    *t0 = start_iteration * num_tree_per_iteration;
    *t1 = end * num_tree_per_iteration;
  }
  // predict_type: 0 normal, 1 raw, 2 leaf index, 3 contrib.  Returns number of outputs written.
  int64_t PredictRow(const double* row, int ncol, int predict_type, int start_iteration, int num_iteration, double* out) const {
    int t0, t1;
    IterRange(start_iteration, num_iteration, &t0, &t1);
    const int K = num_tree_per_iteration;
    std::vector<double> padded;
    if (ncol < max_feature_idx + 1) {      // missing trailing columns read as 0
      padded.assign(row, row + ncol);
      padded.resize(max_feature_idx + 1, 0.0);
      row = padded.data();
    }
    if (predict_type == 2) {
      for (int t = t0; t < t1; ++t) out[t - t0] = trees[t]->LeafIndex(row);
    } else if (predict_type == 3) {
      const int nf1 = max_feature_idx + 2;
      for (int k = 0; k < K * nf1; ++k) out[k] = 0;
      for (int t = t0; t < t1; ++t) trees[t]->AddContrib(row, max_feature_idx + 1, out + (t % K) * nf1);
    } else {
      for (int k = 0; k < K; ++k) out[k] = 0;
      for (int t = t0; t < t1; ++t) out[t % K] += trees[t]->Predict(row);
      ConvertScores(out, 1, K, 1, (t1 - t0) / K, predict_type == 1);
    }
    return NumPredictPerRow(predict_type, start_iteration, num_iteration);
  }
};

}  // namespace b200gbm
