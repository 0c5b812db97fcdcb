// Strategy enumeration, resharding cost model, follow-merged cost graph and ILP assembly.
// See planner.h for the design; reference counterparts are cited per function.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <functional>
#include <map>
#include <numeric>
#include <random>
#include <set>
#include <sstream>

#include "planner.h"

namespace abp {

// ---------------------------------------------------------------------------------------------
// alpha-beta collectives (same structure as LogicalDeviceMesh, alpa/shard_parallel/auto_sharding.py:121-141)
// ---------------------------------------------------------------------------------------------
double MeshEnv::all_gather_cost(double bytes, int a) const {
  const double n = shape[a];
  return alpha[a] + beta[a] * (n - 1) / n * bytes + 0.1;
}
double MeshEnv::all_reduce_cost(double bytes, int a) const {
  const double n = shape[a];
  return alpha[a] + beta[a] * 2 * (n - 1) / n * bytes + 0.01;
}
double MeshEnv::reduce_scatter_cost(double bytes, int a) const {
  const double n = shape[a];
  return alpha[a] + beta[a] * (n - 1) / n * bytes + 0.001;
}
double MeshEnv::all_to_all_cost(double bytes, int a) const {
  // NVSwitch: full-rate path between every pair, no ring penalty (the reference uses n/2 for V100 rings)
  const double n = shape[a];
  return alpha[a] + beta[a] * (n - 1) / n / n * bytes + 0.001;
}

int Graph::add_node(Node n) {
  n.id = static_cast<int>(nodes_.size());
  nodes_.push_back(std::move(n));
  return nodes_.back().id;
}

static double tensor_bytes(const Output& t) {
  double b = t.dtype_bytes;
  for (int64_t s : t.shape) b *= static_cast<double>(s);
  return b;
}

static int num_shards(const Spec& s, const MeshEnv& env) {
  int n = 1;
  for (const auto& axes : s)
    for (int a : axes) n *= env.shape[a];
  return n;
}

// ---------------------------------------------------------------------------------------------
// Batch-dim inference (reference: BuildInstructionBatchDimMap, auto_sharding_util.cc:300)
// ---------------------------------------------------------------------------------------------
void Graph::infer_batch_labels() {
  for (auto& n : nodes_) {
    if (n.kind == kInput) {
      if (n.is_batch_input && !n.outputs.empty() && !n.outputs[0].labels.empty())
        n.batch_label = n.outputs[0].labels[0];
      continue;
    }
    n.batch_label = -1;
    for (const auto& op : n.operands) {
      const Node& p = nodes_[op.node];
      if (p.batch_label < 0) continue;
      const Output& po = p.outputs[op.out_idx];
      for (size_t d = 0; d < po.labels.size() && d < op.labels.size(); ++d) {
        if (po.labels[d] == p.batch_label && op.labels[d] >= 0) {
          n.batch_label = op.labels[d];
          break;
        }
      }
      if (n.batch_label >= 0) break;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Strategies
// ---------------------------------------------------------------------------------------------
static Spec spec_from_labels(const std::vector<int>& labels, const std::vector<std::vector<int>>& label_axes) {
  Spec s(labels.size());
  for (size_t d = 0; d < labels.size(); ++d)
    if (labels[d] >= 0) s[d] = label_axes[labels[d]];
  return s;
}

static std::string spec_str(const Spec& s) {
  if (s.empty()) return "R";
  std::string r;
  for (const auto& axes : s) {
    if (axes.empty()) {
      r += "R";
    } else {
      r += "S";
      for (int a : axes) r += std::to_string(a);
    }
  }
  return r;
}

// Fill specs, all-reduce axes and costs of a strategy from its label->axes assignment.
static void finalize_strategy(const Node& n, const MeshEnv& env, Strategy& st) {
  st.in_specs.clear();
  st.out_specs.clear();
  st.allreduce_axes.clear();
  for (const auto& op : n.operands) st.in_specs.push_back(spec_from_labels(op.labels, st.label_axes));
  // labels that appear in at least one operand
  std::vector<char> in_operand(n.labels.size(), 0);
  for (const auto& op : n.operands)
    for (int l : op.labels)
      if (l >= 0) in_operand[l] = 1;
  st.comm_cost = 0;
  st.memory_cost = 0;
  for (const auto& out : n.outputs) {
    Spec os = spec_from_labels(out.labels, st.label_axes);
    std::vector<char> in_out(n.labels.size(), 0);
    for (int l : out.labels)
      if (l >= 0) in_out[l] = 1;
    std::vector<char> in_dep = in_operand;
    if (!out.depends.empty()) {
      std::fill(in_dep.begin(), in_dep.end(), 0);
      for (int oi : out.depends)
        if (oi >= 0 && oi < (int)n.operands.size())
          for (int l : n.operands[oi].labels)
            if (l >= 0) in_dep[l] = 1;
    }
    std::vector<int> ar;
    for (size_t l = 0; l < n.labels.size(); ++l)
      if (in_dep[l] && !in_out[l])
        for (int a : st.label_axes[l]) ar.push_back(a);
    std::sort(ar.begin(), ar.end());
    const double local = tensor_bytes(out) / num_shards(os, env);
    for (int a : ar) st.comm_cost += env.all_reduce_cost(local, a);
    if (n.allocates) st.memory_cost += local;
    st.out_specs.push_back(std::move(os));
    st.allreduce_axes.push_back(std::move(ar));
  }
  std::ostringstream nm;
  for (size_t i = 0; i < st.out_specs.size(); ++i) nm << (i ? "," : "") << spec_str(st.out_specs[i]);
  nm << " = ";
  for (size_t i = 0; i < st.in_specs.size(); ++i) nm << (i ? " x " : "") << spec_str(st.in_specs[i]);
  bool any_ar = false;
  for (const auto& ar : st.allreduce_axes) any_ar |= !ar.empty();
  if (any_ar) {
    nm << " + allreduce@";
    std::set<int> axes;
    for (const auto& ar : st.allreduce_axes) axes.insert(ar.begin(), ar.end());
    for (int a : axes) nm << a;
  }
  st.name = nm.str();
}

static bool strategy_allowed(const Node& n, const MeshEnv& env, const Options& opt, const Strategy& st) {
  const int nd = static_cast<int>(env.shape.size());
  // Pure data parallelism: tensors that carry the batch dim shard only that dim; parameters stay
  // replicated.  Intermediate leaders without a known batch dim (broadcasts / constants created inside
  // the step, e.g. the seed of the backward pass) stay free so they can match their consumers.
  if (opt.force_data_parallel && (n.batch_label >= 0 || n.kind == kInput)) {
    for (size_t l = 0; l < st.label_axes.size(); ++l)
      if (!st.label_axes[l].empty() && static_cast<int>(l) != n.batch_label) return false;
  }
  if (opt.force_batch_dim_to_mesh_dim >= 0 && opt.force_batch_dim_to_mesh_dim < nd && n.batch_label >= 0) {
    const int k = opt.force_batch_dim_to_mesh_dim;
    if (env.shape[k] > 1 && n.labels[n.batch_label].kind == kShardable &&
        n.labels[n.batch_label].size % env.shape[k] == 0) {
      const auto& ax = st.label_axes[n.batch_label];
      if (std::find(ax.begin(), ax.end(), k) == ax.end()) return false;
      // the batch axis must not be used by any other label (implied by one-axis-one-label)
    }
  }
  return true;
}

// Ratio between tensor-core math and NVLink traffic on the H100 SXM from data-sheet rates: 989e12 dense bf16 FLOP/s
// against 4.5e11 B/s per direction of NVLink 4 (~2200 FLOP per byte moved).
constexpr double kFlopsPerCommUnit = 2200.0;

// Reference: AnnotateShardingWithSimpleHeuristic (auto_sharding_util.cc:2017-2110): program inputs are laid out by a
// rule of thumb -- the largest / first / last dim tiled over the mesh (the two largest dims on a 2-D mesh for
// "shard-largest"), replicated when the size does not divide -- and everything else follows from the solver.
static bool simple_heuristic_ok(const Node& n, const MeshEnv& env, const Options& opt, const Strategy& st) {
  if (n.outputs.empty()) return true;
  const auto& out = n.outputs[0];
  const int rank = static_cast<int>(out.shape.size());
  std::vector<int> active;
  for (size_t a = 0; a < env.shape.size(); ++a)
    if (env.shape[a] > 1) active.push_back(static_cast<int>(a));
  Spec want(rank);
  if (rank > 0 && !active.empty()) {
    const int64_t ndev = env.num_devices();
    auto divisible = [&](int d, int64_t by) { return out.labels[d] >= 0 && out.shape[d] % by == 0 && out.shape[d] >= by; };
    if (opt.force_simple_heuristic == "shard-first") {
      if (divisible(0, ndev)) want[0] = active;
    } else if (opt.force_simple_heuristic == "shard-last") {
      if (divisible(rank - 1, ndev)) want[rank - 1] = active;
    } else {  // shard-largest
      std::vector<int> order(rank);
      std::iota(order.begin(), order.end(), 0);
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return out.shape[a] > out.shape[b]; });
      if (active.size() == 1 || rank == 1) {
        if (divisible(order[0], ndev)) want[order[0]] = active;
      } else {
        const int d1 = order[0], d0 = order[1];
        if (divisible(d0, env.shape[active[0]]) && divisible(d1, env.shape[active[1]])) {
          want[d0] = {active[0]};
          want[d1] = {active[1]};
        }
      }
    }
  }
  return spec_from_labels(out.labels, st.label_axes) == want;
}

// Reference: BuildStrategyAndCost (auto_sharding.cc:490) + DotHandler (auto_sharding_dot_handler.cc:34-408).
static void enumerate_leader(Node& n, const MeshEnv& env, const Options& opt) {
  n.strategies.clear();
  std::vector<int> active;
  for (size_t a = 0; a < env.shape.size(); ++a)
    if (env.shape[a] > 1) active.push_back(static_cast<int>(a));
  const int L = static_cast<int>(n.labels.size());
  const bool heavy = n.flops > 0 && n.kind == kCompute;
  std::vector<int> assign(active.size(), -1);
  std::function<void(size_t)> rec = [&](size_t i) {
    if (i == active.size()) {
      Strategy st;
      st.label_axes.assign(L, {});
      for (size_t k = 0; k < active.size(); ++k)
        if (assign[k] >= 0) st.label_axes[assign[k]].push_back(active[k]);
      for (int l = 0; l < L; ++l) {
        int64_t prod = 1;
        for (int a : st.label_axes[l]) prod *= env.shape[a];
        if (prod > 1 && (n.labels[l].kind != kShardable || n.labels[l].size % prod != 0)) return;
        if (st.label_axes[l].size() > 1 && !opt.allow_mixed_mesh_shape && !opt.force_data_parallel &&
            static_cast<int>(l) != n.batch_label && n.kind != kInput)
          return;
        if (st.label_axes[l].size() > 1) std::sort(st.label_axes[l].begin(), st.label_axes[l].end());
      }
      double dup = 1;   // how many times the op's FLOPs are executed across the mesh, relative to once
      for (size_t k = 0; k < active.size(); ++k)
        if (assign[k] < 0) dup *= env.shape[active[k]];
      if (heavy && dup > 1 && !opt.allow_recompute_heavy_op) return;  // heavy ops use the whole mesh (no duplicated
                                                                      // FLOPs), like the reference's dot handler
      if (!strategy_allowed(n, env, opt, st)) return;
      if (n.kind == kInput && !opt.force_simple_heuristic.empty() && !simple_heuristic_ok(n, env, opt, st)) return;
      finalize_strategy(n, env, st);
      if (heavy && dup > 1) {
        // recomputation: every device of the unused mesh axes repeats the math; charged at the link-equivalent price
        // of the extra time (kFlopsPerCommUnit FLOPs take as long as one cost unit = one byte over the slow axis)
        st.compute_cost = n.flops / env.num_devices() * (dup - 1) / kFlopsPerCommUnit;
        st.name += " [recompute x" + std::to_string((int)dup) + "]";
      }
      if (n.is_parameter && !opt.allow_replicated_parameters) {
        bool repl = true;
        for (const auto& ax : st.label_axes) repl &= ax.empty();
        if (repl && !active.empty()) return;
      }
      n.strategies.push_back(std::move(st));
      return;
    }
    for (int l = -1; l < L; ++l) {
      assign[i] = l;
      rec(i + 1);
    }
  };
  rec(0);
  if (n.strategies.empty()) {  // constraints too tight: relax heavy/force filters, keep correctness
    Strategy st;
    st.label_axes.assign(L, {});
    finalize_strategy(n, env, st);
    n.strategies.push_back(std::move(st));
  }
}

// Reference: FollowInsStrategyVector (auto_sharding.cc:130): strategy k mirrors strategy k of the
// followed operand's producer.
static void derive_follower(Node& n, const Graph& g, const MeshEnv& env) {
  n.strategies.clear();
  const Operand& fop = n.operands[n.follow];
  const Node& p = g.node(fop.node);
  const int L = static_cast<int>(n.labels.size());
  for (const auto& ps : p.strategies) {
    const Spec& sp = ps.out_specs[fop.out_idx];
    Strategy st;
    st.label_axes.assign(L, {});
    std::vector<char> used_axis(env.shape.size(), 0);
    for (size_t d = 0; d < fop.labels.size() && d < sp.size(); ++d) {
      const int l = fop.labels[d];
      if (l < 0 || sp[d].empty() || !st.label_axes[l].empty()) continue;
      if (n.labels[l].kind != kShardable) continue;
      int64_t prod = 1;
      for (int a : sp[d]) prod *= env.shape[a];
      if (n.labels[l].size % prod != 0) continue;
      bool clash = false;
      for (int a : sp[d]) clash |= used_axis[a];
      if (clash) continue;
      st.label_axes[l] = sp[d];
      for (int a : sp[d]) used_axis[a] = 1;
    }
    finalize_strategy(n, env, st);
    n.strategies.push_back(std::move(st));
  }
}

void Graph::build_strategies(const MeshEnv& env, const Options& opt) {
  infer_batch_labels();
  for (auto& n : nodes_) {
    if (n.follow >= 0 && n.follow < static_cast<int>(n.operands.size()))
      derive_follower(n, *this, env);
    else
      enumerate_leader(n, env, opt);
  }
}

// ---------------------------------------------------------------------------------------------
// Resharding cost (reference: ClusterEnvironment::ReshardingCost, auto_sharding_strategy.h:476-553)
// ---------------------------------------------------------------------------------------------
double Graph::resharding_cost(const Output& t, const Spec& src, const Spec& dst, const MeshEnv& env,
                              const Options& opt) const {
  if (src == dst) return 0;
  const int nd = static_cast<int>(env.shape.size());
  const double full = tensor_bytes(t);
  auto dim_of = [&](const Spec& s, int a) {
    for (size_t d = 0; d < s.size(); ++d)
      if (std::find(s[d].begin(), s[d].end(), a) != s[d].end()) return static_cast<int>(d);
    return -1;
  };
  double cost = 0;
  // shards contributed by axes that stay put (they divide the message size)
  for (int a = 0; a < nd; ++a) {
    if (env.shape[a] <= 1) continue;
    const int sd = dim_of(src, a), dd = dim_of(dst, a);
    if (sd == dd) continue;
    double other = 1;
    for (int b = 0; b < nd; ++b)
      if (b != a && dim_of(src, b) >= 0) other *= env.shape[b];
    const double bytes = full / other;
    if (sd >= 0 && dd < 0) {
      if (!opt.allow_all_gather) return kInf;
      cost += env.all_gather_cost(bytes, a);
    } else if (sd < 0 && dd >= 0) {
      // local slice: no wire traffic, but a copy kernel and a second layout of the same value; the small charge makes
      // "keep the producer's layout" win ties, so equal-communication plans do not shard state at random
      cost += 0.05 + 1e-3 * bytes / env.shape[a];
    } else {
      if (!opt.allow_all_to_all) return kInf;
      cost += env.all_to_all_cost(bytes, a);
    }
  }
  return cost;
}

// ---------------------------------------------------------------------------------------------
// Cost graph with follow-merging (reference: CostGraph::MergeNode/Simplify, auto_sharding_strategy.h:706-1000)
// ---------------------------------------------------------------------------------------------
IlpProblem Graph::build_ilp(const MeshEnv& env, const Options& opt) {
  const int n = size();
  leader_of.assign(n, -1);
  for (int i = 0; i < n; ++i) {
    const Node& nd = nodes_[i];
    if (nd.follow >= 0 && nd.follow < static_cast<int>(nd.operands.size()))
      leader_of[i] = leader_of[nd.operands[nd.follow].node];
    else
      leader_of[i] = i;
  }
  IlpProblem p;
  std::vector<int> ilp_idx(n, -1);
  for (int i = 0; i < n; ++i)
    if (leader_of[i] == i) {
      ilp_idx[i] = p.N++;
      p.leader_node.push_back(i);
      p.s_len.push_back(static_cast<int>(nodes_[i].strategies.size()));
      p.c.emplace_back(nodes_[i].strategies.size(), 0.0);
      p.m.emplace_back(nodes_[i].strategies.size(), 0.0);
    }
  std::map<std::pair<int, int>, int> edge_idx;
  auto edge = [&](int a, int b) -> std::vector<double>& {
    auto key = std::make_pair(a, b);
    auto it = edge_idx.find(key);
    if (it == edge_idx.end()) {
      edge_idx[key] = static_cast<int>(p.edges.size());
      p.edges.push_back(key);
      p.r.emplace_back(static_cast<size_t>(p.s_len[a]) * p.s_len[b], 0.0);
      return p.r.back();
    }
    return p.r[it->second];
  };
  auto add_cost = [&](int ga, int gb, int ka, int kb, double v) {
    // ga, gb: ILP node ids; ka, kb strategy indices
    if (ga == gb) {
      if (ka == kb) p.c[ga][ka] = std::min(kInf, p.c[ga][ka] + v);
      return;
    }
    if (ga < gb)
      edge(ga, gb)[static_cast<size_t>(ka) * p.s_len[gb] + kb] += v;
    else
      edge(gb, ga)[static_cast<size_t>(kb) * p.s_len[ga] + ka] += v;
  };
  for (int i = 0; i < n; ++i) {
    const Node& nd = nodes_[i];
    const int gi = ilp_idx[leader_of[i]];
    for (size_t k = 0; k < nd.strategies.size(); ++k) {
      p.c[gi][k] += nd.strategies[k].comm_cost + nd.strategies[k].compute_cost;
      p.m[gi][k] += nd.strategies[k].memory_cost;
    }
    for (size_t o = 0; o < nd.operands.size(); ++o) {
      const Operand& op = nd.operands[o];
      const Node& pr = nodes_[op.node];
      const int gp = ilp_idx[leader_of[op.node]];
      const Output& t = pr.outputs[op.out_idx];
      const bool mutated = std::find(nd.mutated_operands.begin(), nd.mutated_operands.end(), (int)o) !=
                           nd.mutated_operands.end();
      auto edge_cost = [&](const Spec& src, const Spec& dst) {
        if (mutated && src != dst) return kInf;   // an in-place update of a re-laid-out copy would be lost
        return resharding_cost(t, src, dst, env, opt);
      };
      if (gp == gi) {
        for (size_t k = 0; k < nd.strategies.size(); ++k)
          add_cost(gp, gi, k, k, edge_cost(pr.strategies[k].out_specs[op.out_idx], nd.strategies[k].in_specs[o]));
      } else {
        for (size_t kp = 0; kp < pr.strategies.size(); ++kp)
          for (size_t k = 0; k < nd.strategies.size(); ++k) {
            const double v = edge_cost(pr.strategies[kp].out_specs[op.out_idx], nd.strategies[k].in_specs[o]);
            if (v != 0) add_cost(gp, gi, kp, k, v);
          }
      }
    }
  }
  // donation aliases: input spec must equal the spec of the value that replaces it
  // (reference: alias constraints, auto_sharding.cc:1501-1576)
  for (const auto& al : alias_pairs) {
    const Node& a = nodes_[al.first];
    const int bnode = al.second >> 8, bout = al.second & 0xff;
    const Node& b = nodes_[bnode];
    const int ga = ilp_idx[leader_of[al.first]], gb = ilp_idx[leader_of[bnode]];
    for (size_t ka = 0; ka < a.strategies.size(); ++ka)
      for (size_t kb = 0; kb < b.strategies.size(); ++kb) {
        if (ga == gb && ka != kb) continue;
        if (a.strategies[ka].out_specs[0] != b.strategies[kb].out_specs[bout]) add_cost(ga, gb, ka, kb, kInf);
      }
  }
  // manual sharding pins (reference: ManualShardingOption -> fixed in/out shardings)
  for (const auto& pin : pinned_outputs) {
    const Node& nd = nodes_[std::get<0>(pin)];
    const int gi = ilp_idx[leader_of[std::get<0>(pin)]];
    const int oi = std::get<1>(pin);
    bool any = false;
    for (size_t k = 0; k < nd.strategies.size(); ++k)
      if (oi < (int)nd.strategies[k].out_specs.size() && nd.strategies[k].out_specs[oi] == std::get<2>(pin)) any = true;
    if (!any) continue;  // unreachable spec: leave the node free, the lowering reshards at the boundary
    for (size_t k = 0; k < nd.strategies.size(); ++k)
      if (oi >= (int)nd.strategies[k].out_specs.size() || nd.strategies[k].out_specs[oi] != std::get<2>(pin))
        p.c[gi][k] = kInf;
  }
  for (auto& row : p.r)
    for (auto& v : row) v = std::min(v, kInf);

  // ---- memory constraint rows (reference: liveness sets auto_sharding.cc:2196-2216, constraint
  // alpa/shard_parallel/auto_sharding.py:773-779).  Value i is alive from its definition to its last use; program
  // inputs (parameters, optimizer state, the batch) and values nobody consumes (program outputs) for the whole step.
  p.memory_budget = opt.memory_budget_per_device;
  {
    std::vector<int> last(n, -1);
    for (int i = 0; i < n; ++i)
      for (const auto& op : nodes_[i].operands) last[op.node] = std::max(last[op.node], i);
    for (int i = 0; i < n; ++i)
      if (nodes_[i].kind == kInput || last[i] < 0) last[i] = n - 1;
    std::vector<std::vector<int>> dying(n);
    for (int i = 0; i < n; ++i) dying[last[i]].push_back(i);
    // running per-(leader, strategy) coefficients of the live set
    std::vector<std::vector<double>> coef(p.N);
    for (int g = 0; g < p.N; ++g) coef[g].assign(p.s_len[g], 0.0);
    std::vector<int> live_count(p.N, 0);
    double min_now = 0, max_now = 0;          // sum over live values of their cheapest / dearest layout
    std::vector<double> vmin(n, 0), vmax(n, 0);
    for (int i = 0; i < n; ++i) {
      double lo = std::numeric_limits<double>::infinity(), hi = 0;
      for (const auto& st : nodes_[i].strategies) {
        lo = std::min(lo, st.memory_cost);
        hi = std::max(hi, st.memory_cost);
      }
      vmin[i] = nodes_[i].strategies.empty() ? 0 : lo;
      vmax[i] = hi;
    }
    p.min_peak_memory = 0;
    for (int t = 0; t < n; ++t) {
      const int g = ilp_idx[leader_of[t]];
      for (size_t k = 0; k < nodes_[t].strategies.size() && k < coef[g].size(); ++k)
        coef[g][k] += nodes_[t].strategies[k].memory_cost;
      ++live_count[g];
      min_now += vmin[t];
      max_now += vmax[t];
      p.min_peak_memory = std::max(p.min_peak_memory, min_now);
      const bool peak = !dying[t].empty() || t == n - 1;   // something is released right after: a local maximum
      if (peak && p.memory_budget > 0 && max_now > p.memory_budget) {
        std::vector<std::tuple<int, int, double>> row;
        for (int gg = 0; gg < p.N; ++gg) {
          if (live_count[gg] == 0) continue;
          for (int k = 0; k < p.s_len[gg]; ++k)
            if (coef[gg][k] > 0) row.emplace_back(gg, k, coef[gg][k]);
        }
        p.mem_time.push_back(t);
        p.mem_rows.push_back(std::move(row));
      }
      for (int d : dying[t]) {
        const int gd = ilp_idx[leader_of[d]];
        for (size_t k = 0; k < nodes_[d].strategies.size() && k < coef[gd].size(); ++k)
          coef[gd][k] = std::max(0.0, coef[gd][k] - nodes_[d].strategies[k].memory_cost);
        --live_count[gd];
        min_now -= vmin[d];
        max_now -= vmax[d];
      }
    }
  }
  p.original_N = p.N;
  p.original_s_len = p.s_len;
  return p;
}

// Peak of the live-set memory under the currently chosen strategies (bytes per device).
double Graph::peak_memory(const IlpProblem& p, const std::vector<int>& s_val) const {
  const int n = size();
  std::vector<int> ilp_idx(n, -1);
  for (int i = 0; i < p.original_N && i < (int)p.leader_node.size(); ++i) ilp_idx[p.leader_node[i]] = i;
  std::vector<int> last(n, -1);
  for (int i = 0; i < n; ++i)
    for (const auto& op : nodes_[i].operands) last[op.node] = std::max(last[op.node], i);
  for (int i = 0; i < n; ++i)
    if (nodes_[i].kind == kInput || last[i] < 0) last[i] = n - 1;
  std::vector<std::vector<int>> dying(n);
  for (int i = 0; i < n; ++i) dying[last[i]].push_back(i);
  auto mem = [&](int i) {
    const int k = s_val[ilp_idx[leader_of[i]]];
    return k < (int)nodes_[i].strategies.size() ? nodes_[i].strategies[k].memory_cost : 0.0;
  };
  double now = 0, peak = 0;
  for (int t = 0; t < n; ++t) {
    now += mem(t);
    peak = std::max(peak, now);
    for (int d : dying[t]) now -= mem(d);
  }
  return peak;
}

// ---------------------------------------------------------------------------------------------
// Cost-graph simplification by exact elimination (see planner.h)
// ---------------------------------------------------------------------------------------------
IlpProblem Graph::simplify(const IlpProblem& p) const {
  const int N = p.N;
  std::vector<std::vector<double>> c = p.c;
  // adjacency: neighbour -> matrix oriented [self][other]
  std::vector<std::map<int, std::vector<double>>> adj(N);
  auto transposed = [&](const std::vector<double>& m, int rows, int cols) {
    std::vector<double> t(m.size());
    for (int i = 0; i < rows; ++i)
      for (int j = 0; j < cols; ++j) t[(size_t)j * rows + i] = m[(size_t)i * cols + j];
    return t;
  };
  auto add_edge = [&](int a, int b, const std::vector<double>& mab) {   // mab: [s_a][s_b]
    auto it = adj[a].find(b);
    if (it == adj[a].end()) {
      adj[a][b] = mab;
      adj[b][a] = transposed(mab, p.s_len[a], p.s_len[b]);
    } else {
      auto& m1 = it->second;
      auto& m2 = adj[b][a];
      for (int i = 0; i < p.s_len[a]; ++i)
        for (int j = 0; j < p.s_len[b]; ++j) {
          const double v = std::min(kInf, m1[(size_t)i * p.s_len[b] + j] + mab[(size_t)i * p.s_len[b] + j]);
          m1[(size_t)i * p.s_len[b] + j] = v;
          m2[(size_t)j * p.s_len[a] + i] = v;
        }
    }
  };
  for (size_t e = 0; e < p.edges.size(); ++e) add_edge(p.edges[e].first, p.edges[e].second, p.r[e]);
  std::vector<char> locked(N, 0), gone(N, 0);
  for (const auto& row : p.mem_rows)
    for (const auto& t : row) locked[std::get<0>(t)] = 1;     // memory terms need the node's own variables
  for (const auto& al : p.alias) locked[al.first] = locked[al.second] = 1;

  IlpProblem out;
  out.memory_budget = p.memory_budget;
  out.min_peak_memory = p.min_peak_memory;
  out.original_N = N;
  out.original_s_len = p.s_len;
  out.leader_node = p.leader_node;          // indexed by ORIGINAL node (used by apply_solution after expand)
  std::vector<int> work;
  for (int i = 0; i < N; ++i) work.push_back(i);
  bool progress = true;
  while (progress) {
    progress = false;
    for (int v = 0; v < N; ++v) {
      if (gone[v] || locked[v] || adj[v].size() > 2) continue;
      const int sv = p.s_len[v];
      IlpProblem::Elim el;
      el.node = v;
      if (adj[v].empty()) {
        int best = 0;
        for (int k = 1; k < sv; ++k)
          if (c[v][k] < c[v][best]) best = k;
        el.choice = {best};
        out.constant += c[v][best];
      } else if (adj[v].size() == 1) {
        const int a = adj[v].begin()->first;
        const auto& m = adj[v].begin()->second;     // [sv][sa]
        const int sa = p.s_len[a];
        el.a = a;
        el.choice.assign(sa, 0);
        for (int ka = 0; ka < sa; ++ka) {
          double bestv = std::numeric_limits<double>::infinity();
          for (int k = 0; k < sv; ++k) {
            const double val = c[v][k] + m[(size_t)k * sa + ka];
            if (val < bestv) {
              bestv = val;
              el.choice[ka] = k;
            }
          }
          c[a][ka] = std::min(kInf, c[a][ka] + bestv);
        }
        adj[a].erase(v);
      } else {
        auto it = adj[v].begin();
        const int a = it->first;
        const std::vector<double> ma = it->second;   // [sv][sa]
        ++it;
        const int b = it->first;
        const std::vector<double> mb = it->second;   // [sv][sb]
        const int sa = p.s_len[a], sb = p.s_len[b];
        if ((long long)sa * sb * sv > (1 << 22)) continue;   // keep the folded matrix small
        el.a = a;
        el.b = b;
        el.choice.assign((size_t)sa * sb, 0);
        std::vector<double> mab((size_t)sa * sb, 0.0);
        for (int ka = 0; ka < sa; ++ka)
          for (int kb = 0; kb < sb; ++kb) {
            double bestv = std::numeric_limits<double>::infinity();
            int arg = 0;
            for (int k = 0; k < sv; ++k) {
              const double val = c[v][k] + ma[(size_t)k * sa + ka] + mb[(size_t)k * sb + kb];
              if (val < bestv) {
                bestv = val;
                arg = k;
              }
            }
            mab[(size_t)ka * sb + kb] = std::min(kInf, bestv);
            el.choice[(size_t)ka * sb + kb] = arg;
          }
        adj[a].erase(v);
        adj[b].erase(v);
        add_edge(a, b, mab);
      }
      adj[v].clear();
      gone[v] = 1;
      out.eliminated.push_back(std::move(el));
      progress = true;
    }
  }
  std::vector<int> new_idx(N, -1);
  for (int i = 0; i < N; ++i)
    if (!gone[i]) {
      new_idx[i] = out.N++;
      out.kept.push_back(i);
      out.s_len.push_back(p.s_len[i]);
      out.c.push_back(c[i]);
      out.m.push_back(p.m[i]);
    }
  for (int a = 0; a < N; ++a) {
    if (gone[a]) continue;
    for (const auto& [b, m] : adj[a]) {
      if (b <= a || gone[b]) continue;
      out.edges.push_back({new_idx[a], new_idx[b]});
      out.r.push_back(m);
    }
  }
  for (const auto& al : p.alias) out.alias.push_back({new_idx[al.first], new_idx[al.second]});
  out.mem_time = p.mem_time;
  for (const auto& row : p.mem_rows) {
    std::vector<std::tuple<int, int, double>> r2;
    for (const auto& t : row) r2.emplace_back(new_idx[std::get<0>(t)], std::get<1>(t), std::get<2>(t));
    out.mem_rows.push_back(std::move(r2));
  }
  return out;
}

std::vector<int> Graph::expand(const IlpProblem& reduced, const std::vector<int>& s_reduced) const {
  std::vector<int> s(reduced.original_N, 0);
  if (reduced.kept.empty() && reduced.eliminated.empty()) return s_reduced;   // not a simplified problem
  for (size_t i = 0; i < reduced.kept.size(); ++i) s[reduced.kept[i]] = s_reduced[i];
  for (auto it = reduced.eliminated.rbegin(); it != reduced.eliminated.rend(); ++it) {
    if (it->a < 0)
      s[it->node] = it->choice[0];
    else if (it->b < 0)
      s[it->node] = it->choice[s[it->a]];
    else
      s[it->node] = it->choice[(size_t)s[it->a] * reduced.original_s_len[it->b] + s[it->b]];
  }
  return s;
}

// ---------------------------------------------------------------------------------------------
// Built-in solver: iterated conditional modes with restarts (used when HiGHS is unavailable and as
// a warm start).  The ILP itself is usually solved by scipy's HiGHS through the Python driver.
// ---------------------------------------------------------------------------------------------
std::vector<int> Graph::solve_builtin(const IlpProblem& p, double* objective) const {
  std::vector<std::vector<std::pair<int, int>>> adj(p.N);  // (edge id, is_first)
  for (size_t e = 0; e < p.edges.size(); ++e) {
    adj[p.edges[e].first].push_back({static_cast<int>(e), 1});
    adj[p.edges[e].second].push_back({static_cast<int>(e), 0});
  }
  // memory rows enter as a stiff penalty on the excess over the budget (the exact constraint is HiGHS's job)
  auto mem_excess = [&](const std::vector<int>& s) {
    double worst = 0;
    for (const auto& row : p.mem_rows) {
      double m = 0;
      for (const auto& t : row)
        if (s[std::get<0>(t)] == std::get<1>(t)) m += std::get<2>(t);
      worst = std::max(worst, m - p.memory_budget);
    }
    return worst;
  };
  auto total = [&](const std::vector<int>& s) {
    double t = p.mem_rows.empty() ? 0.0 : 1e3 * std::max(0.0, mem_excess(s));
    for (int i = 0; i < p.N; ++i) t += p.c[i][s[i]];
    for (size_t e = 0; e < p.edges.size(); ++e) {
      const int a = p.edges[e].first, b = p.edges[e].second;
      t += p.r[e][static_cast<size_t>(s[a]) * p.s_len[b] + s[b]];
    }
    return t;
  };
  std::mt19937 rng(42);
  std::vector<int> best;
  double best_cost = std::numeric_limits<double>::infinity();
  for (int restart = 0; restart < 8; ++restart) {
    std::vector<int> s(p.N, 0);
    for (int i = 0; i < p.N; ++i) {
      if (restart == 0)
        s[i] = static_cast<int>(std::min_element(p.c[i].begin(), p.c[i].end()) - p.c[i].begin());
      else
        s[i] = static_cast<int>(rng() % p.s_len[i]);
    }
    bool changed = true;
    int sweeps = 0;
    while (changed && sweeps++ < 50) {
      changed = false;
      for (int i = 0; i < p.N; ++i) {
        int arg = s[i];
        double bestv = std::numeric_limits<double>::infinity();
        for (int k = 0; k < p.s_len[i]; ++k) {
          double v = p.c[i][k];
          for (const auto& [e, first] : adj[i]) {
            const int a = p.edges[e].first, b = p.edges[e].second;
            v += first ? p.r[e][static_cast<size_t>(k) * p.s_len[b] + s[b]]
                       : p.r[e][static_cast<size_t>(s[a]) * p.s_len[b] + k];
          }
          if (!p.mem_rows.empty()) {
            const int keep = s[i];
            s[i] = k;
            v += 1e3 * std::max(0.0, mem_excess(s));
            s[i] = keep;
          }
          if (v < bestv - 1e-9) {
            bestv = v;
            arg = k;
          }
        }
        if (arg != s[i]) {
          s[i] = arg;
          changed = true;
        }
      }
    }
    const double t = total(s);
    if (t < best_cost) {
      best_cost = t;
      best = s;
    }
  }
  if (objective) *objective = best_cost;
  return best;
}

void Graph::apply_solution(const IlpProblem& p, const std::vector<int>& s_val) {
  std::vector<int> ilp_idx(size(), -1);
  for (int i = 0; i < p.N; ++i) ilp_idx[p.leader_node[i]] = i;
  for (int i = 0; i < size(); ++i) nodes_[i].chosen = s_val[ilp_idx[leader_of[i]]];
}

// ---------------------------------------------------------------------------------------------
// ZeRO rewrite (reference: GenerateReduceScatter, auto_sharding_util.cc:1458-1747).
// A gradient that is all-reduced over mesh axis `a` and then only feeds element-wise optimizer math
// whose other operands are parameters / optimizer state can instead be reduce-scattered: the
// optimizer math runs on 1/n of the elements and the state inputs become sharded along `a`.
// Here the rewrite is expressed on the chosen strategies: for every parameter-group (an in-place
// update node or an element-wise chain ending in a donated output) we shard one more tensor dim.
// Returns the number of rewritten all-reduces.  The Python lowering consumes the updated specs.
// ---------------------------------------------------------------------------------------------
int Graph::rewrite_reduce_scatter(const MeshEnv& env, const Options& opt) {
  (void)opt;
  int rewritten = 0;
  const int n = size();
  // users map
  std::vector<std::vector<int>> users(n);
  for (int i = 0; i < n; ++i)
    for (const auto& op : nodes_[i].operands) users[op.node].push_back(i);
  for (int i = 0; i < n; ++i) {
    Node& nd = nodes_[i];
    if (nd.chosen < 0 || nd.kind != kCompute) continue;
    Strategy& st = nd.strategies[nd.chosen];
    if (st.allreduce_axes.empty() || st.allreduce_axes[0].size() != 1 || nd.outputs.size() != 1) continue;
    const int a = st.allreduce_axes[0][0];
    // every transitive user must be "zero-compatible": flagged by the front end through flops<0
    // (element-wise optimizer math) -- see shard/planner.py which marks those nodes.
    bool ok = !users[i].empty();
    std::vector<int> chain;
    std::vector<int> stack(users[i].begin(), users[i].end());
    std::set<int> seen;
    while (!stack.empty() && ok) {
      const int u = stack.back();
      stack.pop_back();
      if (!seen.insert(u).second) continue;
      if (nodes_[u].flops >= 0) {
        ok = false;
        break;
      }
      chain.push_back(u);
      for (int v : users[u]) stack.push_back(v);
    }
    if (!ok) continue;
    // pick the first output dim that is unsharded and divisible
    const Output& out = nd.outputs[0];
    int dim = -1;
    for (size_t d = 0; d < out.shape.size(); ++d)
      if (st.out_specs[0][d].empty() && out.shape[d] % env.shape[a] == 0 && out.shape[d] >= env.shape[a]) {
        dim = static_cast<int>(d);
        break;
      }
    if (dim < 0) continue;
    st.out_specs[0][dim].push_back(a);
    st.name += " [rs@" + std::to_string(a) + " dim " + std::to_string(dim) + "]";
    st.allreduce_axes[0].clear();
    st.comm_cost = env.reduce_scatter_cost(tensor_bytes(out) / num_shards(st.out_specs[0], env) * env.shape[a], a);
    ++rewritten;
    // encode: reduce-scatter is signalled to the lowering by out_spec containing an axis that no
    // label carries; chain nodes and the state inputs they touch are re-specced by the Python side.
  }
  return rewritten;
}

}  // namespace abp
