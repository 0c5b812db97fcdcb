// alpa_b200 native planner: op-graph IR, sharding strategies, cost graph, ILP assembly.
//
// This is the H100-native equivalent of the reference's C++ auto-sharding pass
// (XLA/service/spmd/auto_sharding.cc, auto_sharding_strategy.h, auto_sharding_dot_handler.cc,
// auto_sharding_util.cc).  Instead of per-HLO-opcode handlers, every op is described by an
// einsum-like *label signature*: each operand/output dim carries a label; a strategy is an
// assignment of logical-mesh axes to labels.  The reference's dot strategies fall out of that
// assignment (m->0,n->1 is "SS = SR x RS"; m->0,k->1 is "SR = SS x SR + all-reduce(1)", ...).
#pragma once
#include <cstdint>
#include <limits>
#include <string>
#include <map>
#include <tuple>
#include <vector>

namespace abp {

constexpr double kInf = 1e13;  // same sentinel magnitude the reference uses for "infinite" cost

enum LabelKind : int { kShardable = 0, kNoShard = 1 };
enum NodeKind : int { kInput = 0, kCompute = 1, kConstant = 2 };

struct Label {
  int64_t size = 1;
  int kind = kShardable;
};

// dim_axes[d] = mesh axes (major->minor) tiling tensor dim d.
using Spec = std::vector<std::vector<int>>;

struct Operand {
  int node = -1;
  int out_idx = 0;
  std::vector<int> labels;  // per dim; -1 = broadcast (operand has size 1 there) -> replicated
};

struct Output {
  std::vector<int64_t> shape;
  std::vector<int> labels;  // per dim; -1 = size-1 dim that is never sharded
  int dtype_bytes = 4;
  // operand indices this output is computed from; empty = all.  A sharded label that is missing from the output
  // makes it a partial sum only if one of THESE operands carries the label (convolution_backward's grad_bias does
  // not depend on the input activations, so sharding the input channels leaves it complete).
  std::vector<int> depends;
};

struct Strategy {
  std::string name;
  std::vector<std::vector<int>> label_axes;  // per label
  std::vector<Spec> out_specs;               // per output
  std::vector<Spec> in_specs;                // per operand
  std::vector<std::vector<int>> allreduce_axes;  // per output: mesh axes holding partial sums
  double compute_cost = 0, comm_cost = 0, memory_cost = 0;
};

struct Node {
  int id = -1;
  std::string name;
  int kind = kCompute;
  std::vector<Label> labels;
  std::vector<Operand> operands;
  std::vector<Output> outputs;
  int follow = -1;            // operand index whose producer this node follows; -1 = leader
  int batch_label = -1;       // label carrying the batch dim (inferred), -1 = none
  bool is_parameter = false;  // trainable state (inputs not listed in batch_argnums)
  bool is_batch_input = false;
  double flops = 0;
  // operands this op updates in place (fused optimizer, running statistics): their layout must be the producer's --
  // a re-laid-out copy would swallow the update
  std::vector<int> mutated_operands;
  // false: the outputs are views / aliases of operands (getitem, reshape, in-place updates): no new memory
  bool allocates = true;
  // filled by the planner
  std::vector<Strategy> strategies;
  int chosen = -1;
};

struct MeshEnv {
  std::vector<int> shape;           // logical mesh shape (1-D or 2-D)
  std::vector<double> alpha, beta;  // per axis
  double all_gather_cost(double bytes, int axis) const;
  double all_reduce_cost(double bytes, int axis) const;
  double reduce_scatter_cost(double bytes, int axis) const;
  double all_to_all_cost(double bytes, int axis) const;
  int num_devices() const {
    int n = 1;
    for (int s : shape) n *= s;
    return n;
  }
};

struct Options {
  bool force_data_parallel = false;
  int force_batch_dim_to_mesh_dim = -1;
  bool allow_all_gather = true;
  bool allow_all_to_all = true;
  bool allow_replicated_parameters = true;
  bool allow_mixed_mesh_shape = false;  // allow one tensor dim tiled by both mesh axes
  bool prefer_reduce_scatter = false;
  bool force_zero_stage_3 = false;
  double memory_budget_per_device = -1;  // bytes; <0 = unlimited
  // heavy ops (matmul / conv) may be computed with duplicated FLOPs on part of the mesh at a compute-cost penalty
  // (reference: RecomputeSplitBothContract + allow_recompute_heavy_op, auto_sharding_dot_handler.cc:250)
  bool allow_recompute_heavy_op = false;
  // "", "shard-largest", "shard-first", "shard-last": fix the layout of every program input by a rule of thumb and
  // let the solver propagate it (reference: AnnotateShardingWithSimpleHeuristic, auto_sharding_util.cc:2017)
  std::string force_simple_heuristic;
};

// The serialized ILP, same structure as the reference's solver call
// (alpa/shard_parallel/auto_sharding.py:617-629): N nodes, per-node strategy counts and costs,
// E edges with |s_i| x |s_j| resharding cost matrices, optional alias pairs and liveness sets.
struct IlpProblem {
  int N = 0;
  std::vector<int> s_len;                 // strategies per (merged) node
  std::vector<int> leader_node;           // graph node id of each ILP node
  std::vector<std::vector<double>> c;     // node cost (comm + compute) per strategy
  std::vector<std::vector<double>> m;     // memory per strategy
  std::vector<std::pair<int, int>> edges; // ILP node indices
  std::vector<std::vector<double>> r;     // row-major |s_i| x |s_j|
  std::vector<std::pair<int, int>> alias; // ILP node pairs that must pick the same strategy index
  // Memory constraint (reference: sum_i m[i][j] s[i][j] <= M for every time step over the live set,
  // alpa/shard_parallel/auto_sharding.py:773-779 with liveness from auto_sharding.cc:2196-2216).  Row t lists
  // (ILP node, strategy, bytes) of every value alive at program point `mem_time[t]`; followers are charged to their
  // leader's variables.  Only rows that can exceed the budget are kept.
  double memory_budget = -1;
  std::vector<int> mem_time;
  std::vector<std::vector<std::tuple<int, int, double>>> mem_rows;
  double min_peak_memory = 0;             // peak over time of the cheapest layout of each live value (lower bound)
  // cost-graph simplification record (simplify / expand): eliminated ILP nodes in elimination order
  struct Elim {
    int node = -1;                  // eliminated node (index in the ORIGINAL problem)
    int a = -1, b = -1;             // its neighbours (original indices); b = -1 for a degree-1 / degree-0 node
    std::vector<int> choice;        // best own strategy per (ka) or per (ka * s_len[b] + kb)
  };
  std::vector<Elim> eliminated;
  std::vector<int> kept;                  // reduced node -> original node
  int original_N = 0;
  std::vector<int> original_s_len;
  double constant = 0;                    // objective part fixed by eliminated isolated nodes
};

class Graph {
 public:
  int add_node(Node n);
  Node& node(int i) { return nodes_[i]; }
  const Node& node(int i) const { return nodes_[i]; }
  int size() const { return static_cast<int>(nodes_.size()); }

  void infer_batch_labels();
  void build_strategies(const MeshEnv& env, const Options& opt);
  IlpProblem build_ilp(const MeshEnv& env, const Options& opt);
  // Solve with the built-in solver (exact on forests after merging, iterated local search otherwise).
  std::vector<int> solve_builtin(const IlpProblem& p, double* objective) const;
  // Apply ILP node choices: sets `chosen` on every node (followers inherit their leader's index).
  void apply_solution(const IlpProblem& p, const std::vector<int>& s_val);
  // Exact cost-graph simplification (the role of CostGraph::Simplify, auto_sharding_strategy.h:900): nodes with at
  // most two neighbours are eliminated by min-plus folding (degree 0/1 into the neighbour's node cost, degree 2
  // into an edge between the neighbours), repeatedly.  Chains of element-wise ops, views and per-parameter optimizer
  // groups disappear; the ILP keeps only the branching structure.  `expand` maps a solution of the reduced problem
  // back.  Nodes that appear in memory rows are never eliminated.
  IlpProblem simplify(const IlpProblem& p) const;
  std::vector<int> expand(const IlpProblem& reduced, const std::vector<int>& s_reduced) const;
  // Peak memory (bytes per device) of a full assignment, over the exported memory rows' program points.
  double peak_memory(const IlpProblem& p, const std::vector<int>& s_val) const;
  double resharding_cost(const Output& t, const Spec& src, const Spec& dst, const MeshEnv& env,
                         const Options& opt) const;
  // ZeRO: turn gradient all-reduces feeding sharded-able optimizer updates into reduce-scatters.
  int rewrite_reduce_scatter(const MeshEnv& env, const Options& opt);

  std::vector<int> leader_of;        // node -> leader node id (after build_ilp)
  std::vector<std::pair<int, int>> alias_pairs;  // (input node, producing node/out) donation aliases
  // manual sharding: (node, out_idx, spec) -- strategies whose output spec differs are forbidden
  std::vector<std::tuple<int, int, Spec>> pinned_outputs;

 private:
  std::vector<Node> nodes_;
};

// ---------------- inter-op planner ----------------
// ---------------------------------------------------------------------------------------------
// Cost model over lowered programs (cost_model.cpp; reference: XLA/service/gpu/gpu_cost_model.cc)
// ---------------------------------------------------------------------------------------------
enum CostKind : int { kDot = 0, kAllReduce = 1, kAllGather = 2, kReduceScatter = 3, kAllToAll = 4, kP2P = 5 };

struct CostTables {
  // (kind, group size) -> sorted [(size, seconds)]; size = bytes for collectives, FLOPs for kDot
  std::map<std::pair<int, int>, std::vector<std::pair<double, double>>> tables;
  double flops_per_second = 1.4e15, hbm_bytes_per_second = 6.5e12, link_bytes_per_second = 7.7e11;
  double allreduce_bus_bytes_per_second = 7.25e11, latency = 12e-6, launch_overhead = 2e-6;

  static double interp(const std::vector<std::pair<double, double>>& table, double size);
  void add(int kind, int group_size, double size, double seconds);
  double collective_seconds(int kind, int group_size, double bytes) const;
  double gemm_seconds(double flops) const;
  double estimate(const std::vector<std::pair<double, double>>& ops,
                  const std::vector<std::tuple<int, int, double>>& collectives, double overlap) const;
};

// Reference: alpa/pipeline_parallel/stage_construction.py:234-340 (training_dp / training_dp_impl)
struct StageDpResult {
  double cost = kInf;
  // (layer_start, layer_end_exclusive, submesh_choice, autosharding_choice)
  std::vector<std::vector<int>> stages;
};
StageDpResult training_dp(int num_layers, int num_devices, int num_microbatches,
                          const std::vector<std::pair<int, int>>& submesh_choices,
                          int num_autosharding_configs,
                          const std::vector<double>& compute_cost,       // [L][L][S][C]
                          const std::vector<int>& max_n_succ_stages);     // [L][L][S][C]
StageDpResult inference_dp(int num_layers, int num_devices,
                           const std::vector<std::pair<int, int>>& submesh_choices,
                           int num_autosharding_configs, const std::vector<double>& compute_cost);

// Reference: alpa/pipeline_parallel/layer_construction.py:342-457 (cluster_jaxpr_by_cost)
// Returns layer id per op (contiguous, non-decreasing).
std::vector<int> cluster_ops_by_cost(const std::vector<double>& op_flops,
                                     const std::vector<std::vector<double>>& cut_bytes_hint,
                                     const std::vector<double>& cut_cost,  // cost of cutting after op i
                                     int layer_num, double eps);

}  // namespace abp
