// plan.h -- the fusion planner: the parsed op list and the plan options in; the step list, the reference counts and the weight
// schedule out.  Host-only (no CUDA header), so the plan of any model text can be inspected without a GPU (plan_summary).
#pragma once

#include "engine.h"

namespace osb {

enum StepKind { SK_SINGLE = 0, SK_ATTENTION, SK_GROUPNORM, SK_LAYERNORM, SK_GELU, SK_SILU, SK_LINEAR, SK_SDPA, SK_MHA, SK_CONV_ADD, SK_GEGLU, SK_RMSNORM, SK_ROPE, SK_GEMV_GROUP, SK_SWIGLU };
inline constexpr const char* step_kind_names[] = { "SINGLE", "ATTENTION", "GROUPNORM", "LAYERNORM", "GELU", "SILU", "LINEAR", "SDPA", "MHA", "CONV_ADD", "GEGLU", "RMSNORM", "ROPE", "GEMV_GROUP", "SWIGLU" };
static_assert(sizeof(step_kind_names) / sizeof(step_kind_names[0]) == SK_SWIGLU + 1, "one name per StepKind");

// One execution step: ops [first, first + count), run by one fused handler (or by its own handler for SK_SINGLE).  ATTENTION (count 4:
// with the scale Mul), GROUPNORM (count 7: with the SiLU tail) and GELU (count 6: with the GEGLU Mul) tell their optional tail by `count`.
struct Step {
    StepKind kind = SK_SINGLE;
    size_t first = 0, count = 1;
    int bias_in = -1;        // LINEAR: the input of the Add right after the MatMul that holds the bias (-1: no bias)
    int residual_in = -1;    // LINEAR, CONV_ADD: the input of the step's last Add that holds the residual (-1: no residual)
};

struct WeightUse { size_t op, in, bytes; };   // static weight `in` of op `op`

using UpcastRule = std::function<bool(const std::string& type, const std::string& name)>;

// The reference's m_requires_upcast: under fp16 arithmetic, an op the rule names computes in fp32.
inline bool runs_upcast(const OpDef& op, bool fp16_arithmetic, const UpcastRule& requires_upcast)
{
    return fp16_arithmetic && requires_upcast && requires_upcast(op.type, op.name);
}

bool side_branch_from_env();   // OSB_SIDE_BRANCH=1, read once per process

// everything the planner reads
struct PlanOptions {
    bool fuse_nodes = true, fuse_attention = false, sdpa_rewrite = false;
    bool uint8_arithmetic = false, uint8_qdq = false, fp16_arithmetic = false;
    // opt-in: inside the captured UNet graph the 112 latent-independent steps on a side branch did not shorten the critical path in practice
    bool side_branch = side_branch_from_env();
    UpcastRule requires_upcast;
    std::vector<std::string> extra_outputs;
};

struct Plan {
    std::vector<Step> steps;
    std::map<std::string, int> uses;                   // static consumer counts, extra outputs included: the initial reference counts
    std::vector<std::vector<WeightUse>> step_weights;  // per step, in graph order
    size_t largest_step_bytes = 0;                     // the largest step's weights, each rounded up to 256 bytes: sizes the weight ring
    std::vector<long> stats_consumer;                  // per step: the GroupNorm step that takes its statistics from this step's output (-1: none)
    // Side branch (side_branch and fuse_nodes only; empty when nothing qualifies): steps that do not depend on the primary graph input -- the
    // time-embedding MLP and every resnet's time_emb_proj, the cross-attention K / V projections of the text context.
    std::vector<char> is_side;                         // per step
    std::vector<char> kv_side;                         // per step: an SK_MHA step whose K / V inputs are side tensors
    std::vector<std::vector<size_t>> side_deps;        // per main step: side steps whose outputs it reads
};

Plan make_plan(const std::vector<OpDef>& ops, const PlanOptions& o);

// Parse `model_text` and plan it: one line per execution step ("KIND ops first_op_type first_op_name" plus the [side], [kv-side] and
// [gn-stats] marks), then a "#summary" line with the op, step and per-kind counts.  The CPU test-suite pins the planner through it.
std::string plan_summary(const std::string& model_text, bool fp16_arithmetic, bool fuse_nodes, bool fuse_attention, bool sdpa_rewrite);

inline bool is_float_weight(const TensorRef& r) { return r.present && r.wtype != DType::none && r.wtype != DType::i64; }
size_t ref_bytes(const TensorRef& r);   // payload bytes of a static weight

}  // namespace osb
