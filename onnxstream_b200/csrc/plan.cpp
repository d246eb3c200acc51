// plan.cpp -- the fusion planner (see plan.h): pattern matchers over the parsed op list, the GroupNorm-statistics pairing, the per-step
// weight schedule and the side-branch analysis.
#include "plan.h"

#include <algorithm>
#include <cstdlib>
#include <initializer_list>

namespace osb {

size_t ref_bytes(const TensorRef& r)
{
    size_t n = 1; for (auto d : r.shape) n *= (size_t)d;
    return n * dtype_size(r.wtype);
}

bool side_branch_from_env()
{
    static const bool on = [] { const char* e = getenv("OSB_SIDE_BRANCH"); return e && e[0] == '1'; }();
    return on;
}

namespace {

bool is_scalar_weight(const TensorRef& r) { return is_float_weight(r) && r.shape.empty(); }
bool softmax_last_axis(const OpDef& sm) { return sm.attrs.size() == 1 && sm.attrs[0].first == "axis" && sm.attrs[0].second == "-1"; }

// Each matcher returns the number of ops of its pattern starting at op i (0: no match) and sets the operands its step kind names.
struct Planner {
    const std::vector<OpDef>& ops;
    const PlanOptions& o;
    const std::map<std::string, int>& uses;

    bool upcast(const OpDef& op) const { return runs_upcast(op, o.fp16_arithmetic, o.requires_upcast); }
    // ops i, i + 1, ... have these types
    bool types_at(size_t i, std::initializer_list<const char*> seq) const
    {
        if (i + seq.size() > ops.size()) return false;
        for (const char* t : seq) if (ops[i++].type != t) return false;
        return true;
    }
    // activation `name` has exactly n consumers
    bool used(const std::string& name, int n) const
    {
        auto it = uses.find(name);
        return it != uses.end() && it->second == n;
    }
    // out[0] of op a is the input `idx` of op b and has no other consumer
    bool feeds(const OpDef& a, const OpDef& b, size_t idx) const
    {
        return a.out.size() == 1 && idx < b.in.size() && b.in[idx].present && b.in[idx].wtype == DType::none &&
               b.in[idx].name == a.out[0].name && used(a.out[0].name, 1);
    }

    size_t attention(size_t i, Step&) const
    {
        if (!(o.fuse_attention || o.fuse_nodes) || o.uint8_arithmetic) return 0;
        bool with_scale = types_at(i, { "MatMul", "Mul", "Softmax", "MatMul" });
        if (!with_scale && !types_at(i, { "MatMul", "Softmax", "MatMul" })) return 0;
        const OpDef& mm0 = ops[i];
        const OpDef* mul = with_scale ? &ops[i + 1] : nullptr;
        const OpDef& sm = ops[i + (with_scale ? 2 : 1)];
        const OpDef& mm1 = ops[i + (with_scale ? 3 : 2)];
        if (mm0.in.size() != 2 || mm0.out.size() != 1 || sm.in.size() != 1 || sm.out.size() != 1 || mm1.in.size() != 2 || mm1.out.size() != 1) return 0;
        if (mm0.in[0].wtype != DType::none || mm0.in[1].wtype != DType::none || mm1.in[1].wtype != DType::none) return 0;
        if (!softmax_last_axis(sm)) return 0;
        if (mul && (mul->in.size() != 2 || mul->out.size() != 1 || !is_scalar_weight(mul->in[1]))) return 0;
        if (!feeds(mm0, mul ? *mul : sm, 0)) return 0;
        if (mul && !feeds(*mul, sm, 0)) return 0;
        if (!feeds(sm, mm1, 0)) return 0;
        // shapes the reference's branch accepts: 3-D or 4-D with a leading 1 (src/onnxstream.cpp:6707-6724)
        auto& qs = mm0.in[0].shape; auto& ks = mm0.in[1].shape; auto& vs = mm1.in[1].shape;
        if (qs.size() != ks.size() || qs.size() != vs.size()) return 0;
        if (!(qs.size() == 3 || (qs.size() == 4 && qs[0] == 1 && ks[0] == 1 && vs[0] == 1))) return 0;
        return with_scale ? 4 : 3;
    }

    // Whole multi-head attention of the diffusers export (SURVEY Appendix C.1): three bias-free projections, the
    // Reshape/Transpose/Reshape head split of each (K additionally pre-transposed), MatMul-Mul-Softmax-MatMul, and the head
    // merge -- 20 ops.  Executed as 3 projection GEMMs + strided per-head GEMMs reading the projections in place.
    size_t mha(size_t i, Step&) const
    {
        if (!types_at(i, { "MatMul", "Reshape", "Transpose", "Reshape", "MatMul", "Reshape", "Transpose", "Reshape", "Transpose",
                           "MatMul", "Reshape", "Transpose", "Reshape", "MatMul", "Mul", "Softmax", "MatMul", "Reshape", "Transpose", "Reshape" })) return 0;
        for (int k = 0; k < 20; k++) if (ops[i + k].out.size() != 1 || upcast(ops[i + k])) return 0;
        auto lin = [&](const OpDef& o) { return o.in.size() == 2 && o.in[0].present && o.in[0].wtype == DType::none && is_float_weight(o.in[1]) && o.in[1].shape.size() == 2 && o.in[0].shape.size() == 3 && o.in[0].shape[0] == 1; };
        if (!lin(ops[i]) || !lin(ops[i + 4]) || !lin(ops[i + 9])) return 0;
        auto perm = [&](const OpDef& o, const char* p) { auto a = o.attr("perm"); return a && *a == p && o.in.size() == 1; };
        if (!perm(ops[i + 2], "0,2,1,3") || !perm(ops[i + 6], "0,2,1,3") || !perm(ops[i + 11], "0,2,1,3") || !perm(ops[i + 18], "0,2,1,3") || !perm(ops[i + 8], "0,2,1")) return 0;
        // chains
        if (!feeds(ops[i], ops[i + 1], 0) || !feeds(ops[i + 1], ops[i + 2], 0) || !feeds(ops[i + 2], ops[i + 3], 0)) return 0;
        if (!feeds(ops[i + 4], ops[i + 5], 0) || !feeds(ops[i + 5], ops[i + 6], 0) || !feeds(ops[i + 6], ops[i + 7], 0) || !feeds(ops[i + 7], ops[i + 8], 0)) return 0;
        if (!feeds(ops[i + 9], ops[i + 10], 0) || !feeds(ops[i + 10], ops[i + 11], 0) || !feeds(ops[i + 11], ops[i + 12], 0)) return 0;
        if (ops[i + 13].in.size() != 2 || !feeds(ops[i + 3], ops[i + 13], 0) || !feeds(ops[i + 8], ops[i + 13], 1)) return 0;
        if (ops[i + 14].in.size() != 2 || !feeds(ops[i + 13], ops[i + 14], 0) || !is_scalar_weight(ops[i + 14].in[1])) return 0;
        auto& sm = ops[i + 15];
        if (sm.in.size() != 1 || !feeds(ops[i + 14], sm, 0) || !softmax_last_axis(sm)) return 0;
        if (ops[i + 16].in.size() != 2 || !feeds(sm, ops[i + 16], 0) || !feeds(ops[i + 12], ops[i + 16], 1)) return 0;
        if (!feeds(ops[i + 16], ops[i + 17], 0) || !feeds(ops[i + 17], ops[i + 18], 0) || !feeds(ops[i + 18], ops[i + 19], 0)) return 0;
        // shapes
        auto& qs = ops[i + 3].out[0].shape; auto& kts = ops[i + 8].out[0].shape; auto& vs = ops[i + 12].out[0].shape; auto& os = ops[i + 19].out[0].shape;
        auto& q4 = ops[i + 1].out[0].shape; auto& k4 = ops[i + 5].out[0].shape; auto& v4 = ops[i + 10].out[0].shape; auto& o4 = ops[i + 17].out[0].shape;
        if (qs.size() != 3 || kts.size() != 3 || vs.size() != 3 || os.size() != 3 || q4.size() != 4 || k4.size() != 4 || v4.size() != 4 || o4.size() != 4) return 0;
        int64_t h = qs[0], T = qs[1], d = qs[2], Tk = kts[2];
        if (kts[0] != h || kts[1] != d || vs[0] != h || vs[1] != Tk || vs[2] != d || d % 8) return 0;
        int64_t C = h * d;
        if (ops[i].out[0].shape != std::vector<int64_t>{ 1, T, C } || ops[i + 4].out[0].shape != std::vector<int64_t>{ 1, Tk, C } || ops[i + 9].out[0].shape != std::vector<int64_t>{ 1, Tk, C }) return 0;
        if (q4 != std::vector<int64_t>{ 1, T, h, d } || k4 != std::vector<int64_t>{ 1, Tk, h, d } || v4 != std::vector<int64_t>{ 1, Tk, h, d } || o4 != std::vector<int64_t>{ 1, h, T, d }) return 0;
        if (os != std::vector<int64_t>{ 1, T, C }) return 0;
        for (int k : { 1, 3, 5, 7, 10, 12, 17, 19 }) if (ops[i + k].in.size() != 2 || ops[i + k].in[1].wtype != DType::i64) return 0;
        return 20;
    }

    // Transpose(K) -> MatMul(Q, Kt) -> Div(s) -> Add(mask) -> Softmax(-1) -> MatMul(P, V)   (src/onnxstream.cpp:3643-3695)
    size_t sdpa(size_t i, Step&) const
    {
        if (!o.sdpa_rewrite || o.uint8_arithmetic) return 0;
        if (!types_at(i, { "Transpose", "MatMul", "Div", "Add", "Softmax", "MatMul" })) return 0;
        const OpDef &tr = ops[i], &mm0 = ops[i + 1], &dv = ops[i + 2], &ad = ops[i + 3], &sm = ops[i + 4], &mm1 = ops[i + 5];
        if (tr.in.size() != 1 || mm0.in.size() != 2 || dv.in.size() != 2 || ad.in.size() != 2 || sm.in.size() != 1 || mm1.in.size() != 2) return 0;
        if (!softmax_last_axis(sm)) return 0;
        if (!feeds(tr, mm0, 1) || !feeds(mm0, dv, 0) || !feeds(dv, ad, 0) || !feeds(ad, sm, 0) || !feeds(sm, mm1, 0)) return 0;
        return 6;
    }

    size_t groupnorm(size_t i, Step&) const
    {
        if (!types_at(i, { "Reshape", "InstanceNormalization", "Reshape", "Mul", "Add" })) return 0;
        const OpDef &r0 = ops[i], &inrm = ops[i + 1], &r1 = ops[i + 2], &mul = ops[i + 3], &add = ops[i + 4];
        if (r0.in.size() != 2 || inrm.in.size() != 3 || r1.in.size() != 2 || mul.in.size() != 2 || add.in.size() != 2) return 0;
        if (r0.in[0].wtype != DType::none || r0.in[0].shape.size() != 4 || r0.in[0].shape[0] != 1) return 0;
        if (r0.out[0].shape.size() != 3 || r0.out[0].shape[0] != 1) return 0;
        if (!feeds(r0, inrm, 0) || !feeds(inrm, r1, 0) || !feeds(r1, mul, 0) || !feeds(mul, add, 0)) return 0;
        if (r1.out[0].shape != r0.in[0].shape) return 0;
        int64_t C = r0.in[0].shape[1], G = r0.out[0].shape[1];
        if (G <= 0 || C % G) return 0;
        auto chan_w = [&](const TensorRef& r) {
            if (!is_float_weight(r)) return false;
            int64_t n = 1; for (auto d : r.shape) n *= d;
            if (n != C) return false;
            // [C,1,1] or [1,C,1,1] or [C]
            if (r.shape.size() == 3) return r.shape[0] == C;
            if (r.shape.size() == 4) return r.shape[1] == C;
            return false;
        };
        if (!chan_w(mul.in[1]) || !chan_w(add.in[1])) return 0;
        if (!is_float_weight(inrm.in[1]) || !is_float_weight(inrm.in[2])) return 0;
        if (G > 64) return 0;  // per-group affine is read through the 64-element host mirror
        if (types_at(i + 5, { "Sigmoid", "Mul" })) {   // SiLU tail
            const OpDef &sg = ops[i + 5], &m2 = ops[i + 6];
            if (sg.in.size() == 1 && m2.in.size() == 2 && used(add.out[0].name, 2) && sg.in[0].name == add.out[0].name &&
                feeds(sg, m2, 1) && m2.in[0].name == add.out[0].name && m2.in[0].wtype == DType::none) return 7;
        }
        return 5;
    }

    size_t layernorm(size_t i, Step&) const
    {
        if (!types_at(i, { "ReduceMean", "Sub", "Pow", "ReduceMean", "Add", "Sqrt", "Div", "Mul", "Add" })) return 0;
        const OpDef &rm0 = ops[i], &sub = ops[i + 1], &pw = ops[i + 2], &rm1 = ops[i + 3], &ade = ops[i + 4], &sq = ops[i + 5], &dv = ops[i + 6], &mul = ops[i + 7], &add = ops[i + 8];
        auto last_axis = [](const OpDef& o) { auto a = o.attr("axes"); auto k = o.attr("keepdims"); return a && (*a == "-1") && (!k || *k == "1"); };
        if (!last_axis(rm0) || !last_axis(rm1)) return 0;
        if (rm0.in.size() != 1 || rm0.in[0].wtype != DType::none) return 0;
        const std::string& x = rm0.in[0].name;
        if (sub.in.size() != 2 || sub.in[0].name != x || sub.in[0].wtype != DType::none || !feeds(rm0, sub, 1)) return 0;
        const std::string& d = sub.out[0].name;
        if (!used(d, 2)) return 0;
        if (pw.in.size() != 2 || pw.in[0].name != d || !is_scalar_weight(pw.in[1])) return 0;
        if (!feeds(pw, rm1, 0) || !feeds(rm1, ade, 0) || ade.in.size() != 2 || !is_scalar_weight(ade.in[1])) return 0;
        if (!feeds(ade, sq, 0)) return 0;
        if (dv.in.size() != 2 || dv.in[0].name != d || dv.in[0].wtype != DType::none || !feeds(sq, dv, 1)) return 0;
        if (!feeds(dv, mul, 0) || mul.in.size() != 2 || !is_float_weight(mul.in[1])) return 0;
        if (!feeds(mul, add, 0) || add.in.size() != 2 || !is_float_weight(add.in[1])) return 0;
        int64_t C = rm0.in[0].shape.empty() ? 0 : rm0.in[0].shape.back();
        auto vecC = [&](const TensorRef& r) { return r.shape.size() == 1 && r.shape[0] == C; };
        if (!vecC(mul.in[1]) || !vecC(add.in[1])) return 0;
        return 9;
    }

    size_t gelu(size_t i, Step&) const
    {
        if (!types_at(i, { "Div", "Erf", "Add", "Mul", "Mul" })) return 0;
        const OpDef &dv = ops[i], &erf = ops[i + 1], &ad = ops[i + 2], &m0 = ops[i + 3], &m1 = ops[i + 4];
        if (dv.in.size() != 2 || dv.in[0].wtype != DType::none || !is_scalar_weight(dv.in[1])) return 0;
        const std::string& x = dv.in[0].name;
        if (!feeds(dv, erf, 0) || !feeds(erf, ad, 0) || ad.in.size() != 2 || !is_scalar_weight(ad.in[1])) return 0;
        if (m0.in.size() != 2 || m0.in[0].name != x || m0.in[0].wtype != DType::none || !feeds(ad, m0, 1)) return 0;
        if (!feeds(m0, m1, 0) || m1.in.size() != 2 || !is_scalar_weight(m1.in[1])) return 0;
        // GEGLU: Mul(a, gelu(gate)) right after
        if (types_at(i + 5, { "Mul" })) {
            const OpDef& g = ops[i + 5];
            if (g.in.size() == 2 && g.in[0].wtype == DType::none && feeds(m1, g, 1) && g.in[0].shape == m1.out[0].shape) return 6;
        }
        return 5;
    }

    // GEGLU gate: Slice(x, 0:inner), Slice(x, inner:2*inner) on the last axis, gelu_erf of the second, Mul -- one kernel, no
    // materialised halves.  The slice bounds are int64 weights, so they are verified when the step executes (fused_geglu falls
    // back to the op-by-op path if they are not the two halves).  Led by MatMul(x, W[K, 2 inner]) -> Add(bias) whose result only the
    // two Slices read, the step takes those too (10 ops): the gate runs in the GEMM epilogue where fused_geglu can launch it so.
    size_t geglu(size_t i, Step& s) const
    {
        if (types_at(i, { "MatMul", "Add" })) {
            Step lin;
            if (linear(i, lin) != 2 || lin.bias_in < 0 || upcast(ops[i])) return 0;
            const std::string& x = ops[i + 1].out[0].name;
            if (!used(x, 2) || geglu(i + 2, s) != 8 || ops[i + 2].in[0].name != x) return 0;
            s.bias_in = lin.bias_in;
            return 10;
        }
        if (!types_at(i, { "Slice", "Slice" })) return 0;
        const OpDef &s0 = ops[i], &s1 = ops[i + 1];
        if (s0.in.size() != 5 || s1.in.size() != 5 || s0.out.size() != 1 || s1.out.size() != 1) return 0;
        if (s0.in[0].wtype != DType::none || s1.in[0].wtype != DType::none || s0.in[0].name != s1.in[0].name) return 0;
        for (int k = 1; k < 5; k++) if (!s0.in[k].present || s0.in[k].wtype != DType::i64 || !s1.in[k].present || s1.in[k].wtype != DType::i64) return 0;
        if (s0.out[0].shape != s1.out[0].shape || s0.out[0].shape.empty()) return 0;
        for (auto& name : o.extra_outputs) if (name == s0.out[0].name || name == s1.out[0].name) return 0;
        if (gelu(i + 2, s) != 6) return 0;
        const OpDef &dv = ops[i + 2], &m0 = ops[i + 5], &gm = ops[i + 7];
        // gate half: read by Div and by the first Mul of the chain, nothing else; value half: read by the last Mul only
        if (!used(s1.out[0].name, 2) || !used(s0.out[0].name, 1)) return 0;
        if (dv.in[0].name != s1.out[0].name || m0.in[0].name != s1.out[0].name || gm.in[0].name != s0.out[0].name) return 0;
        return 8;
    }

    size_t silu(size_t i, Step&) const
    {
        if (!types_at(i, { "Sigmoid", "Mul" })) return 0;
        const OpDef &sg = ops[i], &m = ops[i + 1];
        if (sg.in.size() != 1 || sg.in[0].wtype != DType::none || m.in.size() != 2) return 0;
        if (m.in[0].name != sg.in[0].name || m.in[0].wtype != DType::none || !feeds(sg, m, 1)) return 0;
        return 2;
    }

    // decode-shaped MatMul: activation with <= 8 rows times a static 2-D weight
    bool is_gemv_matmul(const OpDef& mm) const
    {
        if (mm.type != "MatMul" || mm.in.size() != 2 || mm.out.size() != 1 || mm.in[0].wtype != DType::none || !is_float_weight(mm.in[1]) || mm.in[1].shape.size() != 2) return false;
        const auto& as = mm.in[0].shape;
        if (as.empty() || as.back() != mm.in[1].shape[0]) return false;
        int64_t rows = 1; for (size_t k = 0; k + 1 < as.size(); k++) rows *= as[k];
        return rows >= 1 && rows <= 8 && !upcast(mm);
    }
    // 2 or 3 consecutive decode MatMuls of the same activation (q / k / v projections): one grouped GEMV launch
    size_t gemv_group(size_t i, Step&) const
    {
        size_t n = 0;
        while (n < 3 && i + n < ops.size()) {
            const OpDef& mm = ops[i + n];
            if (!is_gemv_matmul(mm)) break;
            if (n && (mm.in[0].name != ops[i].in[0].name || mm.in[1].shape[0] != ops[i].in[1].shape[0] || (mm.in[1].wtype == DType::u8) != (ops[i].in[1].wtype == DType::u8))) break;
            n++;
        }
        // leave the last MatMul to the Linear matcher when an Add takes its result (bias / residual epilogue)
        if (n >= 2 && types_at(i + n, { "Add" }))
            for (auto& r : ops[i + n].in) if (r.present && r.wtype == DType::none && r.name == ops[i + n - 1].out[0].name) { n--; break; }
        return n >= 2 ? n : 0;
    }
    // gated MLP of llm.cpp's graphs: MatMul(x, Wg) -> Sigmoid -> Mul (SiLU) -> MatMul(x, Wu) -> Mul: one grouped GEMV + one elementwise pass
    size_t swiglu(size_t i, Step&) const
    {
        if (!types_at(i, { "MatMul", "Sigmoid", "Mul", "MatMul", "Mul" })) return 0;
        const OpDef &g = ops[i], &sg = ops[i + 1], &m1 = ops[i + 2], &u = ops[i + 3], &m2 = ops[i + 4];
        if (!is_gemv_matmul(g) || !is_gemv_matmul(u)) return 0;
        if (g.in[0].name != u.in[0].name || g.in[1].shape != u.in[1].shape || (g.in[1].wtype == DType::u8) != (u.in[1].wtype == DType::u8)) return 0;
        if (upcast(sg) || upcast(m1) || upcast(m2) || m1.in.size() != 2 || m2.in.size() != 2) return 0;
        const std::string& gn = g.out[0].name;
        if (!used(gn, 2)) return 0;                       // the gate feeds Sigmoid and the SiLU Mul only
        if (sg.in.size() != 1 || sg.in[0].name != gn || sg.in[0].wtype != DType::none) return 0;
        bool silu = false;
        for (int k = 0; k < 2; k++) if (m1.in[k].wtype == DType::none && m1.in[k].name == gn && feeds(sg, m1, 1 - k)) silu = true;
        if (!silu) return 0;
        bool gate = false;
        for (int k = 0; k < 2; k++) if (feeds(m1, m2, k) && feeds(u, m2, 1 - k)) gate = true;
        return gate ? 5 : 0;
    }

    // RMSNorm as llm.cpp's graphs spell it: Pow(x, 2) -> ReduceMean(-1) -> Add(eps) -> Sqrt -> Div(1, .) -> Mul(x, .) -> Mul(w, .)
    size_t rmsnorm(size_t i, Step&) const
    {
        if (!types_at(i, { "Pow", "ReduceMean", "Add", "Sqrt", "Div", "Mul", "Mul" })) return 0;
        const OpDef &pw = ops[i], &rm = ops[i + 1], &ad = ops[i + 2], &sq = ops[i + 3], &dv = ops[i + 4], &m1 = ops[i + 5], &m2 = ops[i + 6];
        if (pw.in.size() != 2 || pw.in[0].wtype != DType::none || !is_scalar_weight(pw.in[1])) return 0;
        auto a = rm.attr("axes"); auto kd = rm.attr("keepdims");
        if (!a || *a != "-1" || (kd && *kd != "1")) return 0;
        if (!feeds(pw, rm, 0) || ad.in.size() != 2 || !feeds(rm, ad, 0) || !is_scalar_weight(ad.in[1]) || !feeds(ad, sq, 0)) return 0;
        if (dv.in.size() != 2 || !is_scalar_weight(dv.in[0]) || !feeds(sq, dv, 1)) return 0;
        const std::string& x = pw.in[0].name;
        if (m1.in.size() != 2 || m2.in.size() != 2) return 0;
        int xi = -1;
        for (int k = 0; k < 2; k++) if (m1.in[k].wtype == DType::none && m1.in[k].name == x && feeds(dv, m1, 1 - k)) xi = k;
        if (xi < 0) return 0;
        int wi = -1;
        const int64_t C = pw.in[0].shape.empty() ? 0 : pw.in[0].shape.back();
        for (int k = 0; k < 2; k++) if (is_float_weight(m2.in[k]) && m2.in[k].shape.size() == 1 && m2.in[k].shape[0] == C && feeds(m1, m2, 1 - k)) wi = k;
        if (wi < 0) return 0;
        // all seven ops in the same arithmetic class (the reference's m_requires_upcast looks at each op's name)
        for (int k = 1; k < 7; k++) if (upcast(ops[i + k]) != upcast(ops[i])) return 0;
        return 7;
    }

    // rotary embedding: Slice(x, first half) , Slice(x, second half), Neg, Concat(-x2, x1), Mul(x, cos), Mul(rot, sin), Add
    size_t rope(size_t i, Step&) const
    {
        if (!types_at(i, { "Slice", "Slice", "Neg", "Concat", "Mul", "Mul", "Add" })) return 0;
        const OpDef &s1 = ops[i], &s2 = ops[i + 1], &ng = ops[i + 2], &cc = ops[i + 3], &m1 = ops[i + 4], &m2 = ops[i + 5], &ad = ops[i + 6];
        if (s1.in.size() != 5 || s2.in.size() != 5 || s1.in[0].wtype != DType::none || s1.in[0].name != s2.in[0].name) return 0;
        for (int k = 1; k < 5; k++) if (s1.in[k].wtype != DType::i64 || s2.in[k].wtype != DType::i64) return 0;
        const auto& xs = s1.in[0].shape;
        if (xs.empty() || xs.back() % 2) return 0;
        const int64_t D = xs.back();
        std::vector<int64_t> hs = xs; hs.back() = D / 2;
        if (s1.out[0].shape != hs || s2.out[0].shape != hs) return 0;            // (start / end values are checked at run time)
        if (!feeds(s2, ng, 0) || cc.in.size() != 2 || !feeds(ng, cc, 0) || !feeds(s1, cc, 1)) return 0;
        auto ax = cc.attr("axis");
        if (!ax || (*ax != "-1" && *ax != std::to_string((int)xs.size() - 1))) return 0;
        const std::string& x = s1.in[0].name;
        if (m1.in.size() != 2 || m2.in.size() != 2 || ad.in.size() != 2) return 0;
        if (m1.in[0].wtype != DType::none || m1.in[0].name != x || m1.in[1].wtype != DType::none) return 0;      // Mul(x, cos)
        if (!feeds(cc, m2, 0) || m2.in[1].wtype != DType::none) return 0;                                         // Mul(rot, sin)
        if (!feeds(m1, ad, 0) || !feeds(m2, ad, 1)) return 0;
        auto n_of = [](const TensorRef& r) { int64_t n = 1; for (auto d : r.shape) n *= d; return n; };
        // cos / sin: one row shared by every head (decode), or one row per position of x [.., heads, T, D] (prefill), broadcast over the heads
        const int64_t T = xs.size() >= 2 ? xs[xs.size() - 2] : 1;
        auto table_ok = [&](const TensorRef& r) {
            const int64_t n = n_of(r);
            if (n == D) return true;
            if (n != T * D || r.shape.size() < 2 || r.shape.back() != D || r.shape[r.shape.size() - 2] != T) return false;
            for (size_t k = 0; k + 2 < r.shape.size(); k++) if (r.shape[k] != 1) return false;
            return true;
        };
        if (!table_ok(m1.in[1]) || !table_ok(m2.in[1])) return 0;
        if (!used(x, 3)) return 0;                       // x: two Slices and the Mul
        for (int k = 0; k < 7; k++) if (upcast(ops[i + k])) return 0;
        return 7;
    }

    // Conv -> Add(conv_out, other) with `other` an activation of the same shape: residual add in the conv epilogue
    // (resnet `x + conv2(...)`, transformer `proj_out(...) + residual`)
    size_t conv_add(size_t i, Step& s) const
    {
        if (!types_at(i, { "Conv", "Add" })) return 0;
        const OpDef &cv = ops[i], &ad = ops[i + 1];
        if (cv.out.size() != 1 || ad.in.size() != 2 || upcast(cv) || upcast(ad)) return 0;
        for (int k = 0; k < 2; k++)
            if (feeds(cv, ad, k) && ad.in[1 - k].present && ad.in[1 - k].wtype == DType::none && ad.in[1 - k].shape == cv.out[0].shape && cv.out[0].shape.size() == 4) {
                s.residual_in = 1 - k;
                return 2;
            }
        return 0;
    }

    // MatMul(x, W[K,N]) -> Add(bias[N], y) [-> Add(y, residual)], or MatMul -> Add(residual)
    size_t linear(size_t i, Step& s) const
    {
        if (!types_at(i, { "MatMul", "Add" })) return 0;
        const OpDef &mm = ops[i], &ad = ops[i + 1];
        if (mm.in.size() != 2 || mm.in[0].wtype != DType::none || !is_float_weight(mm.in[1]) || mm.in[1].shape.size() != 2) return 0;
        int64_t N = mm.in[1].shape[1];
        if (ad.in.size() != 2) return 0;
        int bias_in = -1;
        for (int k = 0; k < 2; k++) if (is_float_weight(ad.in[k]) && ad.in[k].shape.size() == 1 && ad.in[k].shape[0] == N) bias_in = k;
        if (bias_in < 0) {
            // MatMul -> Add(activation of the same shape): the residual add of a bias-free projection (LLM blocks) in the GEMM / GEMV epilogue
            if (upcast(mm) || upcast(ad)) return 0;
            for (int k = 0; k < 2; k++)
                if (feeds(mm, ad, k) && ad.in[1 - k].present && ad.in[1 - k].wtype == DType::none && ad.in[1 - k].shape == mm.out[0].shape && ad.in[1 - k].name != mm.out[0].name) {
                    s.residual_in = 1 - k;
                    return 2;
                }
            return 0;
        }
        if (!feeds(mm, ad, 1 - bias_in)) return 0;
        if (upcast(mm) != upcast(ad)) return 0;
        s.bias_in = bias_in;
        // optional residual
        if (types_at(i + 2, { "Add" })) {
            const OpDef& ra = ops[i + 2];
            if (ra.in.size() == 2 && !upcast(ra)) {
                for (int k = 0; k < 2; k++)
                    if (feeds(ad, ra, k) && ra.in[1 - k].present && ra.in[1 - k].wtype == DType::none && ra.in[1 - k].shape == ad.out[0].shape) {
                        s.residual_in = 1 - k;
                        return 3;
                    }
            }
        }
        return 2;
    }
};

// in priority order: the first that matches at an op claims it
const struct { StepKind kind; size_t (Planner::*match)(size_t, Step&) const; } fusions[] = {
    { SK_MHA, &Planner::mha }, { SK_SDPA, &Planner::sdpa }, { SK_ATTENTION, &Planner::attention }, { SK_GROUPNORM, &Planner::groupnorm },
    { SK_LAYERNORM, &Planner::layernorm }, { SK_GEGLU, &Planner::geglu }, { SK_GELU, &Planner::gelu }, { SK_RMSNORM, &Planner::rmsnorm },
    { SK_ROPE, &Planner::rope }, { SK_SWIGLU, &Planner::swiglu }, { SK_GEMV_GROUP, &Planner::gemv_group }, { SK_SILU, &Planner::silu },
    { SK_LINEAR, &Planner::linear }, { SK_CONV_ADD, &Planner::conv_add },
};

// Which steps are off the critical path?  primary input = the graph input that starts the LONGEST op chain to the end of the graph
// (a UNet's latent; the time step and the text context join it from the side).  A step is "side" when none of its activation
// inputs depends on the primary input, it has no int64 traffic, and it is not a graph output producer that the epilogue reads.
void plan_side_branch(const std::vector<OpDef>& ops, Plan& p)
{
    const auto& steps = p.steps;
    p.is_side.assign(steps.size(), 0);
    p.side_deps.assign(steps.size(), {});
    std::map<std::string, int> producer;           // tensor -> producing op
    for (size_t i = 0; i < ops.size(); i++) for (auto& o : ops[i].out) if (o.present) producer[o.name] = (int)i;
    // graph inputs = activation names never produced
    std::vector<std::string> inputs;
    for (auto& op : ops) for (auto& r : op.in) if (r.present && r.wtype == DType::none && !producer.count(r.name) && std::find(inputs.begin(), inputs.end(), r.name) == inputs.end()) inputs.push_back(r.name);
    if (inputs.size() < 2 || inputs.size() > 60) return;
    std::map<std::string, uint64_t> dep;           // tensor -> bitmask of graph inputs it depends on
    for (size_t k = 0; k < inputs.size(); k++) dep[inputs[k]] = 1ull << k;
    // primary input = the one whose OWN prefix (ops that depend on it alone) produces the largest tensor: a UNet's latent feeds
    // conv_in (C x H x W), while the time step and the text context only ever make vectors / a few token rows before they join it
    std::vector<int64_t> own_max(inputs.size(), 0);
    for (auto& op : ops) {
        uint64_t m = 0;
        for (auto& r : op.in) if (r.present && r.wtype == DType::none) m |= dep[r.name];
        for (auto& o : op.out) if (o.present) {
            dep[o.name] = m;
            if (m && !(m & (m - 1))) {          // exactly one input
                int k = 0; while (!((m >> k) & 1)) k++;
                int64_t n = 1; for (auto d : o.shape) n *= std::max<int64_t>(d, 1);
                own_max[k] = std::max(own_max[k], n);
            }
        }
    }
    size_t pk = 0;
    for (size_t k = 1; k < inputs.size(); k++) if (own_max[k] > own_max[pk]) pk = k;
    const uint64_t primary = 1ull << pk;
    std::map<std::string, size_t> step_of;         // tensor -> producing step
    for (size_t si = 0; si < steps.size(); si++)
        for (size_t oi = steps[si].first; oi < steps[si].first + steps[si].count; oi++) for (auto& o : ops[oi].out) if (o.present) step_of[o.name] = si;
    // (a step with no activation input at all -- constants folded by ops -- depends on nothing: it goes first too, or a side
    // consumer of its output would run before it)
    size_t n_side = 0;
    for (size_t si = 0; si < steps.size(); si++) {
        bool side = true;
        for (size_t oi = steps[si].first; oi < steps[si].first + steps[si].count && side; oi++) {
            for (auto& r : ops[oi].in) if (r.present && r.wtype == DType::none && (dep[r.name] & primary)) side = false;
            for (auto& o : ops[oi].out) if (o.present && p.uses.find(o.name) == p.uses.end()) side = false;   // a graph output
        }
        if (side) { p.is_side[si] = 1; n_side++; }
    }
    p.kv_side.assign(steps.size(), 0);
    for (size_t si = 0; si < steps.size(); si++)
        if (steps[si].kind == SK_MHA) {
            size_t i = steps[si].first;
            auto side_in = [&](size_t oi) { const TensorRef& r = ops[oi].in[0]; return r.present && r.wtype == DType::none && !(dep[r.name] & primary); };
            if (side_in(i + 4) && side_in(i + 9) && !side_in(i)) { p.kv_side[si] = 1; n_side++; }
        }
    if (n_side == 0) { p.is_side.clear(); p.kv_side.clear(); return; }
    for (size_t si = 0; si < steps.size(); si++) {
        if (p.is_side[si]) continue;
        auto& deps = p.side_deps[si];
        for (size_t oi = steps[si].first; oi < steps[si].first + steps[si].count; oi++)
            for (auto& r : ops[oi].in) if (r.present && r.wtype == DType::none) {
                auto it = step_of.find(r.name);
                if (it != step_of.end() && p.is_side[it->second] && std::find(deps.begin(), deps.end(), it->second) == deps.end()) deps.push_back(it->second);
            }
    }
}

}  // namespace

Plan make_plan(const std::vector<OpDef>& ops, const PlanOptions& o)
{
    Plan p;
    for (auto& op : ops) for (auto& r : op.in) if (r.present && r.wtype == DType::none) p.uses[r.name]++;
    for (auto& n : o.extra_outputs) p.uses[n]++;
    const Planner P{ ops, o, p.uses };
    // uint8 modes and fuse_nodes off run op by op; the two attention rewrites have guards of their own
    const bool fuse = o.fuse_nodes && !o.uint8_arithmetic && !o.uint8_qdq;
    for (size_t i = 0; i < ops.size();) {
        Step s; s.first = i;
        for (auto& f : fusions) {
            if (!fuse && f.kind != SK_SDPA && f.kind != SK_ATTENTION) continue;
            if (size_t n = (P.*f.match)(i, s)) { s.kind = f.kind; s.count = n; break; }
        }
        p.steps.push_back(s);
        i += s.count;
    }
    const auto& steps = p.steps;
    // GroupNorm steps whose input is produced by the step right before them (conv / conv + residual / per-channel Add / Concat): that
    // producer gathers the statistics (fuse_nodes only; the op list is unchanged, only the GroupNorm's stats pass disappears)
    p.stats_consumer.assign(steps.size(), -1);
    for (size_t j = 1; j < steps.size(); j++) {
        if (steps[j].kind != SK_GROUPNORM) continue;
        const Step& pstep = steps[j - 1];
        const OpDef& last = ops[pstep.first + pstep.count - 1];
        if (last.out.size() != 1 || last.out[0].name != ops[steps[j].first].in[0].name) continue;
        if (pstep.kind == SK_CONV_ADD || (pstep.kind == SK_SINGLE && (last.type == "Conv" || last.type == "Add" || last.type == "Concat"))) p.stats_consumer[j - 1] = (long)j;
    }
    p.step_weights.assign(steps.size(), {});
    for (size_t si = 0; si < steps.size(); si++) {
        size_t step_bytes = 0;
        for (size_t oi = steps[si].first; oi < steps[si].first + steps[si].count; oi++)
            for (size_t k = 0; k < ops[oi].in.size(); k++) {
                auto& r = ops[oi].in[k];
                if (!r.present || r.wtype == DType::none) continue;
                size_t b = ref_bytes(r);
                p.step_weights[si].push_back({ oi, k, b });
                step_bytes += (b + 255) & ~(size_t)255;
            }
        p.largest_step_bytes = std::max(p.largest_step_bytes, step_bytes);
    }
    if (o.side_branch && o.fuse_nodes) plan_side_branch(ops, p);
    return p;
}

std::string plan_summary(const std::string& model_text, bool fp16_arithmetic, bool fuse_nodes, bool fuse_attention, bool sdpa_rewrite)
{
    PlanOptions o;
    o.fp16_arithmetic = fp16_arithmetic;
    o.fuse_nodes = fuse_nodes;
    o.fuse_attention = fuse_attention;
    o.sdpa_rewrite = sdpa_rewrite;
    const std::vector<OpDef> ops = parse_model_text(model_text, false);
    const Plan p = make_plan(ops, o);
    std::string out;
    std::map<std::string, size_t> counts;
    for (size_t si = 0; si < p.steps.size(); si++) {
        const Step& s = p.steps[si];
        const char* kn = step_kind_names[s.kind];
        const OpDef& op = ops[s.first];
        const bool side = si < p.is_side.size() && p.is_side[si], kvs = si < p.kv_side.size() && p.kv_side[si];
        const bool stats = p.stats_consumer[si] >= 0;
        out += std::string(kn) + " " + std::to_string(s.count) + " " + op.type + " " + op.name + (side ? " [side]" : "") + (kvs ? " [kv-side]" : "") + (stats ? " [gn-stats]" : "") + "\n";
        counts[kn]++;
        if (side) counts["side"]++;
        if (kvs) counts["kv_side"]++;
        if (stats) counts["gn_stats_producers"]++;
    }
    out += "#summary ops=" + std::to_string(ops.size()) + " steps=" + std::to_string(p.steps.size()) + " largest_node_bytes=" + std::to_string(p.largest_step_bytes);
    for (auto& kv : counts) out += " " + kv.first + "=" + std::to_string(kv.second);
    out += "\n";
    return out;
}

}  // namespace osb
