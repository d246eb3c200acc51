// engine_run.cpp -- the op interpreter: executes the steps of the plan (plan.h), op by op or through a fused handler.
//
// Semantics follow the reference's Model::run() branch by branch (src/onnxstream.cpp:3550-8269); the citation at
// each handler names the branch it restates.  What differs is *where* things run: float payloads are HBM-resident
// and every handler enqueues CUDA kernels on the compute stream; int64 tensors (shape arithmetic) stay on the host
// and are evaluated with the reference's own integer semantics, bit-exactly.
#include "engine_impl.h"
#include "plan.h"
#include "workspace.h"

#include <limits>
#include <cuda_fp16.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <thread>
#include <tuple>

namespace osb {

namespace {

inline int K(DType t) { return (int)t; }

std::vector<int64_t> parse_ints(const std::string& s)
{
    std::vector<int64_t> v;
    size_t start = 0;
    while (start <= s.size()) {
        size_t pos = s.find(',', start);
        std::string tok = s.substr(start, pos == std::string::npos ? std::string::npos : pos - start);
        if (!tok.empty()) v.push_back(std::stoll(tok));
        if (pos == std::string::npos) break;
        start = pos + 1;
    }
    return v;
}

[[noreturn]] void fail(const OpDef& op, const std::string& msg) { throw std::invalid_argument(op.type + ": " + msg); }

// Model::range_to_scale (src/onnxstream.cpp:3234-3245): (float range) / 255.0 in double, rounded to float; zero point truncated to uint8
static void range_to_scale(float lo, float hi, float& scale, int& zp)
{
    if (lo > 0 && hi > 0) lo = 0;
    else if (lo < 0 && hi < 0) hi = 0;
    scale = (float)((hi - lo) / 255.0);
    zp = (int)(uint8_t)(std::abs(lo) / scale);
}

}  // namespace

// ================================================================================================================
struct Engine::Impl {
    Engine& E;
    cudaStream_t st;      // the stream every handler launches on: the compute stream, or the side stream while the side branch is enqueued
    explicit Impl(Engine& e) : E(e), st(e.m_stream) {}
    ~Impl()
    {
        for (auto e : side_events) if (e) cudaEventDestroy(e);
        if (side_stream) { cudaStreamSynchronize(side_stream); osb_workspace_release(side_stream); cudaStreamDestroy(side_stream); }
    }

    // ---- tensor store (the reference's m_data + m_intermediate_refs, src/onnxstream.h:937,1023) ----
    std::unordered_map<std::string, std::vector<Tensor>> store;
    std::vector<std::string> order;
    std::map<std::string, int> refs;

    // ---- plan ----
    Plan plan;
    std::string plan_signature;
    size_t next_stage = 0;
    std::map<std::pair<size_t, size_t>, std::pair<WeightStreamer::Slot*, size_t>> staged;  // (op, in) -> (slot, blob)
    std::map<size_t, WeightStreamer::Slot*> step_slot;                                     // step -> its slot

    std::unordered_map<std::string, Tensor> resident;
    size_t resident_bytes = 0;

    // ---- side branch (resident weights only): the side steps of the plan (Plan::is_side, Plan::kv_side) are enqueued FIRST, on a second
    // stream with its own activation pool, and run concurrently with the main chain; a main step waits on the event of the side step it
    // consumes.  Inside a captured graph these become parallel branches.  ~15 % of a UNet step's launches leave the critical path.
    cudaStream_t side_stream = nullptr;
    DevicePool side_pool;
    bool on_side = false;
    std::vector<cudaEvent_t> side_events;              // per step (side steps only)
    DevicePool& pool() { return on_side ? side_pool : E.m_pool; }
    struct MhaKV { Tensor kl, vl; cudaEvent_t ev = nullptr; };
    std::map<size_t, MhaKV> mha_kv;                    // step -> K / V projections computed ahead on the side stream (valid for one run)
    void mha_project(size_t i, const Tensor& x, const Tensor* xq, Tensor* ql, Tensor& kl, Tensor& vl, int64_t Tka);
    void mha_prepass(size_t si);
    // fused flash kernel (K / V projections of exactly Tk rows) or the GEMM -> softmax -> GEMM chain (Tk padded to 8): one rule for
    // mha_prepass and fused_mha, which must agree on the K / V buffers
    bool mha_flash(int64_t T, int64_t Tk, int64_t d, DType ty, float scale) const
    {
        // the flash kernels take the running maximum over the raw scores, which is the maximum of the scaled logits only for scale > 0
        if (!flash_on() || !(scale > 0.f && scale < INFINITY)) return false;
        return ty == DType::f32 ? osb_flash_attention_f32x_ok(T, Tk, d, K(ty)) : osb_flash_attention_ok(T, Tk, d, K(ty));
    }
    // the flash attention kernels are on: b200_flash_attention, and not the CUDA-core GEMM path (b200_gemm_impl = 1)
    bool flash_on() const { return E.flash_attention && E.gemm_impl != 1; }

    // int64 graph inputs and CUDA graphs: an op that consumes the host VALUES of such a tensor (other than through its device mirror)
    // makes the run un-capturable -- a replay would reuse the values of the captured run
    bool capture_unsafe = false;
    bool last_run_capture_safe = false;
    static bool i64_safe_consumer(const OpDef& op, size_t k, const Tensor& t)
    {
        if (!t.i64_dev) return false;
        if (op.type == "Gather") return k == 1;
        if (op.type == "Cast") return true;
        return k == 0 && (op.type == "Unsqueeze" || op.type == "Squeeze" || op.type == "Reshape" || op.type == "Flatten" || op.type == "Identity");
    }

    struct OpTime { std::string type; cudaEvent_t a, b; };
    std::vector<OpTime> op_times;
    std::vector<Tensor> kept_inputs;      // b200_keep_inputs: device copies of the graph inputs of earlier runs, by name
    DevPtr gn_stats;
    // GroupNorm statistics gathered by the producer (conv epilogue / per-channel Add) instead of a pass of their own.  `gn_ring` holds
    // two fp64 [2 * 64] slots: a producer accumulates into the current slot (all zero by invariant), the GroupNorm's apply pass reads it
    // and zeroes the OTHER slot, which becomes current.  The whole ring is zeroed at the start of every run.
    DevPtr gn_ring;
    int gn_slot = 0;
    // per slot: how many leading doubles the last statistics written into it cover (2 * its GroupNorm's groups).  The apply pass
    // zeroes the other slot's first 2 * G doubles only; sums a GroupNorm with more groups left beyond them are zeroed separately.
    int gn_slot_used[2] = { 0, 0 };
    long stats_want = -1;                 // set while a producer step runs: the GroupNorm step that wants its statistics
    int stats_groups = 0;
    long stats_ready_for = -1;            // GroupNorm step whose statistics sit in the current slot
    double* gn_slot_ptr(int slot) { return (double*)((char*)gn_ring->ptr + slot * 1024); }
    static bool gn_split_enabled() { static const bool v = [] { const char* e = getenv("OSB_GN_SPLIT"); return !(e && e[0] == '0'); }(); return v; }
    static bool gn_apply_ok(const Tensor& t, int64_t C, int G)
    {
        const int vec = t.type == DType::f16 ? 8 : 4;
        return (t.type == DType::f16 || t.type == DType::f32) && t.layout == Layout::nhwc && t.shape.size() == 4 && G >= 1 && G <= 64 && C % G == 0 && C % vec == 0 && C <= 4096;
    }
    size_t cur_step = 0, cur_b = 0, cur_B = 1;
    std::unordered_map<std::string, Tensor> silu_cache;   // SiLU results of small tensors, valid for one run (see fused_silu)
    int runs_done = 0;

    // ------------------------------------------------------------------------------------------------------
    // helpers: allocation, conversion, layout
    // ------------------------------------------------------------------------------------------------------
    Tensor make(DType t, const std::vector<int64_t>& shape, Layout l = Layout::plain)
    {
        Tensor r;
        r.type = t; r.shape = shape; r.layout = l;
        int64_t n = 1; for (auto d : shape) n *= d;
        r.dev = pool().alloc((size_t)n * dtype_size(t));
        return r;
    }

    void ck(int err, const char* what) { check_cuda(err, what); }

    Tensor convert(const Tensor& x, DType to)
    {
        if (x.type == to) return x;
        Tensor r = make(to, x.shape, x.layout);
        ck(osb_convert(x.data(), K(x.type), r.mdata(), K(to), (size_t)x.numel(), x.scale, x.zero_point, st), "osb_convert");
        if (to == DType::u8) { r.scale = x.scale; r.zero_point = x.zero_point; }
        return r;
    }

    // NHWC physical <-> NCHW physical for logical [1,C,H,W] (or [1,C,L] with W = 1)
    Tensor to_plain(const Tensor& x)
    {
        if (x.layout == Layout::plain) return x;
        int64_t C = x.shape[1], HW = x.numel() / C;
        Tensor r = make(x.type, x.shape, Layout::plain);
        r.scale = x.scale; r.zero_point = x.zero_point;
        ck(osb_transpose2d(x.data(), r.mdata(), (int)dtype_size(x.type), 1, HW, C, st), "osb_transpose2d");
        return r;
    }
    Tensor to_nhwc(const Tensor& x)
    {
        if (x.layout == Layout::nhwc) return x;
        if (x.shape.size() < 3) throw std::invalid_argument("Model::get_tensor_data: transpose required but invalid shape.");
        int64_t C = x.shape[1], HW = x.numel() / C;
        Tensor r = make(x.type, x.shape, Layout::nhwc);
        r.scale = x.scale; r.zero_point = x.zero_point;
        ck(osb_transpose2d(x.data(), r.mdata(), (int)dtype_size(x.type), 1, C, HW, st), "osb_transpose2d");
        return r;
    }

    Tensor quantize_dynamic(const Tensor& x);     // percentile range -> uint8 (Model::quantize, src/onnxstream.cpp:3247-3330)
    Tensor dequantize(const Tensor& x, DType to);
    bool percentile_range(const Tensor& x, float& lo, float& hi);
    DevPtr pct_dev;
    std::shared_ptr<PinnedBuf> pct_host;

    // ops with a uint8 kernel under m_use_uint8_arithmetic (the reference's qu8 branches: Conv 4600-4660, MatMul 5780-5800, Add / Mul
    // 846-927 + 1666-1746, Softmax 5971-5972) plus the type-agnostic data movers; every other op sees dequantised inputs here
    // (the reference throws for most of them: a superset, never a different result)
    static bool op_takes_u8(const OpDef& op)
    {
        static const std::set<std::string> k = { "Conv", "MatMul", "Add", "Mul", "Softmax", "InstanceNormalization", "Reshape", "Transpose", "Concat", "Split", "Slice", "Unsqueeze", "Squeeze",
                                                 "Flatten", "Resize", "Gather", "Expand", "Identity" };
        return k.count(op.type) != 0;
    }

    bool upcast_op(const OpDef& op) const { return runs_upcast(op, E.use_fp16_arithmetic, E.requires_upcast); }

    // the rows of an activation [..., K]: the product of its leading dimensions
    static int64_t act_rows(const Tensor& a) { int64_t rows = 1; for (size_t k = 0; k + 1 < a.shape.size(); k++) rows *= a.shape[k]; return rows; }
    // OSB_W8_GEMV=0 keeps uint8 weights off the uint8 GEMV, so the fp32-copy route can be timed against it
    static bool w8_gemv_on() { static const bool v = [] { const char* e = getenv("OSB_W8_GEMV"); return !(e && e[0] == '0'); }(); return v; }

    // The stored-blob routes: the kernels that read the static weight (input 1) of a MatMul, Gemm or Conv as stored -- the same operand the
    // load-time conversion (src/onnxstream.cpp:2885-2900) would have made, with no converted copy in HBM.  For one node at most one applies:
    // the weight type separates uint8 from fp16, the activation rows the GEMV from the GEMM (uint8 at 2, fp16 at 8, plan.cpp
    // is_gemv_matmul).  A refused launch always ends on the node's converted-weight route.
    enum class WRoute { none, u8_gemv, f16_gemv, f16_gemm, u8_gemm, f16_conv, u8_conv };
    struct ConvDims { int64_t H, W, Cin, Cout; int kh, kw, stride; int64_t Ho, Wo; };
    // the route of op `op` (a Conv when `cv` is given) on activation `a`
    WRoute weight_route(const OpDef& op, const Tensor& a, const ConvDims* cv = nullptr) const
    {
        // W8A32: the tensor-core GEMM and conv apply the scale in their epilogue (osb_tc_gemm_f32x_u8w, osb_tc_conv_f32x_u8w).  Not under uint8
        // arithmetic or QDQ, not under fp16 arithmetic (W8A16 keeps its route), not with the CUDA-core GEMM (b200_gemm_impl = 1);
        // OSB_W8A32_TC=0 turns it off, so the fp32-copy route can be timed against it.
        static const bool w8a32_tc = [] { const char* e = getenv("OSB_W8A32_TC"); return !(e && e[0] == '0'); }();
        const TensorRef& wr = op.in[1];
        const bool u8_tc = w8a32_tc && a.type == DType::f32 && wr.wtype == DType::u8 && !E.use_uint8_arithmetic && !E.use_uint8_qdq && !E.use_fp16_arithmetic &&
                           E.gemm_impl != 1;
        if (cv) {
            const ConvDims& c = *cv;
            // fp16 shape rule (H100, DESIGN.md section 5): outputs of 128 x 128 pixels and more, where it measured 1.17-6.6x the expanded route
            // at every SD VAE decoder shape, and every output the expanded route cannot take; at 64 x 64 and below (the SD 1.5 UNet, the
            // decoder's latent level) the expanded route measured faster on most shapes and keeps them
            if (a.type == DType::f32 && wr.wtype == DType::f16 && E.gemm_impl != 1 && osb_tc_conv_f32x_f16w_ok(c.H, c.W, c.Cin, c.Cout, c.kh, c.kw, c.stride, c.Ho, c.Wo) &&
                (c.Ho * c.Wo >= 128 * 128 || !osb_tc_conv_f32x_ok(c.H, c.W, c.Cin, c.Cout, c.kh, c.kw, c.stride, c.Ho, c.Wo)))
                return WRoute::f16_conv;
            if (u8_tc && osb_tc_conv_f32x_u8w_ok(c.H, c.W, c.Cin, c.Cout, c.kh, c.kw, c.stride, c.Ho, c.Wo, wr.zero_point)) return WRoute::u8_conv;
            return WRoute::none;
        }
        if (wr.shape.size() != 2 || a.shape.empty() || a.shape.back() != wr.shape[0]) return WRoute::none;
        const int64_t Kd = wr.shape[0], N = wr.shape[1], rows = act_rows(a);
        const bool gemv = op.type != "Gemm";     // a Gemm never takes a GEMV
        if (wr.wtype == DType::u8) {
            // the uint8 GEMV dequantises in registers, for fp16 and fp32 arithmetic alike
            if (gemv && w8_gemv_on() && !E.use_uint8_arithmetic && !E.use_uint8_qdq && (a.type == DType::f16 || a.type == DType::f32) && rows <= 2 &&
                N % 16 == 0 && N >= 256 && Kd >= 64 && weight_target(op, wr, false) == a.type)
                return WRoute::u8_gemv;
            return u8_tc && rows > 2 && osb_tc_gemm_f32x_u8w_ok(rows, N, Kd, N, wr.zero_point) ? WRoute::u8_gemm : WRoute::none;
        }
        // fp32 arithmetic meeting an fp16 blob: the GEMV widens it in registers, the tensor-core GEMM splits it in shared memory (a ragged N
        // only with resident weights, on the row-padded copy)
        if (wr.wtype != DType::f16 || a.type != DType::f32 || E.use_fp16_arithmetic || upcast_op(op) || rows < 1) return WRoute::none;
        if (rows <= 8) return gemv ? WRoute::f16_gemv : WRoute::none;
        return E.gemm_impl != 1 && (N % 8 == 0 || E.resident_weights) && osb_tc_gemm_f32x_f16w_ok(rows, N, Kd, (N + 7) / 8 * 8) ? WRoute::f16_gemm : WRoute::none;
    }
    bool run_stored(WRoute r, size_t oi, const Tensor& a, const Tensor* bias, const Tensor* residual, size_t out_oi, Tensor* out = nullptr);
    // the q, k and v projections of the fused attention block at op i (activations xq, xk, xv) all on the uint8 tensor-core GEMM
    bool mha_stored(size_t i, const Tensor& xq, const Tensor& xk, const Tensor& xv) const
    {
        return weight_route(E.m_ops[i], xq) == WRoute::u8_gemm && weight_route(E.m_ops[i + 4], xk) == WRoute::u8_gemm &&
               weight_route(E.m_ops[i + 9], xv) == WRoute::u8_gemm;
    }
    void project_stored(size_t oi, const Tensor& x, Tensor& out);

    DType act_dtype() const { return E.use_fp16_arithmetic ? DType::f16 : DType::f32; }

    // ------------------------------------------------------------------------------------------------------
    // weights
    // ------------------------------------------------------------------------------------------------------
    static std::string weight_file(const TensorRef& r, bool& is_conv_weight)
    {
        std::string fn = r.name;
        size_t p = fn.find("_nchw.bin");
        is_conv_weight = p != std::string::npos;
        if (is_conv_weight) fn = fn.substr(0, p) + "_nhwc.bin";   // src/onnxstream.cpp:2666-2692
        return fn;
    }

    // target dtype of a static weight for `op` (src/onnxstream.cpp:2845-2909)
    DType weight_target(const OpDef& op, const TensorRef& r, bool requires_float) const
    {
        if (r.wtype == DType::i64) return DType::i64;
        if (upcast_op(op)) requires_float = true;
        bool skip_fp16 = true;
        for (auto& i : op.in) if (i.present && (i.wtype == DType::none || i.wtype == DType::f16)) { skip_fp16 = false; break; }
        bool half_ok = E.use_fp16_arithmetic && !requires_float;
        switch (r.wtype) {
        case DType::u8:
            if (E.use_uint8_arithmetic) return DType::u8;
            return (half_ok && !skip_fp16) ? DType::f16 : DType::f32;
        case DType::f16: return half_ok ? DType::f16 : DType::f32;
        case DType::f32: return (half_ok && !skip_fp16) ? DType::f16 : DType::f32;
        default: return r.wtype;
        }
    }

    // Make sure every weight up to and including the current step is in flight; run ahead while the ring has room.
    // Consecutive small nodes are staged as ONE slot (one cudaMemcpyAsync, one collective): a UNet has ~700 weight-bearing nodes, most
    // of them a few KB (biases, norm affine), and a per-node copy + event + NCCL call costs more than moving them.  A group never
    // exceeds `group_bytes` (and therefore never the ring = the largest node), so the "HBM-resident streamed weights <= one node"
    // bound is unchanged; the slot is released when its LAST step has been enqueued.
    void pump_weights()
    {
        if (!E.m_streamer) return;
        if (E.resident_weights && !E.m_first_run) return;  // served from the HBM cache
        static const size_t group_bytes = [] { const char* e = getenv("OSB_WEIGHT_GROUP_KB"); return (size_t)(e ? atoi(e) : 8192) << 10; }();
        const auto& weights = plan.step_weights;
        while (next_stage < weights.size()) {
            if (weights[next_stage].empty()) { next_stage++; continue; }
            // group = [next_stage, last]: grows while the sum stays under the cap (a node larger than the cap is a group of its own)
            size_t last = next_stage, total = 0;
            auto node_bytes = [&](size_t si) { size_t b = 0; for (auto& w : weights[si]) b += (w.bytes + 255) & ~(size_t)255; return b; };
            total = node_bytes(next_stage);
            const size_t cap = std::min(group_bytes, E.m_streamer->capacity() / 2);   // two groups in flight: upload(k+1) overlaps compute(k)
            for (size_t j = next_stage + 1; j < weights.size(); j++) {
                size_t b = node_bytes(j);
                if (total + b > cap) break;
                total += b;
                if (b) last = j;
            }
            bool must = next_stage <= cur_step;
            std::vector<WeightStreamer::Request> req;
            for (size_t si = next_stage; si <= last; si++)
                for (auto& w : weights[si]) {
                    const TensorRef& r = E.m_ops[w.op].in[w.in];
                    bool conv_w;
                    req.push_back({ weight_file(r, conv_w), r.wtype, w.bytes });
                }
            auto* slot = E.m_streamer->stage(*E.m_source, req, must);
            if (!slot) break;
            size_t k = 0;
            for (size_t si = next_stage; si <= last; si++)
                for (auto& w : weights[si]) staged[{ w.op, w.in }] = { slot, k++ };
            step_slot[last] = slot;
            next_stage = last + 1;
        }
    }

    // keep_stored: a uint8 or fp16 blob stays as stored -- the consumer dequantises / widens it in registers (decode GEMV): no float copy in HBM
    Tensor get_weight(size_t op_idx, size_t in_idx, bool requires_float = false, bool conv_layout = false, bool keep_stored = false)
    {
        const OpDef& op = E.m_ops[op_idx];
        const TensorRef& r = op.in[in_idx];
        bool conv_w;
        std::string fn = weight_file(r, conv_w);
        if (conv_w && !conv_layout) throw std::invalid_argument("Model::get_tensor_data: nchw layout not supported. (not implemented)");
        if (!conv_w && conv_layout) throw std::invalid_argument("Model::get_tensor_data: unable to determine tensor data file compatible with required_layout.");
        DType target = weight_target(op, r, requires_float);
        if (keep_stored && (r.wtype == DType::u8 || r.wtype == DType::f16)) target = r.wtype;

        Tensor t;
        t.name = fn;
        t.is_weight = true;
        t.shape = r.shape;
        if (conv_w) {
            if (t.shape.size() != 4) throw std::invalid_argument("Model::get_tensor_data: layout is nhwc but invalid shape.");
            t.shape = { r.shape[0], r.shape[2], r.shape[3], r.shape[1] };  // OHWI
        }
        t.scale = r.scale; t.zero_point = r.zero_point;
        size_t bytes = ref_bytes(r);
        int64_t numel = t.numel();

        if (r.wtype == DType::i64) {
            // shape constants: host only
            auto v = std::make_shared<std::vector<int64_t>>((size_t)numel);
            std::vector<char> tmp;
            auto it = staged.find({ op_idx, in_idx });
            const void* src = nullptr;
            if (it != staged.end()) src = it->second.first->blobs[it->second.second].host;
            else { tmp.resize(std::max<size_t>(bytes, 8)); src = E.m_source->fetch(fn, r.wtype, bytes, tmp.data()); }
            memcpy(v->data(), src, bytes);
            t.type = DType::i64; t.i64 = v;
            return t;
        }

        std::string rkey = fn + "|" + std::to_string((int)target);
        if (E.resident_weights) {
            auto it = resident.find(rkey);
            if (it != resident.end()) return it->second;
        }

        auto it = staged.find({ op_idx, in_idx });
        if (it == staged.end()) throw std::runtime_error("internal: weight not staged: " + fn);
        WeightStreamer::Slot* slot_ = it->second.first;
        const WeightStreamer::Blob* slot = &slot_->blobs[it->second.second];
        ck(cudaStreamWaitEvent(st, slot_->ready, 0), "cudaStreamWaitEvent(compute, weight ready)");

        // host mirror for small constants (scalars, eps, Resize scales, per-group affine of InstanceNorm)
        if (numel <= 64 && slot->host) {
            auto hv = std::make_shared<std::vector<float>>((size_t)numel);
            for (int64_t i = 0; i < numel; i++) {
                float f = 0.f;
                if (r.wtype == DType::f32) f = ((const float*)slot->host)[i];
                else if (r.wtype == DType::f16) { __half h; memcpy(&h, (const char*)slot->host + 2 * i, 2); f = __half2float(h); }
                else if (r.wtype == DType::u8) f = (float)((int)((const uint8_t*)slot->host)[i] - r.zero_point) * r.scale;
                (*hv)[i] = f;
            }
            t.host_f32 = hv;
        }

        if (target == r.wtype) {
            t.type = target;
            t.dev_raw = slot->dev;
            if (E.resident_weights) {
                Tensor c = make(target, t.shape);
                ck(cudaMemcpyAsync(c.mdata(), slot->dev, bytes, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync(resident)");
                t.dev = c.dev; t.dev_raw = nullptr;
            }
        } else {
            Tensor raw = t;
            raw.type = r.wtype; raw.dev_raw = slot->dev;
            Tensor c = convert(raw, target);
            t.type = target; t.dev = c.dev; t.dev_raw = nullptr;
            if (target != DType::u8) { t.scale = 0; t.zero_point = 0; }
        }
        if (E.resident_weights) { resident[rkey] = t; resident_bytes += (size_t)numel * dtype_size(target); }
        return t;
    }

    // The resident weight `name` ([Kd][N], b) as a row-padded copy [Kd][Np], Np = N rounded up to the 16-byte vector, zero in the pad:
    // made once and kept with the resident weights, it lets the vector GEMV stream a weight whose rows are not 16-byte granular (a
    // 32003-entry vocabulary; the scalar kernel ran at a fifth of the rate)
    Tensor padded_weight(const std::string& name, const Tensor& b, int64_t Kd, int64_t N)
    {
        const size_t es = dtype_size(b.type);
        const int64_t vec = 16 / (int64_t)es, Np = (N + vec - 1) / vec * vec;
        const std::string pkey = name + "|pad" + std::to_string((int)b.type);
        auto it = resident.find(pkey);
        if (it == resident.end()) {
            Tensor bp = make(b.type, { Kd, Np });
            ck(cudaMemsetAsync(bp.mdata(), 0, (size_t)(Kd * Np) * es, st), "cudaMemsetAsync(padded weight)");
            ck(cudaMemcpy2DAsync(bp.mdata(), (size_t)Np * es, b.data(), (size_t)N * es, (size_t)N * es, (size_t)Kd, cudaMemcpyDeviceToDevice, st),
               "cudaMemcpy2DAsync(padded weight)");
            resident_bytes += (size_t)(Kd * Np) * es;
            it = resident.emplace(pkey, bp).first;
        }
        return it->second;
    }

    // ------------------------------------------------------------------------------------------------------
    // store access
    // ------------------------------------------------------------------------------------------------------
    size_t batch_of(const std::string& name)
    {
        auto it = store.find(name);
        return it == store.end() ? 0 : it->second.size();
    }

    Tensor get_act(const OpDef& op, const std::string& name)
    {
        auto it = store.find(name);
        if (it == store.end()) throw std::invalid_argument("Model::get_tensor_data: input tensor not found: " + name);
        auto& v = it->second;
        return v.size() == 1 ? v[0] : v.at(cur_b);
    }

    // generic input fetch: weight or activation
    Tensor in(size_t op_idx, size_t k, bool requires_float = false)
    {
        const OpDef& op = E.m_ops[op_idx];
        if (k >= op.in.size() || !op.in[k].present) throw std::invalid_argument(op.type + ": missing input.");
        const TensorRef& r = op.in[k];
        if (r.wtype != DType::none) {
            auto key = std::make_pair(op_idx, k);
            auto it = wcache.find(key);
            if (it != wcache.end()) return it->second;
            Tensor t = get_weight(op_idx, k, requires_float, false);
            wcache[key] = t;
            return t;
        }
        Tensor t = get_act(op, r.name);
        if (t.type == DType::i64 && t.tainted && !i64_safe_consumer(op, k, t)) capture_unsafe = true;
        if (t.type == DType::u8 && (!E.use_uint8_arithmetic || requires_float || !op_takes_u8(op)))
            t = dequantize(t, (E.use_fp16_arithmetic && !requires_float && !upcast_op(op)) ? DType::f16 : DType::f32);
        if (requires_float && t.type == DType::f16) t = convert(t, DType::f32);
        if (!E.use_fp16_arithmetic && t.type == DType::f16) t = convert(t, DType::f32);   // fp16 STORAGE (m_force_fp16_storage / fp16 inputs), fp32 arithmetic
        if (upcast_op(op) && t.type == DType::f16) t = convert(t, DType::f32);
        return t;
    }
    std::map<std::pair<size_t, size_t>, Tensor> wcache;  // weights of the current step (shared by all batch items)
    static constexpr size_t W_STORED = ~(size_t)0;        // wcache input slot of a weight kept as its stored fp16 / uint8 blob (the stored-blob routes)
    // input 1 of op oi for the step: its stored blob (a slot of its own, so the blob never stands in for the converted copy), or the
    // converted copy; conv_layout: an OHWI conv weight
    Tensor weight1(size_t oi, bool stored, bool conv_layout)
    {
        const auto key = std::make_pair(oi, stored ? W_STORED : (size_t)1);
        auto it = wcache.find(key);
        return it != wcache.end() ? it->second : (wcache[key] = get_weight(oi, 1, false, conv_layout, stored));
    }
    // an optional bias / residual of a GEMM epilogue in the activation type and plain layout (empty when absent)
    Tensor epilogue_operand(const Tensor* t, DType ty)
    {
        if (!t) return Tensor();
        Tensor r = to_plain(*t);
        return r.type == ty ? r : convert(r, ty);
    }

    bool next_is_sole_consumer(size_t step_idx, const std::string& name)
    {
        // src/onnxstream.cpp:3009-3020: skip the storage conversion when the very next queued op is the only consumer
        if (step_idx + 1 >= plan.steps.size()) return false;
        const Step& ns = plan.steps[step_idx + 1];
        const OpDef& nop = E.m_ops[ns.first];
        for (auto& i : nop.in) if (i.present && i.wtype == DType::none && i.name == name) return refs[name] == 1;
        return false;
    }

    void push(size_t op_idx, size_t out_idx, Tensor t)
    {
        const OpDef& op = E.m_ops[op_idx];
        const TensorRef& o = op.out[out_idx];
        t.name = o.name;
        t.is_weight = false;
        if (!t.dev && t.dev_raw) {   // a view of the weight ring must not outlive the node: give it its own storage
            Tensor c = make(t.type, t.shape, t.layout);
            ck(cudaMemcpyAsync(c.mdata(), t.dev_raw, (size_t)t.numel() * dtype_size(t.type), cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync(weight view)");
            t.dev = c.dev; t.dev_raw = nullptr;
        }
        // shape check against model.txt (src/onnxstream.cpp:3070-3089)
        {
            std::vector<int64_t> want = o.shape;
            bool ok = want.size() == t.shape.size();
            if (!ok && E.support_dynamic_shapes && want.empty()) ok = true;
            if (ok && want.size() == t.shape.size())
                for (size_t i = 0; i < want.size(); i++)
                    if (want[i] != t.shape[i] && !(E.support_dynamic_shapes && want[i] == 0)) ok = false;
            if (!ok) fail(op, "unexpected shape of output.");
        }
        // m_range_data_calibrate (src/onnxstream.cpp:2983-3004): widen the recorded range of the producing op by this output's percentiles
        if (E.range_data_calibrate && (t.type == DType::f16 || t.type == DType::f32)) {
            float lo, hi;
            if (percentile_range(t, lo, hi)) {
                auto it = E.range_data.find(op.name);
                if (it == E.range_data.end()) E.range_data[op.name] = { lo, hi };
                else { it->second.first = std::min(it->second.first, lo); it->second.second = std::max(it->second.second, hi); }
            }
        }
        // m_use_uint8_qdq / m_use_uint8_arithmetic: every float output is percentile-quantised to uint8 storage unless the next queued op
        // is its only consumer (src/onnxstream.cpp:3006-3031)
        if ((E.use_uint8_qdq || E.use_uint8_arithmetic) && (t.type == DType::f16 || t.type == DType::f32) && !next_is_sole_consumer(cur_step, o.name))
            t = quantize_dynamic(t);
        // storage dtype rule of push_tensor (src/onnxstream.cpp:3006-3035)
        if (E.use_fp16_arithmetic && t.type == DType::f32 && !E.use_uint8_arithmetic && !E.use_uint8_qdq) {
            if (!next_is_sole_consumer(cur_step, o.name)) t = convert(t, DType::f16);
        }
        // m_force_fp16_storage (src/onnxstream.cpp:3764-3808): before every op the reference re-stores each fp32 tensor of m_data as fp16
        // unless that op is its only remaining consumer -- i.e. a freshly produced fp32 tensor is rounded to fp16 storage here unless the
        // next queued step consumes it alone.  (Names in m_force_uint8_storage_set would be percentile-quantised instead: see quantize_dynamic.)
        if (E.force_fp16_storage && t.type == DType::f32 && !next_is_sole_consumer(cur_step, o.name)) {
            if (E.force_uint8_storage_set.count(o.name)) t = quantize_dynamic(t);
            else t = convert(t, DType::f16);
        }
        auto& v = store[o.name];
        if (v.empty()) order.push_back(o.name);
        if (cur_b == 0) v.clear();
        v.push_back(std::move(t));
    }

    void consume_inputs(const Step& s)
    {
        std::set<std::string> produced;
        for (size_t i = s.first; i < s.first + s.count; i++)
            for (auto& o : E.m_ops[i].out) if (o.present) produced.insert(o.name);
        for (size_t i = s.first; i < s.first + s.count; i++)
            for (auto& r : E.m_ops[i].in) {
                if (!r.present || r.wtype != DType::none || produced.count(r.name)) continue;
                int& c = refs[r.name];
                c--;
                if (c < 0) throw std::runtime_error("Model::get_tensor_data: inconsistent reference count.");
                if (c == 0) {
                    store.erase(r.name);
                    order.erase(std::remove(order.begin(), order.end(), r.name), order.end());
                }
            }
    }

    // ------------------------------------------------------------------------------------------------------
    // op handlers
    // ------------------------------------------------------------------------------------------------------
    void exec_step(size_t si);
    void exec_single(size_t oi);
    // the ops of the group from its `done`-th on, one by one (the earlier ones have run)
    void exec_unfused(const Step& s, size_t done = 0)
    {
        for (size_t k = done; k < s.count; k++) exec_single(s.first + k);
        if (cur_b + 1 == cur_B)   // intermediates of the group have no consumer outside it: drop them
            for (size_t k = 0; k + 1 < s.count; k++)
                for (auto& o : E.m_ops[s.first + k].out) if (o.present) {
                    store.erase(o.name);
                    order.erase(std::remove(order.begin(), order.end(), o.name), order.end());
                }
    }
    void op_conv(size_t oi, const Tensor* residual = nullptr, size_t out_op = (size_t)-1);
    void op_matmul(size_t oi, const Tensor* bias = nullptr, const Tensor* residual = nullptr, size_t out_op = (size_t)-1);
    void op_gemm(size_t oi);
    void op_binary(size_t oi, int bop);
    void op_unary(size_t oi, int uop);
    void op_reshape_like(size_t oi);
    void op_transpose(size_t oi);
    void op_concat(size_t oi);
    void op_split(size_t oi);
    void op_slice(size_t oi);
    void op_resize(size_t oi);
    void op_softmax(size_t oi);
    void op_instnorm(size_t oi);
    void op_reduce_mean(size_t oi);
    void op_gather(size_t oi);
    void op_misc_host(size_t oi);
    void fused_attention(const Step& s);
    void fused_groupnorm(const Step& s);
    void fused_layernorm(const Step& s);
    void fused_gelu(const Step& s);
    void fused_geglu(const Step& s);
    void fused_silu(const Step& s);
    void fused_linear(const Step& s);
    void fused_sdpa(const Step& s);
    void fused_mha(const Step& s);
    void fused_rmsnorm(const Step& s);
    void fused_gemv_group(const Step& s);
    void fused_swiglu(const Step& s);
    bool gemv_group(const Tensor& a, const size_t* op_idx, int n, Tensor* outs);
    Tensor f32x_operand(const Tensor& t, int64_t rows, int64_t L, bool by_rows, int b_side, const std::string& cache_key);
    void fused_rope(const Step& s);

    Tensor binary(int bop, const Tensor& a, const Tensor& b, float out_scale = 0.f, int out_zp = 0);
    Tensor strided(const Tensor& x, const std::vector<int64_t>& out_shape, const std::vector<int64_t>& in_stride,
                   const std::vector<int64_t>* in_div, int64_t in_off);
    void attention_core(const Tensor& q, const Tensor& k, const Tensor& v, float scale, bool k_transposed, const Tensor* mask,
                        int64_t kv_group, Tensor& out);
};

// ---- small utilities --------------------------------------------------------------------------------------------
static std::vector<int64_t> contiguous_strides(const std::vector<int64_t>& shape)
{
    std::vector<int64_t> s(shape.size());
    int64_t acc = 1;
    for (size_t i = shape.size(); i-- > 0;) { s[i] = acc; acc *= shape[i]; }
    return s;
}

// numpy broadcasting of host-evaluated operands (Where, the compare ops): `out` is the broadcast shape of the operands' shapes (empty
// `ok` when they do not broadcast); for_each(f) calls f(i, off) for every output element i in order, off[k] being operand k's flat
// source index (the index arithmetic of Expand), advanced like an odometer: no per-element division, no index buffer
struct Broadcast {
    std::vector<int64_t> out;
    std::vector<std::vector<int64_t>> strides;   // per operand, per output dimension; 0 where the operand broadcasts
    bool ok = true;
    explicit Broadcast(const std::vector<std::vector<int64_t>>& shapes)
    {
        size_t nd = 0;
        for (auto& s : shapes) nd = std::max(nd, s.size());
        out.assign(nd, 1);
        std::vector<std::vector<int64_t>> padded;
        for (auto& s : shapes) {
            std::vector<int64_t> p(nd - s.size(), 1);
            p.insert(p.end(), s.begin(), s.end());
            for (size_t d = 0; d < nd; d++) {
                if (p[d] != out[d] && p[d] != 1 && out[d] != 1) ok = false;
                else if (p[d] != 1) out[d] = p[d];
            }
            padded.push_back(std::move(p));
        }
        for (auto& p : padded) {
            auto cs = contiguous_strides(p);
            for (size_t d = 0; d < nd; d++) if (p[d] == 1) cs[d] = 0;
            strides.push_back(std::move(cs));
        }
    }
    int64_t numel() const { int64_t n = 1; for (auto d : out) n *= d; return n; }
    template <class F> void for_each(F f) const
    {
        const size_t nd = out.size(), k = strides.size();
        const int64_t n = numel();
        std::vector<int64_t> idx(nd, 0), off(k, 0);
        for (int64_t i = 0; i < n; i++) {
            f((size_t)i, off.data());
            for (size_t d = nd; d-- > 0;) {
                if (++idx[d] < out[d]) { for (size_t j = 0; j < k; j++) off[j] += strides[j][d]; break; }
                idx[d] = 0;
                for (size_t j = 0; j < k; j++) off[j] -= strides[j][d] * (out[d] - 1);
            }
        }
    }
};

static float scalar_of(const Tensor& t, const OpDef& op)
{
    if (t.host_f32 && !t.host_f32->empty()) return (*t.host_f32)[0];
    if (t.i64 && !t.i64->empty()) return (float)(*t.i64)[0];
    fail(op, "scalar constant expected (not implemented).");
}

Tensor Engine::Impl::strided(const Tensor& x, const std::vector<int64_t>& out_shape, const std::vector<int64_t>& in_stride,
                             const std::vector<int64_t>* in_div, int64_t in_off)
{
    Tensor r = make(x.type, out_shape);
    r.scale = x.scale; r.zero_point = x.zero_point;
    if (r.numel() == 0) return r;
    // collapse to <= OSB_MAX_DIMS by merging adjacent dims that are contiguous on both sides
    std::vector<int64_t> shp, is, dv, os;
    auto ostr = contiguous_strides(out_shape);
    for (size_t i = 0; i < out_shape.size(); i++) {
        int64_t d = in_div ? (*in_div)[i] : 1;
        if (out_shape[i] == 1) continue;
        if (!shp.empty() && d == 1 && dv.back() == 1 && is.back() == in_stride[i] * out_shape[i] && os.back() == ostr[i] * out_shape[i]) {
            shp.back() *= out_shape[i]; is.back() = in_stride[i]; os.back() = ostr[i];
        } else { shp.push_back(out_shape[i]); is.push_back(in_stride[i]); dv.push_back(d); os.push_back(ostr[i]); }
    }
    if (shp.empty()) { shp.push_back(1); is.push_back(1); dv.push_back(1); os.push_back(1); }
    if (shp.size() > OSB_MAX_DIMS) throw std::invalid_argument("strided copy: too many dimensions (not implemented).");
    ck(osb_strided_copy(x.data(), r.mdata(), (int)dtype_size(x.type), (int)shp.size(), shp.data(), is.data(), dv.data(), in_off, os.data(), 0, st), "osb_strided_copy");
    return r;
}

// numpy-style broadcasting binary op (src/onnxstream.cpp:1666-1949); keeps NHWC when the shapes allow it
Tensor Engine::Impl::binary(int bop, const Tensor& a_in, const Tensor& b_in, float out_scale, int out_zp)
{
    Tensor a = a_in, b = b_in;
    if (a.type != b.type) {  // mixed f16/f32 (upcast ops): compute in f32
        if (a.type == DType::f16) a = convert(a, DType::f32);
        if (b.type == DType::f16) b = convert(b, DType::f32);
    }
    // NHWC fast paths
    auto per_channel = [](const Tensor& t, int64_t C) {
        if (t.layout != Layout::plain) return false;
        int64_t n = t.numel();
        if (n == 1) return true;
        if (n != C) return false;
        if (t.shape.size() == 3) return t.shape[0] == C;
        if (t.shape.size() == 4) return t.shape[0] == 1 && t.shape[1] == C;
        return false;
    };
    Layout out_layout = Layout::plain;
    std::vector<int64_t> ash = a.shape, bsh = b.shape;
    if (a.layout == Layout::nhwc || b.layout == Layout::nhwc) {
        bool done = false;
        if (a.layout == Layout::nhwc && b.layout == Layout::nhwc && a.shape == b.shape) { done = true; }
        else if (a.layout == Layout::nhwc && a.shape.size() == 4 && per_channel(b, a.shape[1])) {
            ash = { a.numel() / a.shape[1], a.shape[1] }; bsh = { b.numel() }; done = true;
        } else if (b.layout == Layout::nhwc && b.shape.size() == 4 && per_channel(a, b.shape[1])) {
            bsh = { b.numel() / b.shape[1], b.shape[1] }; ash = { a.numel() }; done = true;
        }
        if (done) out_layout = Layout::nhwc;
        else { a = to_plain(a); b = to_plain(b); ash = a.shape; bsh = b.shape; }
    }
    size_t nd = std::max(ash.size(), bsh.size());
    if (nd == 0) nd = 1;
    std::vector<int64_t> A(nd, 1), B(nd, 1), O(nd), as(nd), bs(nd);
    std::copy(ash.begin(), ash.end(), A.begin() + (nd - ash.size()));
    std::copy(bsh.begin(), bsh.end(), B.begin() + (nd - bsh.size()));
    for (size_t i = 0; i < nd; i++) {
        if (A[i] != B[i] && A[i] != 1 && B[i] != 1) throw std::invalid_argument("XnnPack::binary: shapes are not broadcastable.");
        O[i] = std::max(A[i], B[i]);
    }
    auto ca = contiguous_strides(A), cb = contiguous_strides(B);
    for (size_t i = 0; i < nd; i++) { as[i] = A[i] == 1 ? 0 : ca[i]; bs[i] = B[i] == 1 ? 0 : cb[i]; }
    // logical output shape
    std::vector<int64_t> out_shape;
    if (out_layout == Layout::nhwc) out_shape = a.layout == Layout::nhwc ? a.shape : b.shape;
    else {
        size_t ond = std::max(a.shape.size(), b.shape.size());
        out_shape.assign(O.end() - ond, O.end());
    }
    Tensor r = make(a.type, out_shape, out_layout);
    // collapse dims for the kernel
    std::vector<int64_t> S, SA, SB;
    for (size_t i = 0; i < nd; i++) {
        if (O[i] == 1) continue;
        if (!S.empty() && SA.back() == as[i] * O[i] && SB.back() == bs[i] * O[i]) { S.back() *= O[i]; SA.back() = as[i]; SB.back() = bs[i]; }
        else { S.push_back(O[i]); SA.push_back(as[i]); SB.push_back(bs[i]); }
    }
    if (S.empty()) { S.push_back(1); SA.push_back(0); SB.push_back(0); }
    if (S.size() > OSB_MAX_DIMS) throw std::invalid_argument("XnnPack::binary: too many dimensions (not implemented).");
    if (a.type == DType::u8) {
        r.scale = out_scale; r.zero_point = out_zp;
        ck(osb_binary_qu8(bop, a.data(), SA.data(), a.scale, a.zero_point, b.data(), SB.data(), b.scale, b.zero_point, r.mdata(), out_scale, out_zp, S.data(), (int)S.size(), st), "osb_binary_qu8");
        return r;
    }
    ck(osb_binary(bop, a.data(), SA.data(), b.data(), SB.data(), r.mdata(), S.data(), (int)S.size(), K(a.type), st), "osb_binary");
    return r;
}


// Model::quantize (src/onnxstream.cpp:3247-3330): percentile range of the tensor (get_percentiles, 0.1 % from either end, per
// reference chunk) -> scale / zero point (range_to_scale, 3234-3245) -> XNNPACK f32->qu8 conversion.  A tensor without a usable
// range (all values equal, non-finite ...) stays as it is, exactly like the reference (quantize returns false).
bool Engine::Impl::percentile_range(const Tensor& x, float& lo, float& hi)
{
    if (x.type != DType::f16 && x.type != DType::f32) return false;
    if (!pct_dev) { pct_dev = pool().alloc(256); pct_host = std::make_shared<PinnedBuf>(64); }
    unsigned* h = (unsigned*)pct_host->ptr;
    h[0] = 0xFFFFFFFFu; h[1] = 0; h[2] = 0;
    ck(cudaMemcpyAsync(pct_dev->ptr, h, 12, cudaMemcpyHostToDevice, st), "percentiles init");
    // the reference chunks the tensor by its pool's worker count; 0 = "all cores" there: use this host's count like it would
    int threads = E.cpu_threads > 0 ? E.cpu_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    ck(osb_percentiles(x.data(), K(x.type), (size_t)x.numel(), threads, 0.001f, 0.001f, pct_dev->ptr, st), "osb_percentiles");
    ck(cudaMemcpyAsync(h + 4, pct_dev->ptr, 12, cudaMemcpyDeviceToHost, st), "percentiles D2H");
    ck(cudaStreamSynchronize(st), "percentiles sync");      // the range decides host-side parameters (scale, zero point)
    if (h[6] == 0) return false;
    lo = osb_percentile_key_to_float(h[4], K(x.type));
    hi = osb_percentile_key_to_float(h[5], K(x.type));
    return std::isfinite(lo) && std::isfinite(hi) && lo < hi;
}


Tensor Engine::Impl::quantize_dynamic(const Tensor& x)
{
    float lo = 0, hi = 0;
    if (!percentile_range(x, lo, hi)) return x;
    Tensor src = x;
    src.scale = 0; src.zero_point = 0;
    range_to_scale(lo, hi, src.scale, src.zero_point);
    Tensor q = convert(src, DType::u8);
    q.scale = src.scale; q.zero_point = src.zero_point;
    return q;
}

Tensor Engine::Impl::dequantize(const Tensor& x, DType to)
{
    Tensor r = convert(x, to);       // (q - zero_point) * scale, src/onnxstream.cpp:3332-3434
    r.scale = 0; r.zero_point = 0;
    return r;
}

// ================================================================================================================
// handlers
// ================================================================================================================

// Conv (src/onnxstream.cpp:4494-4707 -> XnnPack::convolution 1292-1534)
void Engine::Impl::op_conv(size_t oi, const Tensor* residual, size_t out_op)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 3 && op.in.size() != 2) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    std::vector<int64_t> dil, ks, pads, strides;
    int64_t group = 1;
    for (auto& a : op.attrs) {
        if (a.first == "dilations") dil = parse_ints(a.second);
        else if (a.first == "group") group = std::stoll(a.second);
        else if (a.first == "kernel_shape") ks = parse_ints(a.second);
        else if (a.first == "pads") pads = parse_ints(a.second);
        else if (a.first == "strides") strides = parse_ints(a.second);
        else fail(op, "unrecognized attribute: " + a.first + ".");
    }
    if (E.use_nchw_convs) fail(op, "m_use_nchw_convs is not supported by the engine (file-backed conv weights are NHWC, src/onnxstream.cpp:2686-2689).");
    bool is1d = dil.size() == 1;
    if (is1d) {
        dil.push_back(1); ks.push_back(1);
        if (pads.size() != 2) fail(op, "invalid pads attribute value.");
        pads.insert(pads.begin() + 1, 0); pads.push_back(0);
        if (strides.size() != 1) fail(op, "invalid strides attribute value.");
        strides.push_back(strides[0]);
    }
    if (dil.size() != 2 || dil[0] != 1 || dil[1] != 1) fail(op, "invalid dilations attribute value (not implemented).");
    if (group != 1) fail(op, "invalid group attribute value (not implemented).");
    if (ks.size() != 2 || pads.size() != 4 || strides.size() != 2 || strides[0] != strides[1])
        throw std::runtime_error("XnnPack::convolution_nhwc_fp32: one or more arguments are invalid.");

    Tensor x = in(oi, 0);
    if (op.in[1].wtype == DType::none) fail(op, "dynamic convolution weights are not supported (not implemented).");
    const std::vector<int64_t>& wshape = op.in[1].shape;     // OIHW; get_weight returns it as OHWI
    Tensor b; bool has_b = op.in.size() > 2 && op.in[2].present;

    if (x.shape.size() == 3) x.shape.push_back(1);   // Conv1D: trailing unit dim (src/onnxstream.cpp:2919-2920)
    if (x.shape.size() != 4 || wshape.size() != 4) throw std::runtime_error("XnnPack::convolution_nhwc_fp32: one or more arguments are invalid.");
    if (wshape[2] != ks[0] || wshape[3] != ks[1]) fail(op, "invalid shape of W or invalid kernel_shape (not implemented?).");
    x = to_nhwc(x);
    int64_t H = x.shape[2], W = x.shape[3], Cin = x.shape[1], Cout = wshape[0];
    if (wshape[1] != Cin) throw std::runtime_error("XnnPack::convolution: invalid size of W.");
    int kh = (int)ks[0], kw = (int)ks[1], stride = (int)strides[0];
    // padding re-symmetrisation (src/onnxstream.cpp:1315-1331)
    int64_t ph = pads[0] + pads[2], pw = pads[1] + pads[3];
    int pad_top = (int)(ph / 2), pad_left = (int)(pw / 2);
    int64_t Ho = (H + ph - kh) / stride + 1, Wo = (W + pw - kw) / stride + 1;

    // the tensor-core conv on the fp16 / uint8 blob as stored (osb_tc_conv_f32x_f16w / _u8w): no fp32 copy, no bf16x6 expansion
    const ConvDims dims = { H, W, Cin, Cout, kh, kw, stride, Ho, Wo };
    const WRoute route = weight_route(op, x, &dims);
    Tensor w = weight1(oi, route != WRoute::none, true);
    if (has_b) b = in(oi, 2);

    Tensor y;
    if (x.type == DType::u8) {
        if (w.type != DType::u8) fail(op, "wrong data type of W.");
        auto it = E.range_data.find(op.name);
        if (it == E.range_data.end()) fail(op, "range data not found.");
        float oscale; int ozp;
        range_to_scale(it->second.first, it->second.second, oscale, ozp);
        DevPtr b32;
        if (has_b) {
            if (b.type != DType::f32 || !b.on_device()) fail(op, "wrong data type of B.");
            // bias -> int32 = (int32)(b / (sx*sw)) (src/onnxstream.cpp:4639-4660); tiny: do it through the host mirror path
            std::vector<float> hb((size_t)Cout);
            ck(cudaMemcpyAsync(hb.data(), b.data(), Cout * 4, cudaMemcpyDeviceToHost, st), "bias D2H");
            ck(cudaStreamSynchronize(st), "sync");
            std::vector<int32_t> ib((size_t)Cout);
            float s = x.scale * w.scale;
            for (int64_t i = 0; i < Cout; i++) ib[i] = (int32_t)(hb[i] / s);
            b32 = pool().alloc(Cout * 4);
            ck(cudaMemcpyAsync(b32->ptr, ib.data(), Cout * 4, cudaMemcpyHostToDevice, st), "bias H2D");
            ck(cudaStreamSynchronize(st), "sync");
        }
        y = make(DType::u8, { 1, Cout, Ho, Wo }, Layout::nhwc);
        y.scale = oscale; y.zero_point = ozp;
        if (E.gemm_impl != 1 && osb_qu8_tc_conv_ok(Cin, Cout, Ho, Wo, kh, kw, stride, x.data(), w.data(), y.mdata())) {
            // tensor cores (wgmma .u8): the image is padded once with the input zero point -- XNNPACK's padding value, which
            // TMA's zero fill cannot produce -- and the conv runs un-padded on it; zero-point terms are applied in the epilogue
            const int64_t Hp = (Ho - 1) * stride + kh, Wp = (Wo - 1) * stride + kw;
            DevPtr xp = pool().alloc((size_t)(Hp * Wp * Cin)), psum = pool().alloc((size_t)(Hp * Wp) * 4), csum = pool().alloc((size_t)Cout * 4);
            ck(osb_pad_sum_u8(x.data(), xp->ptr, psum->ptr, H, W, Cin, Hp, Wp, pad_top, pad_left, x.zero_point, st), "osb_pad_sum_u8");
            ck(osb_rowsum_u8(w.data(), csum->ptr, Cout, (int64_t)kh * kw * Cin, st), "osb_rowsum_u8");
            ck(osb_qu8_tc_conv(xp->ptr, psum->ptr, w.data(), b32 ? b32->ptr : nullptr, csum->ptr, y.mdata(), Hp, Wp, Cin, Cout, kh, kw, stride, Ho, Wo,
                               x.zero_point, x.scale, w.zero_point, w.scale, ozp, oscale, st), "osb_qu8_tc_conv");
        } else
        ck(osb_conv2d_qu8((const uint8_t*)x.data(), (const uint8_t*)w.data(), b32 ? (const int32_t*)b32->ptr : nullptr, (uint8_t*)y.mdata(),
                          H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, x.zero_point, x.scale, w.zero_point, w.scale, ozp, oscale, st), "osb_conv2d_qu8");
    } else {
        if (w.type != x.type && route == WRoute::none) w = convert(w, x.type);
        if (has_b && b.type != x.type) b = convert(b, x.type);
        y = make(x.type, { 1, Cout, Ho, Wo }, Layout::nhwc);
        Tensor rr;
        if (residual) {
            rr = *residual;
            if (rr.shape.size() == 3) rr.shape.push_back(1);
            rr = to_nhwc(rr);
            if (rr.type != x.type) rr = convert(rr, x.type);
        }
        // the GroupNorm right behind this conv wants per-group (sum, sum of squares) of the output: gathered in the epilogue
        void* gstats = nullptr; int gdone = 0, G = 0;
        if (stats_want >= 0 && gn_ring && cur_B == 1 && E.keep_nhwc && !is1d && gn_split_enabled()) {
            G = stats_groups;
            if (gn_apply_ok(y, Cout, G)) gstats = gn_slot_ptr(gn_slot);
        }
        bool done = false;
        if (route != WRoute::none) {
            const bool f16 = route == WRoute::f16_conv;
            Tensor planes = make(DType::f16, { 3 * H * W * Cin });     // the bf16 planes of x (6 bytes per element)
            const void *bp = has_b ? b.data() : nullptr, *rp = residual ? rr.data() : nullptr;
            const int rc = f16 ? osb_tc_conv_f32x_f16w(x.data(), w.data(), bp, rp, y.mdata(), H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, planes.mdata(), st)
                               : osb_tc_conv_f32x_u8w(x.data(), w.data(), bp, rp, y.mdata(), H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo, w.scale,
                                                      w.zero_point, planes.mdata(), st);
            if (rc == (int)cudaErrorNotSupported) w = convert(w, x.type);     // an operand the kernel cannot address: the fp32 routes below
            else { ck(rc, f16 ? "osb_tc_conv_f32x_f16w" : "osb_tc_conv_f32x_u8w"); done = true; }
        }
        if (!done && x.type == DType::f32 && E.gemm_impl != 1 && osb_tc_conv_f32x_ok(H, W, Cin, Cout, kh, kw, stride, Ho, Wo)) {
            // fp32 conv on the tensor cores: image and OHWI weights as bf16 triple-split expansions (6 Cin channels), fp32 result
            Tensor x6 = f32x_operand(x, H * W, Cin, false, 0, "");
            Tensor w6 = f32x_operand(w, Cout * kh * kw, Cin, false, 1, op.in[1].name + "|bf16x6");
            const int rc = osb_tc_conv_f32x(x6.data(), w6.data(), has_b ? b.data() : nullptr, residual ? rr.data() : nullptr, y.mdata(), H, W, 6 * Cin, Cout, kh, kw, stride,
                                            pad_top, pad_left, Ho, Wo, st);
            if (rc != (int)cudaErrorNotSupported) { ck(rc, "osb_tc_conv_f32x"); done = true; }
        }
        if (!done) {
        ck(osb_conv2d_ex(x.data(), w.data(), has_b ? b.data() : nullptr, nullptr, residual ? rr.data() : nullptr, y.mdata(), H, W, Cin, Cout, kh, kw, stride, pad_top, pad_left, Ho, Wo,
                         K(x.type), E.gemm_impl, st, gstats, G, &gdone), "osb_conv2d");
        if (gdone) stats_ready_for = stats_want;
        }
    }
    if (is1d) y.shape.pop_back();
    if (!E.keep_nhwc || is1d) { Tensor t = y; if (is1d) { t.shape.push_back(1); } t = to_plain(t); if (is1d) t.shape.pop_back(); y = t; }
    push(out_op == (size_t)-1 ? oi : out_op, 0, y);
}

// MatMul (src/onnxstream.cpp:5669-5861 -> XnnPack::matrix_multiply 1035-1215); optional fused bias / residual epilogue
void Engine::Impl::op_matmul(size_t oi, const Tensor* bias, const Tensor* residual, size_t out_op)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 2) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    Tensor a = to_plain(in(oi, 0));
    const WRoute route = weight_route(op, a);
    if (route != WRoute::none && run_stored(route, oi, a, bias, residual, out_op == (size_t)-1 ? oi : out_op)) return;
    Tensor b = to_plain(in(oi, 1));
    std::vector<int64_t> as = a.shape, bs = b.shape;
    bool lead1 = false, first2d = false;
    if (as.size() == 4 && as[0] == 1 && bs.size() == 4 && bs[0] == 1) { as.erase(as.begin()); bs.erase(bs.begin()); lead1 = true; }
    else if (as.size() == 2) { as.insert(as.begin(), 1); if (bs.size() != 3) first2d = true; }
    if (as.size() != 3) fail(op, "shape of input 0 must have 3 dimensions (not implemented).");
    int64_t n = as[0];
    int64_t stride_b;
    if (bs.size() == 2) { stride_b = 0; bs.insert(bs.begin(), n); }
    else { if (bs.size() != 3) fail(op, "shape of input 1 must have 2 or 3 dimensions (not implemented)."); if (bs[0] != n) fail(op, "shape of input 1 not supported (not implemented)."); stride_b = bs[1] * bs[2]; }
    if (as[2] != bs[1]) throw std::runtime_error("XnnPack::matrix_multiply_fp32: invalid shape of inputs.");
    int64_t M = as[1], Kd = as[2], N = bs[2];
    std::vector<int64_t> os = { n, M, N };
    if (lead1) os.insert(os.begin(), 1); else if (first2d) os.erase(os.begin());

    Tensor y;
    if (a.type == DType::u8) {
        if (b.type != DType::u8) fail(op, "wrong data type of input 1.");
        auto it = E.range_data.find(op.name);
        if (it == E.range_data.end()) fail(op, "range data not found.");
        float oscale; int ozp;
        range_to_scale(it->second.first, it->second.second, oscale, ozp);
        y = make(DType::u8, os);
        y.scale = oscale; y.zero_point = ozp;
        for (int64_t i = 0; i < n; i++) {
            const uint8_t* ai = (const uint8_t*)a.data() + i * M * Kd; const uint8_t* bi = (const uint8_t*)b.data() + i * stride_b; uint8_t* yi = (uint8_t*)y.mdata() + i * M * N;
            if (E.gemm_impl != 1 && osb_qu8_tc_gemm_ok(M, N, Kd, ai, bi, yi)) {
                // tensor cores (wgmma .u8) on the raw bytes; row sums of x and column sums of w feed the zero-point terms
                DevPtr rsum = pool().alloc((size_t)M * 4), csum = pool().alloc((size_t)N * 4);
                ck(osb_rowsum_u8(ai, rsum->ptr, M, Kd, st), "osb_rowsum_u8");
                ck(osb_colsum_u8(bi, csum->ptr, Kd, N, st), "osb_colsum_u8");
                ck(osb_qu8_tc_gemm(ai, bi, yi, nullptr, rsum->ptr, csum->ptr, M, N, Kd, 0, a.zero_point, a.scale, b.zero_point, b.scale, ozp, oscale, st), "osb_qu8_tc_gemm");
            } else
            ck(osb_gemm_qu8(ai, bi, yi, nullptr, M, N, Kd, a.zero_point, a.scale, b.zero_point, b.scale, ozp, oscale, st), "osb_gemm_qu8");
        }
    } else {
        if (b.type != a.type) b = convert(b, a.type);
        Tensor bb = epilogue_operand(bias, a.type), rr = epilogue_operand(residual, a.type);
        y = make(a.type, os);
        if (a.type == DType::f32 && n == 1 && E.gemm_impl != 1 && osb_tc_gemm_f32x_ok(M, N, Kd)) {
            // fp32 MatMul on the tensor cores (bf16 triple split); a static [K][N] weight is expanded once when the model is resident
            const bool stat = op.in[1].wtype != DType::none && op.in[1].shape.size() == 2;
            Tensor a6 = f32x_operand(a, M, Kd, false, 0, "");
            Tensor b6 = f32x_operand(b, Kd, N, true, 1, stat ? op.in[1].name + "|bf16x6" : std::string());
            const int rc = osb_tc_gemm_f32x(a6.data(), b6.data(), y.mdata(), bias ? bb.data() : nullptr, residual ? rr.data() : nullptr, M, N, 6 * Kd, 0, st);
            if (rc != (int)cudaErrorNotSupported) {
                ck(rc, "osb_tc_gemm_f32x");
                push(out_op == (size_t)-1 ? oi : out_op, 0, y);
                return;
            }
        }
        const int64_t vec = 16 / (int64_t)dtype_size(a.type);
        if (E.resident_weights && op.in[1].wtype != DType::none && op.in[1].shape.size() == 2 && n == 1 && M <= 8 && N >= 256 && N % vec != 0 && Kd >= 64) {
            // decode GEMV against a resident weight whose rows are not 16-byte granular (a 32003-entry vocabulary): see padded_weight
            const Tensor bp = padded_weight(op.in[1].name, b, Kd, N);
            ck(osb_gemm_ld(a.data(), Kd, bp.data(), bp.shape[1], y.mdata(), N, bias ? bb.data() : nullptr, residual ? rr.data() : nullptr, 1, M, N, Kd,
                           0, 0, 0, 0, K(a.type), E.gemm_impl, st), "osb_gemm_ld(padded weight)");
        } else
        ck(osb_gemm(a.data(), b.data(), y.mdata(), bias ? bb.data() : nullptr, residual ? rr.data() : nullptr, n, M, N, Kd,
                    M * Kd, stride_b, M * N, 0, K(a.type), E.gemm_impl, st), "osb_gemm");
    }
    push(out_op == (size_t)-1 ? oi : out_op, 0, y);
}

// The MatMul / Gemm at op oi on its stored blob by route r (weight_route): y = a . W (+ bias) (+ residual), pushed as output 0 of op out_oi,
// or written into *out (the attention projections).  The blob is the ring slot when streamed, the fp16 / uint8 cache entry when resident
// (a resident ragged N: the row-padded copy, shared by the fp16 GEMV and GEMM); no fp32 or expanded copy is made.  false = the kernel
// refused the operands: nothing pushed, the caller takes its converted-weight route.
bool Engine::Impl::run_stored(WRoute r, size_t oi, const Tensor& a, const Tensor* bias, const Tensor* residual, size_t out_oi, Tensor* out)
{
    const TensorRef& wr = E.m_ops[oi].in[1];
    const int64_t Kd = wr.shape[0], N = wr.shape[1], rows = act_rows(a);
    Tensor w = weight1(oi, true, false);
    int64_t ldb = N;
    if (E.resident_weights && N % 8 != 0 && (r == WRoute::f16_gemm || (r == WRoute::f16_gemv && N >= 256 && Kd >= 64))) { w = padded_weight(wr.name, w, Kd, N); ldb = w.shape[1]; }
    Tensor bb = epilogue_operand(bias, a.type), rr = epilogue_operand(residual, a.type);
    std::vector<int64_t> os = a.shape; os.back() = N;
    Tensor y = out ? *out : make(a.type, os);
    const void *bp = bias ? bb.data() : nullptr, *rp = residual ? rr.data() : nullptr;
    int rc;
    if (r == WRoute::u8_gemv)     // any failure: the converted route
        rc = osb_gemv_w8(a.data(), w.data(), y.mdata(), bp, rp, rows, N, Kd, w.scale, w.zero_point, K(a.type), st) == 0 ? 0 : (int)cudaErrorNotSupported;
    else if (r == WRoute::f16_gemv)
        rc = osb_gemv_f16w(a.data(), w.data(), ldb, y.mdata(), bp, rp, rows, N, Kd, st);
    else {
        Tensor planes = make(DType::f16, { 3 * rows * Kd });     // the bf16 planes of a (6 bytes per element)
        rc = r == WRoute::f16_gemm ? osb_tc_gemm_f32x_f16w(a.data(), w.data(), ldb, y.mdata(), bp, rp, rows, N, Kd, planes.mdata(), st)
                                   : osb_tc_gemm_f32x_u8w(a.data(), w.data(), N, y.mdata(), bp, rp, rows, N, Kd, w.scale, w.zero_point, planes.mdata(), st);
    }
    if (rc == (int)cudaErrorNotSupported) return false;
    ck(rc, r == WRoute::f16_gemv ? "osb_gemv_f16w" : r == WRoute::f16_gemm ? "osb_tc_gemm_f32x_f16w" : "osb_tc_gemm_f32x_u8w");
    if (!out) push(out_oi, 0, y);
    return true;
}

// out [rows, N] = x . W of the attention projection at op oi on its uint8 blob as stored (mha_stored); refused, the fp32 GEMM on its fp32 copy
void Engine::Impl::project_stored(size_t oi, const Tensor& x, Tensor& out)
{
    if (run_stored(WRoute::u8_gemm, oi, x, nullptr, nullptr, oi, &out)) return;
    const TensorRef& wr = E.m_ops[oi].in[1];
    Tensor w = in(oi, 1);
    if (w.type != x.type) w = convert(w, x.type);
    ck(osb_gemm(x.data(), w.data(), out.mdata(), nullptr, nullptr, 1, act_rows(x), wr.shape[1], wr.shape[0], 0, 0, 0, 0, K(x.type), E.gemm_impl, st), "osb_gemm(projection)");
}

// Gemm (src/onnxstream.cpp:4300-4375)
void Engine::Impl::op_gemm(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 3) fail(op, "wrong number of inputs. 2 inputs case not implemented.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    float alpha = 1, beta = 1; int transA = 0, transB = 0;
    for (auto& a : op.attrs) {
        if (a.first == "alpha") alpha = std::stof(a.second);
        else if (a.first == "beta") beta = std::stof(a.second);
        else if (a.first == "transA") transA = std::stoi(a.second);
        else if (a.first == "transB") transB = std::stoi(a.second);
        else fail(op, "unrecognized attribute: " + a.first + ".");
    }
    if (alpha != 1) fail(op, "alpha != 1 case not implemented.");
    if (beta != 1) fail(op, "beta != 1 case not implemented.");
    if (transA != 0) fail(op, "transA != 0 case not implemented.");
    if (transB != 0) fail(op, "transB != 0 case not implemented.");
    Tensor a = to_plain(in(oi, 0));
    const WRoute route = a.shape.size() == 2 && op.in[2].present ? weight_route(op, a) : WRoute::none;
    if (route != WRoute::none) {
        Tensor c = in(oi, 2);
        if (c.numel() == op.in[1].shape[1] && run_stored(route, oi, a, &c, nullptr, oi)) return;
    }
    Tensor b = in(oi, 1), c = in(oi, 2);
    if (a.shape.size() != 2 || b.shape.size() != 2) throw std::runtime_error("XnnPack::matrix_multiply_fp32: not implemented (shape of inputs).");
    if (a.shape[1] != b.shape[0]) throw std::runtime_error("XnnPack::matrix_multiply_fp32: invalid shape of inputs.");
    int64_t M = a.shape[0], Kd = a.shape[1], N = b.shape[1];
    if (c.numel() != N && c.numel() != M * N) throw std::runtime_error("XnnPack::matrix_multiply_fp32: invalid shape of bias.");
    if (b.type != a.type) b = convert(b, a.type);
    if (c.type != a.type) c = convert(c, a.type);
    Tensor y = make(a.type, { M, N });
    if (a.type == DType::f32 && c.numel() == N && E.gemm_impl != 1 && osb_tc_gemm_f32x_ok(M, N, Kd)) {
        Tensor a6 = f32x_operand(a, M, Kd, false, 0, "");
        Tensor b6 = f32x_operand(to_plain(b), Kd, N, true, 1, op.in[1].wtype != DType::none ? op.in[1].name + "|bf16x6" : std::string());
        const int rc = osb_tc_gemm_f32x(a6.data(), b6.data(), y.mdata(), c.data(), nullptr, M, N, 6 * Kd, 0, st);
        if (rc != (int)cudaErrorNotSupported) { ck(rc, "osb_tc_gemm_f32x"); push(oi, 0, y); return; }
    }
    ck(osb_gemm(a.data(), b.data(), y.mdata(), c.data(), nullptr, 1, M, N, Kd, 0, 0, 0, 0, K(a.type), E.gemm_impl, st), "osb_gemm");
    push(oi, 0, y);
}

// host-side int64 arithmetic with the reference's float round trip (src/onnxstream.cpp:3938-3950, 5159-5165, 5637-5649)
static std::shared_ptr<std::vector<int64_t>> i64_binary(int bop, const Tensor& a, const Tensor& b, std::vector<int64_t>& out_shape, const OpDef& op)
{
    auto& A = *a.i64; auto& B = *b.i64;
    size_t na = A.size(), nb = B.size();
    if (!(na == nb || na == 1 || nb == 1)) fail(op, "int64 broadcasting beyond scalars is not supported (not implemented).");
    size_t n = std::max(na, nb);
    out_shape = na >= nb ? a.shape : b.shape;
    if (a.shape.size() > out_shape.size()) out_shape = a.shape;
    auto r = std::make_shared<std::vector<int64_t>>(n);
    for (size_t i = 0; i < n; i++) {
        int64_t x = A[na == 1 ? 0 : i], y = B[nb == 1 ? 0 : i];
        switch (bop) {
        case OSB_BIN_ADD: (*r)[i] = x + y; break;
        case OSB_BIN_SUB: (*r)[i] = x - y; break;
        case OSB_BIN_MUL: (*r)[i] = (int64_t)((float)x * (float)y); break;
        case OSB_BIN_DIV: (*r)[i] = (int64_t)((float)x / (float)y); break;
        default: fail(op, "unsupported int64 op.");
        }
    }
    return r;
}

// Add / Sub / Mul / Div (src/onnxstream.cpp:5056-5175, 5394-5477, 3906-4000, 5605-5668)
void Engine::Impl::op_binary(size_t oi, int bop)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 2) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    Tensor a = in(oi, 0), b = in(oi, 1);
    if (a.type == DType::i64 || b.type == DType::i64) {
        if (a.type == DType::i64 && b.type == DType::i64) {
            Tensor r; r.type = DType::i64;
            r.i64 = i64_binary(bop, a, b, r.shape, op);
            push(oi, 0, r);
            return;
        }
        // int64 (x) float: the int64 side is a host constant -> upload as float (onnx2txt casts such Mul operands, cell 1)
        Tensor& f = a.type == DType::i64 ? b : a;
        Tensor& iv = a.type == DType::i64 ? a : b;
        Tensor c = make(f.type == DType::f16 ? DType::f16 : DType::f32, iv.shape);
        std::vector<float> hv(iv.i64->size());
        for (size_t i = 0; i < hv.size(); i++) hv[i] = (float)(*iv.i64)[i];
        Tensor tmp = make(DType::f32, iv.shape);
        ck(cudaMemcpyAsync(tmp.mdata(), hv.data(), hv.size() * 4, cudaMemcpyHostToDevice, st), "i64->f32 upload");
        ck(cudaStreamSynchronize(st), "sync");
        iv = convert(tmp, c.type);
    }
    if (a.type == DType::u8 || b.type == DType::u8) {
        // qu8 Add / Mul (src/onnxstream.cpp:5097-5125, 3906-4000): both operands uint8, output range from m_range_data
        if (a.type != DType::u8) fail(op, "wrong data type of input 0.");
        if (b.type != DType::u8) fail(op, "wrong data type of input 1.");
        if (bop != OSB_BIN_ADD && bop != OSB_BIN_MUL) fail(op, "qu8 arithmetic is implemented for Add and Mul only (as in the reference).");
        auto it = E.range_data.find(op.name);
        if (it == E.range_data.end()) fail(op, "range data not found.");
        float oscale; int ozp;
        range_to_scale(it->second.first, it->second.second, oscale, ozp);
        push(oi, 0, binary(bop, a, b, oscale, ozp));
        return;
    }
    if (stats_want >= 0 && gn_ring && cur_B == 1 && bop == OSB_BIN_ADD && a.type == b.type && gn_split_enabled()) {
        // x[NHWC] + t[1,C,1,1] feeding a GroupNorm (the time-embedding add of a resnet): one pass adds and gathers the statistics
        for (int k = 0; k < 2; k++) {
            const Tensor& full = k ? b : a; const Tensor& vecv = k ? a : b;
            if (full.layout != Layout::nhwc || full.shape.size() != 4 || vecv.layout != Layout::plain) continue;
            const int64_t C = full.shape[1];
            if (vecv.numel() != C || !(vecv.shape.size() == 4 && vecv.shape[1] == C) || !gn_apply_ok(full, C, stats_groups)) continue;
            Tensor r = make(full.type, full.shape, Layout::nhwc);
            if (osb_channel_add_stats(full.data(), vecv.data(), r.mdata(), K(full.type), C, full.numel() / C, stats_groups, gn_slot_ptr(gn_slot), st) == 0) {
                stats_ready_for = stats_want;
                push(oi, 0, r);
                return;
            }
        }
    }
    push(oi, 0, binary(bop, a, b));
}

// Sigmoid / Erf / Sqrt / Sin / Cos / Neg (src/onnxstream.cpp:4376-4493, 4001-4139, 7475-7542)
void Engine::Impl::op_unary(size_t oi, int uop)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 1) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    Tensor x = in(oi, 0);
    if (x.type == DType::i64) {
        if (uop != OSB_UN_NEG) fail(op, "wrong data type of input.");
        Tensor r; r.type = DType::i64; r.shape = x.shape;
        r.i64 = std::make_shared<std::vector<int64_t>>(*x.i64);
        for (auto& v : *r.i64) v = (int64_t)((float)v * -1.f);   // via float, src/onnxstream.cpp:7510-7521
        push(oi, 0, r);
        return;
    }
    if (x.type != DType::f16 && x.type != DType::f32) fail(op, "wrong data type of input.");
    Tensor y = make(x.type, x.shape, x.layout);
    ck(osb_unary(uop, x.data(), y.mdata(), K(x.type), (size_t)x.numel(), 0.f, st), "osb_unary");
    push(oi, 0, y);
}

// Reshape / Unsqueeze / Squeeze / Flatten: zero-copy (src/onnxstream.cpp:4708-4787, 3859-3905, 7425-7474, 8149-8189)
void Engine::Impl::op_reshape_like(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    Tensor x = in(oi, 0);
    if (x.layout == Layout::nhwc) x = to_plain(x);
    std::vector<int64_t> os;
    if (op.type == "Reshape") {
        if (op.in.size() != 2) fail(op, "wrong number of inputs.");
        for (auto& a : op.attrs) { if (a.first == "allowzero") { if (std::stoi(a.second)) fail(op, "allowzero must be 0 (not implemented)."); } else fail(op, "unrecognized attribute: " + a.first + "."); }
        Tensor sh = in(oi, 1);
        if (sh.type != DType::i64) fail(op, "wrong data type of shape.");
        if (sh.i64->empty()) fail(op, "size of shape must be non-0 (not implemented).");
        os = *sh.i64;
        for (size_t i = 0; i < os.size(); i++) if (os[i] == 0) { if (i >= x.shape.size()) fail(op, "insufficient number of dimensions in shape of data."); os[i] = x.shape[i]; }
        int64_t total = x.numel(), others = 1; int neg = -1;
        for (size_t i = 0; i < os.size(); i++) { if (os[i] == -1) { if (neg >= 0) fail(op, "more than one -1 in shape."); neg = (int)i; } else others *= os[i]; }
        if (neg >= 0) { if (others == 0 || total < others || total % others) fail(op, "unable to infer dimension of output shape."); os[neg] = total / others; }
    } else if (op.type == "Unsqueeze") {
        if (op.in.size() != 2) fail(op, "wrong number of inputs.");
        Tensor ax = in(oi, 1);
        if (ax.type != DType::i64) fail(op, "wrong data type of axes.");
        std::vector<int64_t> axes = *ax.i64;
        int rank = (int)(x.shape.size() + axes.size());
        for (auto& a : axes) { if (a < 0) a += rank; if (a < 0 || a >= rank) fail(op, "wrong data in axes."); }
        std::sort(axes.begin(), axes.end());
        os = x.shape;
        int64_t prev = -1;
        for (auto a : axes) { if (a == prev) fail(op, "duplicate value in axes."); prev = a; if (a > (int64_t)os.size()) fail(op, "wrong data in axes."); os.insert(os.begin() + a, 1); }
    } else if (op.type == "Squeeze") {
        os = x.shape;
        if (op.in.size() == 2 && op.in[1].present) {
            Tensor ax = in(oi, 1);
            std::vector<int64_t> axes = *ax.i64;
            for (auto& a : axes) if (a < 0) a += (int64_t)x.shape.size();
            std::sort(axes.rbegin(), axes.rend());
            for (auto a : axes) { if (a < 0 || a >= (int64_t)os.size() || os[a] != 1) fail(op, "wrong data in axes."); os.erase(os.begin() + a); }
        } else {
            os.erase(std::remove(os.begin(), os.end(), (int64_t)1), os.end());
        }
    } else {  // Flatten
        int64_t axis = 1;
        for (auto& a : op.attrs) { if (a.first == "axis") axis = std::stoll(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
        if (axis < 0) axis += (int64_t)x.shape.size();
        int64_t d0 = 1, d1 = 1;
        for (size_t i = 0; i < x.shape.size(); i++) ((int64_t)i < axis ? d0 : d1) *= x.shape[i];
        os = { d0, d1 };
    }
    Tensor y = x;
    y.shape = os;
    { int64_t n = 1; for (auto d : os) n *= d; if (n != x.numel()) fail(op, "unexpected shape of output."); }
    push(oi, 0, y);
}

// Transpose (src/onnxstream.cpp:5176-5236 -> XnnPack::transpose 1748-1809)
void Engine::Impl::op_transpose(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 1) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    std::vector<int64_t> perm;
    for (auto& a : op.attrs) { if (a.first == "perm") perm = parse_ints(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor x = in(oi, 0);
    if (x.type == DType::i64) fail(op, "int64 transpose is not implemented.");
    if (perm.size() != x.shape.size()) fail(op, "invalid perm attribute.");
    // channel-last relabelling: both directions are free
    if (E.keep_nhwc && x.shape.size() == 4 && x.shape[0] == 1) {
        if (x.layout == Layout::nhwc && perm == std::vector<int64_t>{ 0, 2, 3, 1 }) {
            Tensor y = x; y.layout = Layout::plain; y.shape = { 1, x.shape[2], x.shape[3], x.shape[1] };
            push(oi, 0, y); return;
        }
        if (x.layout == Layout::plain && perm == std::vector<int64_t>{ 0, 3, 1, 2 }) {
            Tensor y = x; y.layout = Layout::nhwc; y.shape = { 1, x.shape[3], x.shape[1], x.shape[2] };
            push(oi, 0, y); return;
        }
    }
    x = to_plain(x);
    {
        // a permutation that only moves unit axes around (LLM decode: (1, 1, heads, d) <-> (1, heads, 1, d)) leaves the bytes where they are
        bool valid = true, view = true; int64_t last = -1;
        for (size_t k = 0; k < perm.size() && valid; k++) {
            if (perm[k] < 0 || perm[k] >= (int64_t)perm.size()) { valid = false; break; }
            if (x.shape[perm[k]] == 1) continue;
            if (perm[k] < last) view = false;
            last = perm[k];
        }
        if (valid && view) {
            Tensor y = x;
            y.shape.resize(perm.size());
            for (size_t k = 0; k < perm.size(); k++) y.shape[k] = x.shape[perm[k]];
            push(oi, 0, y); return;
        }
    }
    auto istr = contiguous_strides(x.shape);
    std::vector<int64_t> os(perm.size()), is(perm.size());
    for (size_t i = 0; i < perm.size(); i++) { if (perm[i] < 0 || perm[i] >= (int64_t)perm.size()) fail(op, "invalid perm attribute."); os[i] = x.shape[perm[i]]; is[i] = istr[perm[i]]; }
    // batched 2-D case (last two dims swapped, leading dims untouched): tiled kernel
    size_t nd = perm.size();
    bool last2 = nd >= 2 && perm[nd - 1] == (int64_t)nd - 2 && perm[nd - 2] == (int64_t)nd - 1;
    for (size_t i = 0; i + 2 < nd && last2; i++) if (perm[i] != (int64_t)i) last2 = false;
    if (last2) {
        int64_t batch = 1; for (size_t i = 0; i + 2 < nd; i++) batch *= x.shape[i];
        if (batch <= 65535) {
            Tensor y = make(x.type, os);
            y.scale = x.scale; y.zero_point = x.zero_point;
            ck(osb_transpose2d(x.data(), y.mdata(), (int)dtype_size(x.type), batch, x.shape[nd - 2], x.shape[nd - 1], st), "osb_transpose2d");
            push(oi, 0, y); return;
        }
    }
    push(oi, 0, strided(x, os, is, nullptr, 0));
}

// Concat (src/onnxstream.cpp:4140-4299)
void Engine::Impl::op_concat(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.empty()) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    int64_t axis = 0; bool has_axis = false;
    for (auto& a : op.attrs) { if (a.first == "axis") { axis = std::stoll(a.second); has_axis = true; } else fail(op, "unrecognized attribute: " + a.first + "."); }
    if (!has_axis) fail(op, "axis attribute not found.");
    std::vector<Tensor> xs;
    for (size_t k = 0; k < op.in.size(); k++) xs.push_back(in(oi, k));
    size_t rank = xs[0].shape.size();
    if (axis < 0) axis += (int64_t)rank;
    if (axis < 0 || axis >= (int64_t)rank) fail(op, "invalid axis attribute.");
    if (xs[0].type == DType::i64) {
        Tensor r; r.type = DType::i64; r.i64 = std::make_shared<std::vector<int64_t>>();
        if (rank > 1) fail(op, "int64 concat of rank > 1 is not implemented.");
        for (auto& t : xs) { if (t.type != DType::i64) fail(op, "wrong data type of input."); r.i64->insert(r.i64->end(), t.i64->begin(), t.i64->end()); }
        r.shape = { (int64_t)r.i64->size() };
        push(oi, 0, r);
        return;
    }
    // uint8 sources (uint8 arithmetic) are copied as bytes only when every non-empty one carries the same scale and zero point.  Otherwise
    // each is dequantised at its own scale, and push re-quantises the float result by the percentile rule like any float output.
    size_t first = 0;
    while (first + 1 < xs.size() && xs[first].numel() == 0) first++;
    bool mixed_q = false;
    for (auto& t : xs)
        if (t.numel() != 0 && (t.type != xs[first].type || (t.type == DType::u8 && (t.scale != xs[first].scale || t.zero_point != xs[first].zero_point))))
            mixed_q = true;
    if (mixed_q) for (auto& t : xs) if (t.type == DType::u8) t = dequantize(t, act_dtype());
    DType ty = xs[first].type;
    bool all_nhwc = true;
    for (auto& t : xs) { if (t.layout != Layout::nhwc) all_nhwc = false; }
    bool nhwc_path = all_nhwc && axis == 1 && rank == 4 && E.keep_nhwc;
    for (auto& t : xs) {
        if (t.type != ty) t = convert(t, ty);
        if (!nhwc_path) t = to_plain(t);
        if (t.shape.size() != rank) fail(op, "invalid shape of input.");
    }
    std::vector<int64_t> os = xs[0].shape;
    os[axis] = 0;
    for (auto& t : xs) { for (size_t d = 0; d < rank; d++) if ((int64_t)d != axis && t.shape[d] != xs[0].shape[d]) fail(op, "invalid shape of input."); os[axis] += t.shape[axis]; }
    if (xs.size() == 2 && !nhwc_path) {
        // one empty source (the first turn's zero-length KV cache): the result is the other source
        for (int e = 0; e < 2; e++)
            if (xs[e].numel() == 0) { Tensor r = xs[1 - e]; r.shape = os; push(oi, 0, r); return; }
    }
    Tensor y = make(ty, os, nhwc_path ? Layout::nhwc : Layout::plain);
    y.scale = xs[first].scale; y.zero_point = xs[first].zero_point;
    if (nhwc_path && xs.size() == 2 && stats_want >= 0 && gn_ring && cur_B == 1 && gn_split_enabled() && gn_apply_ok(y, os[1], stats_groups)) {
        // the skip-connection Concat of a UNet up block feeding its GroupNorm: one pass copies and gathers the statistics
        if (osb_concat2_stats(xs[0].data(), xs[1].data(), y.mdata(), K(ty), xs[0].shape[1], xs[1].shape[1], os[2] * os[3], stats_groups, gn_slot_ptr(gn_slot), st) == 0) {
            stats_ready_for = stats_want;
            push(oi, 0, y);
            return;
        }
    }
    // physical view: [outer, axis_len * inner]
    int64_t outer = 1, inner = 1, total_axis = os[axis];
    if (nhwc_path) { outer = os[2] * os[3]; inner = 1; }
    else { for (int64_t d = 0; d < axis; d++) outer *= os[d]; for (size_t d = axis + 1; d < rank; d++) inner *= os[d]; }
    if (xs.size() == 2 && !nhwc_path) {
        // two sources (KV-cache append): one launch when everything is 16-byte granular
        const int64_t es = (int64_t)dtype_size(ty);
        if (osb_concat2(xs[0].data(), xs[1].data(), y.mdata(), outer, xs[0].shape[axis] * inner * es, xs[1].shape[axis] * inner * es, st) == 0) {
            push(oi, 0, y);
            return;
        }
        (void)cudaGetLastError();
    }
    int64_t off = 0;
    for (auto& t : xs) {
        int64_t len = t.shape[axis] * inner;
        if (len == 0) continue;
        int64_t shape2[2] = { outer, len }, is2[2] = { len, 1 }, dv2[2] = { 1, 1 }, os2[2] = { total_axis * inner, 1 };
        ck(osb_strided_copy(t.data(), y.mdata(), (int)dtype_size(ty), 2, shape2, is2, dv2, 0, os2, off, st), "osb_strided_copy(concat)");
        off += len;
    }
    push(oi, 0, y);
}

// Split (src/onnxstream.cpp:5999-6119)
void Engine::Impl::op_split(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    int64_t axis = 0;
    for (auto& a : op.attrs) { if (a.first == "axis") axis = std::stoll(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor x = to_plain(in(oi, 0));
    if (axis < 0) axis += (int64_t)x.shape.size();
    std::vector<int64_t> sizes;
    if (op.in.size() >= 2 && op.in[1].present) { Tensor s = in(oi, 1); sizes = *s.i64; }
    else { int64_t n = (int64_t)op.out.size(); for (int64_t i = 0; i < n; i++) sizes.push_back(x.shape[axis] / n); }
    if (sizes.size() != op.out.size()) fail(op, "wrong number of outputs.");
    auto istr = contiguous_strides(x.shape);
    int64_t start = 0;
    for (size_t j = 0; j < sizes.size(); j++) {
        std::vector<int64_t> os = x.shape; os[axis] = sizes[j];
        push(oi, j, strided(x, os, istr, nullptr, start * istr[axis]));
        start += sizes[j];
    }
}

// Slice (src/onnxstream.cpp:6499-6695): any axis, step 1 (the reference handles the last two axes only)
void Engine::Impl::op_slice(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() < 3) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    Tensor x = in(oi, 0);
    Tensor starts = in(oi, 1), ends = in(oi, 2);
    std::vector<int64_t> axes, steps_;
    if (op.in.size() > 3 && op.in[3].present) axes = *in(oi, 3).i64; else for (size_t i = 0; i < starts.i64->size(); i++) axes.push_back((int64_t)i);
    if (op.in.size() > 4 && op.in[4].present) steps_ = *in(oi, 4).i64; else steps_.assign(axes.size(), 1);
    if (x.type == DType::i64) {
        if (x.shape.size() != 1 || axes.size() != 1) fail(op, "int64 slice of rank > 1 is not implemented.");
        int64_t n = (int64_t)x.i64->size(), s = (*starts.i64)[0], e = (*ends.i64)[0], stp = steps_[0];
        if (stp != 1) fail(op, "step != 1 not implemented.");
        if (s < 0) s += n;
        if (e < 0) e += n;
        s = std::max<int64_t>(0, std::min(s, n)); e = std::max<int64_t>(0, std::min(e, n));
        Tensor r; r.type = DType::i64; r.i64 = std::make_shared<std::vector<int64_t>>(x.i64->begin() + s, x.i64->begin() + std::max(s, e));
        r.shape = { (int64_t)r.i64->size() };
        push(oi, 0, r);
        return;
    }
    x = to_plain(x);
    std::vector<int64_t> os = x.shape;
    auto istr = contiguous_strides(x.shape);
    int64_t off = 0;
    for (size_t i = 0; i < axes.size(); i++) {
        int64_t ax = axes[i]; if (ax < 0) ax += (int64_t)x.shape.size();
        if (ax < 0 || ax >= (int64_t)x.shape.size()) fail(op, "invalid axes.");
        if (steps_[i] != 1) fail(op, "steps != 1 not implemented.");
        int64_t n = x.shape[ax], s = (*starts.i64)[i], e = (*ends.i64)[i];
        if (s < 0) s += n;
        if (e < 0) e += n;
        s = std::max<int64_t>(0, std::min(s, n)); e = std::max<int64_t>(0, std::min(e, n));
        os[ax] = std::max<int64_t>(0, e - s);
        off += s * istr[ax];
    }
    push(oi, 0, strided(x, os, istr, nullptr, off));
}

// Resize: nearest / asymmetric / floor only (src/onnxstream.cpp:6120-6315)
void Engine::Impl::op_resize(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 3 && op.in.size() != 4) fail(op, "wrong number of inputs (not implemented).");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    if (op.in[1].present && !op.in[1].name.empty()) fail(op, "'roi' input not supported (not implemented).");
    Tensor x = in(oi, 0);
    if (x.shape.size() != 4) fail(op, "input must be 4D (not implemented).");
    if (x.shape[0] != 1) fail(op, "first dimension of input's shape must be 1 (not implemented).");
    std::vector<float> scales(4);
    std::vector<int64_t> os(4);
    if (op.in.size() == 3) {
        Tensor s = in(oi, 2, true);
        if (!s.host_f32 || s.host_f32->size() != 4) fail(op, "invalid data size of scales.");
        scales = *s.host_f32;
        for (int i = 0; i < 4; i++) os[i] = (int64_t)((float)x.shape[i] * scales[i]);
    } else {
        Tensor sz = in(oi, 3);
        if (sz.type != DType::i64 || sz.i64->size() != 4) fail(op, "invalid data size of sizes.");
        for (int i = 0; i < 4; i++) { os[i] = (*sz.i64)[i]; scales[i] = (float)os[i] / (float)x.shape[i]; }
    }
    if (scales[0] != 1 || scales[1] != 1) fail(op, "first and second value of scales must be 1 (not implemented).");
    std::string ctm, mode, nm;
    for (auto& a : op.attrs) {
        if (a.first == "coordinate_transformation_mode") ctm = a.second; else if (a.first == "mode") mode = a.second;
        else if (a.first == "nearest_mode") nm = a.second; else if (a.first == "cubic_coeff_a") {} else fail(op, "unrecognized attribute: " + a.first + ".");
    }
    if (ctm != "asymmetric" || mode != "nearest" || nm != "floor") fail(op, "one or more attributes are not supported (not implemented).");
    int64_t sy = (int64_t)scales[2], sx = (int64_t)scales[3];
    if ((float)sy != scales[2] || (float)sx != scales[3] || sy < 1 || sx < 1) fail(op, "non-integer resize scales are not implemented in the engine.");
    int64_t C = x.shape[1], H = x.shape[2], W = x.shape[3];
    Tensor y;
    if (x.layout == Layout::nhwc && E.keep_nhwc) {
        y = make(x.type, os, Layout::nhwc);
        int64_t shp[3] = { os[2], os[3], C }, is[3] = { W * C, C, 1 }, dv[3] = { sy, sx, 1 }, ost[3] = { os[3] * C, C, 1 };
        ck(osb_strided_copy(x.data(), y.mdata(), (int)dtype_size(x.type), 3, shp, is, dv, 0, ost, 0, st), "osb_strided_copy(resize)");
    } else {
        x = to_plain(x);
        y = make(x.type, os);
        int64_t shp[3] = { C, os[2], os[3] }, is[3] = { H * W, W, 1 }, dv[3] = { 1, sy, sx }, ost[3] = { os[2] * os[3], os[3], 1 };
        ck(osb_strided_copy(x.data(), y.mdata(), (int)dtype_size(x.type), 3, shp, is, dv, 0, ost, 0, st), "osb_strided_copy(resize)");
    }
    y.scale = x.scale; y.zero_point = x.zero_point;
    push(oi, 0, y);
}

// Softmax (src/onnxstream.cpp:5862-5998)
void Engine::Impl::op_softmax(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 1) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    int64_t axis = -1;
    for (auto& a : op.attrs) { if (a.first == "axis") axis = std::stoll(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor x = to_plain(in(oi, 0));
    int64_t rank = (int64_t)x.shape.size();
    if (axis < 0) axis += rank;
    if (axis < 0 || axis >= rank) fail(op, "invalid axis attribute.");
    if (x.type == DType::u8) {
        // qu8 softmax (src/onnxstream.cpp:5960-5995): output scale 2^-8, zero point 0; `axis` moved last by a transpose if needed
        Tensor t = x;
        std::vector<int64_t> perm;
        if (axis != rank - 1) {
            for (int64_t i = 0; i < rank; i++) if (i != axis) perm.push_back(i);
            perm.push_back(axis);
            auto istr = contiguous_strides(x.shape);
            std::vector<int64_t> ps(rank), pst(rank);
            for (int64_t i = 0; i < rank; i++) { ps[i] = x.shape[perm[i]]; pst[i] = istr[perm[i]]; }
            t = strided(x, ps, pst, nullptr, 0);
        }
        Tensor sres = make(DType::u8, t.shape);
        sres.scale = 0x1.0p-8f; sres.zero_point = 0;
        ck(osb_softmax_qu8(t.data(), sres.mdata(), t.numel() / t.shape.back(), t.shape.back(), x.scale, sres.scale, 0, st), "osb_softmax_qu8");
        if (!perm.empty()) {
            std::vector<int64_t> inv(rank);
            for (int64_t i = 0; i < rank; i++) inv[perm[i]] = i;
            auto sstr = contiguous_strides(t.shape);
            std::vector<int64_t> bs(rank);
            for (int64_t i = 0; i < rank; i++) bs[i] = sstr[inv[i]];
            Tensor back = strided(sres, x.shape, bs, nullptr, 0);
            back.scale = sres.scale; back.zero_point = 0;
            sres = back;
        }
        push(oi, 0, sres);
        return;
    }
    if (x.type != DType::f16 && x.type != DType::f32) fail(op, "wrong data type of input.");
    if (axis != rank - 1) {
        // move `axis` last, softmax, move back (src/onnxstream.cpp:5883-5898)
        std::vector<int64_t> perm;
        for (int64_t i = 0; i < rank; i++) if (i != axis) perm.push_back(i);
        perm.push_back(axis);
        auto istr = contiguous_strides(x.shape);
        std::vector<int64_t> ps(rank), pst(rank);
        for (int64_t i = 0; i < rank; i++) { ps[i] = x.shape[perm[i]]; pst[i] = istr[perm[i]]; }
        Tensor t = strided(x, ps, pst, nullptr, 0);
        Tensor s = make(x.type, ps);
        ck(osb_softmax(t.data(), s.mdata(), K(x.type), t.numel() / ps.back(), ps.back(), st), "osb_softmax");
        std::vector<int64_t> inv(rank);
        for (int64_t i = 0; i < rank; i++) inv[perm[i]] = i;
        auto sstr = contiguous_strides(ps);
        std::vector<int64_t> bs(rank);
        for (int64_t i = 0; i < rank; i++) bs[i] = sstr[inv[i]];
        push(oi, 0, strided(s, x.shape, bs, nullptr, 0));
        return;
    }
    Tensor y = make(x.type, x.shape);
    ck(osb_softmax(x.data(), y.mdata(), K(x.type), x.numel() / x.shape.back(), x.shape.back(), st), "osb_softmax");
    push(oi, 0, y);
}

// InstanceNormalization on [1, C, N] (src/onnxstream.cpp:4788-5055)
void Engine::Impl::op_instnorm(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 3) fail(op, "wrong number of inputs.");
    if (op.out.size() != 1) fail(op, "wrong number of outputs.");
    float eps = 1e-5f;
    for (auto& a : op.attrs) { if (a.first == "epsilon") eps = std::stof(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor x = to_plain(in(oi, 0)), sc = in(oi, 1), bi = in(oi, 2);
    if (x.shape.size() != 3 || x.shape[0] != 1) fail(op, "input must be 3D with a leading 1 (not implemented).");
    if (sc.numel() != x.shape[1] || bi.numel() != x.shape[1]) fail(op, "invalid shape of scale or B.");
    if (x.type == DType::u8) {
        // uint8 input (src/onnxstream.cpp:4846-4861, 4948-5040): dequantised in 64 KiB float tiles, statistics in double, result
        // re-quantised to the op's m_range_data scale -- here: dequantise, the fp32 kernel, quantise (XNNPACK's f32->qu8 conversion)
        auto it = E.range_data.find(op.name);
        if (it == E.range_data.end()) fail(op, "range data not found.");
        float oscale; int ozp;
        range_to_scale(it->second.first, it->second.second, oscale, ozp);
        Tensor xf = dequantize(x, DType::f32);
        if (sc.type != DType::f32) sc = convert(sc, DType::f32);
        if (bi.type != DType::f32) bi = convert(bi, DType::f32);
        Tensor yf = make(DType::f32, x.shape);
        ck(osb_instance_norm(xf.data(), yf.mdata(), K(DType::f32), x.shape[1], x.shape[2], sc.data(), bi.data(), eps, st), "osb_instance_norm");
        yf.scale = oscale; yf.zero_point = ozp;
        Tensor q = convert(yf, DType::u8);
        q.scale = oscale; q.zero_point = ozp;
        push(oi, 0, q);
        return;
    }
    if (x.type != DType::f16 && x.type != DType::f32) fail(op, "wrong data type of input.");
    if (sc.type != x.type) sc = convert(sc, x.type);
    if (bi.type != x.type) bi = convert(bi, x.type);
    Tensor y = make(x.type, x.shape);
    ck(osb_instance_norm(x.data(), y.mdata(), K(x.type), x.shape[1], x.shape[2], sc.data(), bi.data(), eps, st), "osb_instance_norm");
    push(oi, 0, y);
}

// ReduceMean over the last axis (src/onnxstream.cpp:5237-5393)
void Engine::Impl::op_reduce_mean(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 1) fail(op, "wrong number of inputs.");
    std::vector<int64_t> axes; int keepdims = 1;
    for (auto& a : op.attrs) { if (a.first == "axes") axes = parse_ints(a.second); else if (a.first == "keepdims") keepdims = std::stoi(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor x = to_plain(in(oi, 0));
    int64_t rank = (int64_t)x.shape.size();
    if (axes.size() != 1 || (axes[0] != -1 && axes[0] != rank - 1)) fail(op, "reduction on axes other than the last one is not supported (not implemented).");
    std::vector<int64_t> os = x.shape;
    if (keepdims) os.back() = 1; else os.pop_back();
    Tensor y = make(x.type, os);
    ck(osb_reduce_mean(x.data(), y.mdata(), K(x.type), x.numel() / x.shape.back(), x.shape.back(), st), "osb_reduce_mean");
    push(oi, 0, y);
}

// Gather axis 0 (src/onnxstream.cpp:6316-6498)
void Engine::Impl::op_gather(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    if (op.in.size() != 2) fail(op, "wrong number of inputs.");
    int64_t axis = 0;
    for (auto& a : op.attrs) { if (a.first == "axis") axis = std::stoll(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
    Tensor data = in(oi, 0), idx = in(oi, 1);
    if (idx.type != DType::i64) fail(op, "wrong data type of indices.");
    if (data.type == DType::i64) {
        if (axis < 0) axis += (int64_t)data.shape.size();
        if (data.shape.size() != 1 || axis != 0) fail(op, "int64 gather of rank > 1 is not implemented.");
        Tensor r; r.type = DType::i64; r.shape = idx.shape; r.i64 = std::make_shared<std::vector<int64_t>>();
        for (auto i : *idx.i64) { int64_t j = i < 0 ? i + (int64_t)data.i64->size() : i; if (j < 0 || j >= (int64_t)data.i64->size()) fail(op, "index out of range."); r.i64->push_back((*data.i64)[j]); }
        push(oi, 0, r);
        return;
    }
    data = to_plain(data);
    if (axis < 0) axis += (int64_t)data.shape.size();
    if (axis != 0) fail(op, "axis != 0 not implemented.");
    int64_t rows = data.shape[0], row_elems = data.numel() / std::max<int64_t>(rows, 1);
    std::vector<int64_t> os = idx.shape;
    os.insert(os.end(), data.shape.begin() + 1, data.shape.end());
    Tensor y = make(data.type, os);
    y.scale = data.scale; y.zero_point = data.zero_point;
    int64_t n = (int64_t)idx.i64->size();
    for (auto i : *idx.i64) if ((i < 0 ? i + rows : i) < 0 || (i < 0 ? i + rows : i) >= rows) fail(op, "index out of range.");
    if (idx.i64_dev) {
        // indices of a graph input (token ids, positions): read from the device mirror, so a captured graph follows new ids on replay
        // (the kernel clamps out-of-range rows; the host check above covers the eager runs)
        ck(osb_gather_rows(data.data(), (const int64_t*)idx.i64_dev->ptr, y.mdata(), n, rows, row_elems * (int64_t)dtype_size(data.type), st), "osb_gather_rows");
        push(oi, 0, y);
        return;
    }
    DevPtr didx = pool().alloc((size_t)n * 8);
    ck(cudaMemcpyAsync(didx->ptr, idx.i64->data(), (size_t)n * 8, cudaMemcpyHostToDevice, st), "gather idx H2D");
    ck(cudaStreamSynchronize(st), "sync");  // host vector may die before the copy otherwise (pageable source)
    ck(osb_gather_rows(data.data(), (const int64_t*)didx->ptr, y.mdata(), n, rows, row_elems * (int64_t)dtype_size(data.type), st), "osb_gather_rows");
    push(oi, 0, y);
}

// Host-evaluated shape / index ops of the LLM graph (src/onnxstream.cpp:7003-7033 Shape, 7352-7424 Cast,
// 7543-7588 ConstantOfShape, 7589-7636 Range, 7637-7766 compare, 7034-7153 Where, 7154-7351 Expand, 7883-7938 Trilu)
void Engine::Impl::op_misc_host(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    auto mk_i64 = [](std::vector<int64_t> v, std::vector<int64_t> shape) { Tensor r; r.type = DType::i64; r.shape = std::move(shape); r.i64 = std::make_shared<std::vector<int64_t>>(std::move(v)); return r; };
    if (op.type == "Shape") {
        Tensor x = in(oi, 0);
        std::vector<int64_t> v = x.shape;
        push(oi, 0, mk_i64(v, { (int64_t)v.size() }));
    } else if (op.type == "Cast") {
        int to = 0;
        for (auto& a : op.attrs) { if (a.first == "to") to = std::stoi(a.second); else fail(op, "unrecognized attribute: " + a.first + "."); }
        Tensor x = in(oi, 0);
        if (x.type == DType::i64 && to == 1 && x.i64_dev) {   // int64 graph input -> float, on the device (capturable)
            Tensor y = make(DType::f32, x.shape);
            ck(osb_convert(x.i64_dev->ptr, OSB_I64, y.mdata(), OSB_F32, (size_t)x.numel(), 0.f, 0, st), "osb_convert(i64)");
            push(oi, 0, y);
        } else if (x.type == DType::i64 && to == 1) {  // int64 -> float
            std::vector<float> hv(x.i64->size());
            for (size_t i = 0; i < hv.size(); i++) hv[i] = (float)(*x.i64)[i];
            Tensor y = make(DType::f32, x.shape);
            ck(cudaMemcpyAsync(y.mdata(), hv.data(), hv.size() * 4, cudaMemcpyHostToDevice, st), "cast H2D");
            ck(cudaStreamSynchronize(st), "sync");
            y.host_f32 = std::make_shared<std::vector<float>>(hv);
            push(oi, 0, y);
        } else if (x.type == DType::i64 && (to == 7 || to == 9 || to == 6)) {
            push(oi, 0, x);
        } else if ((x.type == DType::f32 || x.type == DType::f16) && (to == 1 || to == 10)) {
            push(oi, 0, x);   // float -> float: storage dtype is governed by the arithmetic mode
        } else if ((x.type == DType::f32 || x.type == DType::f16) && (to == 7 || to == 9 || to == 6)) {
            Tensor xf = convert(to_plain(x), DType::f32);
            std::vector<float> hv((size_t)xf.numel());
            ck(cudaMemcpyAsync(hv.data(), xf.data(), hv.size() * 4, cudaMemcpyDeviceToHost, st), "cast D2H");
            ck(cudaStreamSynchronize(st), "sync");
            std::vector<int64_t> v(hv.size());
            for (size_t i = 0; i < v.size(); i++) v[i] = (int64_t)hv[i];
            push(oi, 0, mk_i64(v, x.shape));
        } else fail(op, "unsupported cast (not implemented).");
    } else if (op.type == "ConstantOfShape") {
        float value = 0; bool is_int = true;
        for (auto& a : op.attrs) { if (a.first == "value") { value = std::stof(a.second); is_int = a.second.find('.') == std::string::npos; } else fail(op, "unrecognized attribute: " + a.first + "."); }
        Tensor sh = in(oi, 0);
        std::vector<int64_t> os = *sh.i64;
        int64_t n = 1; for (auto d : os) n *= d;
        if (is_int) push(oi, 0, mk_i64(std::vector<int64_t>((size_t)n, (int64_t)value), os));
        else { Tensor y = make(act_dtype(), os); ck(osb_fill(y.mdata(), K(y.type), (size_t)n, value, st), "osb_fill"); push(oi, 0, y); }
    } else if (op.type == "Range") {
        Tensor s = in(oi, 0), l = in(oi, 1), d = in(oi, 2);
        if (s.type != DType::i64) fail(op, "only int64 is supported.");
        std::vector<int64_t> v;
        for (int64_t x = (*s.i64)[0]; (*d.i64)[0] > 0 ? x < (*l.i64)[0] : x > (*l.i64)[0]; x += (*d.i64)[0]) v.push_back(x);
        int64_t n = (int64_t)v.size();
        push(oi, 0, mk_i64(std::move(v), { n }));
    } else if (op.type == "Less" || op.type == "Greater" || op.type == "Equal" || op.type == "And") {
        Tensor a = in(oi, 0), b = in(oi, 1);
        if (a.type != DType::i64 || b.type != DType::i64) fail(op, "only int64 operands are implemented in the engine.");
        if ((size_t)a.numel() != a.i64->size() || (size_t)b.numel() != b.i64->size()) fail(op, "invalid shape of one or more inputs.");
        const Broadcast bc({ a.shape, b.shape });
        if (!bc.ok) fail(op, "shapes are not broadcastable.");
        const int kind = op.type == "Less" ? 0 : op.type == "Greater" ? 1 : op.type == "Equal" ? 2 : 3;
        std::vector<int64_t> v((size_t)bc.numel());
        bc.for_each([&](size_t i, const int64_t* off) {
            const int64_t x = (*a.i64)[off[0]], y = (*b.i64)[off[1]];
            v[i] = kind == 0 ? x < y : kind == 1 ? x > y : kind == 2 ? x == y : (x && y);
        });
        push(oi, 0, mk_i64(std::move(v), bc.out));
    } else if (op.type == "Where") {
        Tensor c = in(oi, 0), x = in(oi, 1), y = in(oi, 2);
        if (c.type != DType::i64) fail(op, "wrong data type of condition.");
        // condition and branches broadcast against each other (a [1, 1, T, T] causal mask selecting from [1, H, T, T] scores)
        for (const Tensor* t : { &c, &x, &y })
            if (t->type == DType::i64 && (size_t)t->numel() != t->i64->size()) fail(op, "invalid shape of one or more inputs.");
        const Broadcast bc({ c.shape, x.shape, y.shape });
        if (!bc.ok) fail(op, "shapes are not broadcastable.");
        const size_t n = (size_t)bc.numel();
        if (x.type == DType::i64 && y.type == DType::i64) {
            std::vector<int64_t> v(n);
            bc.for_each([&](size_t i, const int64_t* off) { v[i] = (*c.i64)[off[0]] ? (*x.i64)[off[1]] : (*y.i64)[off[2]]; });
            push(oi, 0, mk_i64(std::move(v), bc.out));
        } else {
            // float branches: evaluate on the host (masks are tiny), then upload
            auto to_host = [&](Tensor t) { std::vector<float> hv; if (t.type == DType::i64) { hv.resize(t.i64->size()); for (size_t i = 0; i < hv.size(); i++) hv[i] = (float)(*t.i64)[i]; return hv; }
                Tensor f = convert(to_plain(t), DType::f32); hv.resize((size_t)f.numel()); ck(cudaMemcpyAsync(hv.data(), f.data(), hv.size() * 4, cudaMemcpyDeviceToHost, st), "where D2H"); ck(cudaStreamSynchronize(st), "sync"); return hv; };
            auto hx = to_host(x), hy = to_host(y);
            std::vector<float> hv(n);
            bc.for_each([&](size_t i, const int64_t* off) { hv[i] = (*c.i64)[off[0]] ? hx[off[1]] : hy[off[2]]; });
            Tensor f = make(DType::f32, bc.out);
            ck(cudaMemcpyAsync(f.mdata(), hv.data(), n * 4, cudaMemcpyHostToDevice, st), "where H2D");
            ck(cudaStreamSynchronize(st), "sync");
            push(oi, 0, f);
        }
    } else if (op.type == "Expand") {
        Tensor x = in(oi, 0), sh = in(oi, 1);
        std::vector<int64_t> target = *sh.i64;
        std::vector<int64_t> xs = x.shape;
        size_t nd = std::max(xs.size(), target.size());
        xs.insert(xs.begin(), nd - xs.size(), 1);
        target.insert(target.begin(), nd - target.size(), 1);
        std::vector<int64_t> os(nd);
        for (size_t i = 0; i < nd; i++) os[i] = std::max(xs[i], target[i]);
        if (x.type == DType::i64) {
            auto cs = contiguous_strides(xs);
            int64_t n = 1; for (auto d : os) n *= d;
            std::vector<int64_t> v((size_t)n);
            for (int64_t i = 0; i < n; i++) { int64_t rem = i, src = 0; for (size_t d = nd; d-- > 0;) { int64_t idx = rem % os[d]; rem /= os[d]; if (xs[d] != 1) src += idx * cs[d]; } v[i] = (*x.i64)[src]; }
            push(oi, 0, mk_i64(std::move(v), os));
        } else {
            x = to_plain(x);
            auto cs = contiguous_strides(xs);
            std::vector<int64_t> is(nd);
            for (size_t i = 0; i < nd; i++) is[i] = xs[i] == 1 ? 0 : cs[i];
            push(oi, 0, strided(x, os, is, nullptr, 0));
        }
    } else if (op.type == "ArgMax") {
        // src/onnxstream.cpp:6930-7002: int64 (1, D) input, last axis, keepdims 0, first maximum wins
        if (op.in.size() != 1) fail(op, "wrong number of inputs.");
        if (op.out.size() != 1) fail(op, "wrong number of outputs.");
        int axis = 0, keepdims = 1, select_last = 0;
        for (auto& a : op.attrs) {
            if (a.first == "axis") axis = std::stoi(a.second);
            else if (a.first == "keepdims") keepdims = std::stoi(a.second);
            else if (a.first == "select_last_index") select_last = std::stoi(a.second);
            else fail(op, "unrecognized attribute: " + a.first + ".");
        }
        Tensor x = in(oi, 0);
        if (axis < 0) axis += (int)x.shape.size();
        if (axis < 0 || axis >= (int)x.shape.size()) fail(op, "invalid axis attribute.");
        if (axis != (int)x.shape.size() - 1) fail(op, "argmax supported on last axis only (not implemented).");
        if (keepdims) fail(op, "keepdims must be 0 (not implemented).");
        if (select_last) fail(op, "select_last_index must be 0 (not implemented).");
        if (x.shape.size() != 2 || x.shape[0] != 1) fail(op, "shape of input must be (1,D) (not implemented).");
        if (x.type != DType::i64) fail(op, "wrong data type of input (not implemented).");
        int64_t best = std::numeric_limits<int64_t>::min(), arg = 0;
        for (int64_t i = 0; i < (int64_t)x.i64->size(); i++) if ((*x.i64)[i] > best) { best = (*x.i64)[i]; arg = i; }
        push(oi, 0, mk_i64({ arg }, { 1 }));
    } else if (op.type == "Trilu") {
        // src/onnxstream.cpp:7883-7938: upper triangle of a 2-D float tensor, out[y][x] = x - k >= y ? in[y][x] : 0
        if (op.in.size() != 2) fail(op, "wrong number of inputs.");
        if (op.out.size() != 1) fail(op, "wrong number of outputs.");
        std::string upper = "1";
        for (auto& a : op.attrs) { if (a.first == "upper") upper = a.second; else fail(op, "unrecognized attribute (not implemented)."); }
        if (upper != "1") fail(op, "'upper' must be 1 (not implemented).");
        Tensor x = to_plain(in(oi, 0)), kt = in(oi, 1);
        if (x.type != DType::f32 && x.type != DType::f16) fail(op, "wrong data type of input.");
        if (kt.type != DType::i64) fail(op, "wrong data type of k.");
        if (x.shape.size() != 2) fail(op, "input must be 2D (not implemented).");
        if (!kt.shape.empty()) fail(op, "second input (k) must be a scalar (not implemented).");
        // masks are tiny (causal-mask construction): evaluate on the host, exactly, in the storage type
        const int64_t h = x.shape[0], w = x.shape[1], k = (*kt.i64)[0];
        const size_t es = dtype_size(x.type);
        std::vector<uint8_t> hv((size_t)x.numel() * es);
        ck(cudaMemcpyAsync(hv.data(), x.data(), hv.size(), cudaMemcpyDeviceToHost, st), "trilu D2H");
        ck(cudaStreamSynchronize(st), "sync");
        for (int64_t yy = 0; yy < h; yy++)
            for (int64_t xx = 0; xx < w; xx++)
                if (!(xx - k >= yy)) std::memset(hv.data() + (size_t)(yy * w + xx) * es, 0, es);
        Tensor y = make(x.type, x.shape);
        ck(cudaMemcpyAsync(y.mdata(), hv.data(), hv.size(), cudaMemcpyHostToDevice, st), "trilu H2D");
        ck(cudaStreamSynchronize(st), "sync");
        push(oi, 0, y);
    } else if (op.type == "ScatterND") {
        // src/onnxstream.cpp:7939-8074: full-rank indices only (indices [.., rank]), element-wise scatter into a copy of the input
        if (op.in.size() != 3) fail(op, "wrong number of inputs.");
        if (op.out.size() != 1) fail(op, "wrong number of outputs.");
        if (!op.attrs.empty()) fail(op, "unrecognized attribute (not implemented).");
        Tensor x = to_plain(in(oi, 0)), idx = in(oi, 1), upd = to_plain(in(oi, 2));
        size_t rank = x.shape.size();
        if (!rank || idx.shape.size() != rank + 1 || upd.shape.size() != rank || idx.shape[rank] != (int64_t)rank) fail(op, "invalid shape of one or more inputs.");
        if (idx.type != DType::i64) fail(op, "wrong data type of indices.");
        if (x.type != DType::f32 && x.type != DType::f16) fail(op, "wrong data type of input.");
        if (upd.type != x.type) {
            if (upd.type != DType::f32 && upd.type != DType::f16) fail(op, "wrong data type of updates.");
            upd = convert(upd, x.type);
        }
        const int64_t n_upd = upd.numel();
        if ((size_t)n_upd * rank != idx.i64->size()) fail(op, "sizes of updates and indices not compatible.");
        auto dims = contiguous_strides(x.shape);
        std::vector<int64_t> pos((size_t)n_upd);
        for (int64_t i = 0; i < n_upd; i++) {
            int64_t p_ = 0;
            for (size_t j = 0; j < rank; j++) p_ += (*idx.i64)[(size_t)i * rank + j] * dims[j];
            if (p_ < 0 || p_ >= x.numel()) fail(op, "invalid index in indices.");
            pos[(size_t)i] = p_;
        }
        const size_t es = dtype_size(x.type);
        Tensor y = make(x.type, x.shape);
        ck(cudaMemcpyAsync(y.mdata(), x.data(), (size_t)x.numel() * es, cudaMemcpyDeviceToDevice, st), "scatter copy");
        if (n_upd) {
            DevPtr dpos = pool().alloc((size_t)n_upd * 8);
            ck(cudaMemcpyAsync(dpos->ptr, pos.data(), (size_t)n_upd * 8, cudaMemcpyHostToDevice, st), "scatter pos H2D");
            ck(cudaStreamSynchronize(st), "sync");   // pageable source
            ck(osb_scatter_elems(y.mdata(), (const int64_t*)dpos->ptr, upd.data(), n_upd, (int)es, st), "osb_scatter_elems");
        }
        push(oi, 0, y);
    } else if (op.type == "MaxPool") {
        // src/onnxstream.cpp:8075-8143 + XnnPack::maxpool_nhwc 1537-1664 (padding re-symmetrised: top = (pads[0]+pads[2])/2)
        if (op.in.size() != 1) fail(op, "wrong number of inputs.");
        if (op.out.size() != 1) fail(op, "wrong number of outputs.");
        std::vector<int64_t> dil, ks, pads, strides;
        int ceil_mode = 0;
        auto ints = [](const std::string& v) { std::vector<int64_t> r; size_t p0 = 0; while (p0 <= v.size()) { size_t c = v.find(',', p0); if (c == std::string::npos) c = v.size(); if (c > p0) r.push_back(std::stoll(v.substr(p0, c - p0))); p0 = c + 1; } return r; };
        for (auto& a : op.attrs) {
            if (a.first == "dilations") dil = ints(a.second);
            else if (a.first == "ceil_mode") ceil_mode = std::stoi(a.second);
            else if (a.first == "kernel_shape") ks = ints(a.second);
            else if (a.first == "pads") pads = ints(a.second);
            else if (a.first == "strides") strides = ints(a.second);
            else fail(op, "unrecognized attribute: " + a.first + ".");
        }
        if (dil != std::vector<int64_t>{ 1, 1 }) fail(op, "invalid dilations attribute value (not implemented).");
        if (ceil_mode != 0) fail(op, "invalid ceil_mode attribute value (not implemented).");
        Tensor x = in(oi, 0);
        if (x.type != DType::f32 && x.type != DType::f16) fail(op, "wrong data type of X.");
        if (x.shape.size() != 4 || ks.size() != 2 || pads.size() != 4 || strides.size() != 2 || strides[0] != strides[1])
            throw std::runtime_error("XnnPack::maxpool_nhwc: one or more arguments are invalid.");
        if (x.shape[0] != 1) fail(op, "first dimension of input's shape must be 1 (not implemented).");
        x = to_nhwc(x);
        const int64_t C = x.shape[1], H = x.shape[2], W = x.shape[3];
        const int64_t ph = pads[0] + pads[2], pw = pads[1] + pads[3];
        if (H + ph < ks[0] || W + pw < ks[1] || strides[0] < 1) throw std::runtime_error("XnnPack::maxpool_nhwc: one or more arguments are invalid.");
        const int64_t Ho = (H + ph - ks[0]) / strides[0] + 1, Wo = (W + pw - ks[1]) / strides[0] + 1;
        Tensor y = make(x.type, { 1, C, Ho, Wo }, Layout::nhwc);
        ck(osb_maxpool_nhwc(x.data(), y.mdata(), K(x.type), H, W, C, (int)ks[0], (int)ks[1], (int)strides[0], (int)(ph / 2), (int)(pw / 2), Ho, Wo, st), "osb_maxpool_nhwc");
        push(oi, 0, y);
    } else fail(op, "operation not implemented: " + op.type);
}

// ---- fused groups ------------------------------------------------------------------------------------------------

// softmax(Q K^T s + mask) V, heads batched.  Large Tq: heads with 160 < d <= 512 and no mask (the VAE's attention) run the wide
// flash kernel, fp16 or (fp32, through bf16 planes, where its grid fills half the SMs) the fp32 one; otherwise two GEMMs around a
// scaled softmax on a score tile of q's type (the reference materialises the same tile per part, src/onnxstream.cpp:6803-6922); short
// Tq (decode): the direct online-softmax kernel.
void Engine::Impl::attention_core(const Tensor& q, const Tensor& k, const Tensor& v, float scale, bool k_transposed, const Tensor* mask,
                                  int64_t kv_group, Tensor& out)
{
    int64_t h = q.shape[0], Tq = q.shape[1], d = q.shape[2];
    int64_t Tk = k_transposed ? k.shape[2] : k.shape[1], dv = v.shape[2];
    if (Tq <= 16 || kv_group != 1) {
        ck(osb_attention(q.data(), k.data(), v.data(), mask ? mask->data() : nullptr, out.mdata(), h, Tq, Tk, d, dv, scale, k_transposed ? 1 : 0, kv_group, K(q.type), st), "osb_attention");
        return;
    }
    // wide heads (the VAE's d = 512): one flash kernel, no [Tq, Tk] score buffer
    const bool aligned = (((uintptr_t)q.data() | (uintptr_t)k.data() | (uintptr_t)v.data() | (uintptr_t)out.data()) & 15) == 0;
    if (!mask && dv == d && h <= 65535 && scale > 0.f && flash_on() && aligned && osb_flash_attention_wide_ok(Tq, Tk, d, K(q.type))) {
        // a transposed K with Tk % 8 != 0 (any odd latent) has rows of Tk * 2 bytes, which TMA cannot address: transpose it to
        // [h, Tk, d] (Tk * d scratch) and take the K-major kernel
        Tensor kk = k;
        bool kt = k_transposed;
        if (kt && Tk % 8) {
            kk = make(q.type, { h, Tk, d });
            ck(osb_transpose2d(k.data(), kk.mdata(), (int)dtype_size(q.type), h, d, Tk, st), "osb_transpose2d(K^T)");
            kt = false;
        }
        ck(osb_flash_attention_wide(q.data(), kk.data(), v.data(), out.mdata(), h, Tq, Tk, d, scale, kt ? 1 : 0, K(q.type), st), "osb_flash_attention_wide");
        return;
    }
    // fp32 wide heads: one CTA per head, 64-query tile and 256-column slice of V, each streaming every key; with fewer CTAs than half
    // the H100's 132 SMs the fp32 kernel is slower than the chain (d = 512 on the H100: 0.71x at T = 1024, 32 CTAs; 0.99x at T = 1600,
    // 50 CTAs; 1.28x at T = 2304, 72 CTAs -- DESIGN section 5), so those grids keep the chain
    const bool wide_f32_fills = h * ((Tq + 63) / 64) * ((d + 255) / 256) >= 66;
    if (!mask && dv == d && h <= 65535 && scale > 0.f && flash_on() && aligned && wide_f32_fills &&
        osb_flash_attention_wide_f32x_ok(Tq, Tk, d, K(q.type))) {
        // the launch splits q, k, v into bf16 planes (6 bytes per element) in this scratch; its K split also transposes K^T
        Tensor planes = make(DType::f16, { 3 * (Tq + 2 * Tk) * h * d });
        ck(osb_flash_attention_wide_f32x(q.data(), k.data(), v.data(), out.mdata(), h, Tq, Tk, d, scale, k_transposed ? 1 : 0, planes.mdata(), st),
           "osb_flash_attention_wide_f32x");
        return;
    }
    // chunk heads so the score scratch stays bounded (<= 512 MiB)
    int64_t per_head = Tq * Tk * (int64_t)dtype_size(q.type);
    int64_t hc = std::max<int64_t>(1, std::min<int64_t>(h, ((int64_t)512 << 20) / std::max<int64_t>(per_head, 1)));
    for (int64_t h0 = 0; h0 < h; h0 += hc) {
        int64_t nh = std::min(hc, h - h0);
        Tensor s = make(q.type, { nh, Tq, Tk });
        const char* qp = (const char*)q.data() + h0 * Tq * d * dtype_size(q.type);
        const char* kp = (const char*)k.data() + h0 * Tk * d * dtype_size(q.type);
        const char* vp = (const char*)v.data() + h0 * Tk * dv * dtype_size(q.type);
        char* op_ = (char*)out.mdata() + h0 * Tq * dv * dtype_size(q.type);
        ck(osb_gemm(qp, kp, s.mdata(), nullptr, nullptr, nh, Tq, Tk, d, Tq * d, Tk * d, Tq * Tk, k_transposed ? 0 : 1, K(q.type), E.gemm_impl, st), "osb_gemm(QK)");
        ck(osb_softmax_scaled(s.data(), s.mdata(), K(q.type), nh * Tq, Tk, scale, mask ? mask->data() : nullptr, Tq, st), "osb_softmax_scaled");
        ck(osb_gemm(s.data(), vp, op_, nullptr, nullptr, nh, Tq, dv, Tk, Tq * Tk, Tk * dv, Tq * dv, 0, K(q.type), E.gemm_impl, st), "osb_gemm(PV)");
    }
}

// AttentionFusedOps (src/onnxstream.cpp:3576-3633 rewrite, 6696-6929 execution)
void Engine::Impl::fused_attention(const Step& s)
{
    size_t i = s.first;
    bool with_scale = s.count == 4;
    const OpDef& mm0 = E.m_ops[i];
    size_t mm1i = i + (with_scale ? 3 : 2);
    Tensor q = to_plain(in(i, 0)), k = to_plain(in(i, 1)), v = to_plain(in(mm1i, 1));
    float scale = 1.f;
    if (with_scale) { Tensor sc = in(i + 1, 1); scale = scalar_of(sc, E.m_ops[i + 1]); if (q.type == DType::f16) scale = __half2float(__float2half_rn(scale)); }
    bool lead1 = false;
    std::vector<int64_t> qs = q.shape, ks = k.shape, vs = v.shape;
    if (qs.size() == 4 && qs[0] == 1 && ks.size() == 4 && ks[0] == 1 && vs.size() == 4 && vs[0] == 1) { qs.erase(qs.begin()); ks.erase(ks.begin()); vs.erase(vs.begin()); lead1 = true; }
    if (qs.size() != 3 || ks.size() != 3 || vs.size() != 3) throw std::invalid_argument("AttentionFusedOps: shapes of q, k and v must have 3 dimensions.");
    if (qs[0] != ks[0] || qs[0] != vs[0]) throw std::invalid_argument("AttentionFusedOps: invalid shape(s) of q, k and/or v.");
    if (qs[1] < (int64_t)E.attention_fused_ops_parts) throw std::invalid_argument("AttentionFusedOps: m_attention_fused_ops_parts is not valid.");
    if (ks[1] != qs[2] || vs[1] != ks[2]) throw std::runtime_error("XnnPack::matrix_multiply_fp32: invalid shape of inputs.");
    if (k.type != q.type) k = convert(k, q.type);
    if (v.type != q.type) v = convert(v, q.type);
    Tensor q3 = q, k3 = k, v3 = v; q3.shape = qs; k3.shape = ks; v3.shape = vs;
    std::vector<int64_t> os = { qs[0], qs[1], vs[2] };
    Tensor out = make(q.type, os);
    attention_core(q3, k3, v3, scale, true, nullptr, 1, out);
    if (lead1) out.shape.insert(out.shape.begin(), 1);
    (void)mm0;
    push(mm1i, 0, out);
}

// Multi-head attention block (see Planner::mha in plan.cpp).  Per-op semantics are those of the MatMul / Reshape / Transpose /
// AttentionFusedOps branches (src/onnxstream.cpp:5669-5861, 4708-4787, 5176-5236, 6696-6929); the head split and merge
// become leading-dimension arithmetic on the projection buffers instead of copies.
// The projections of a fused multi-head attention block: the ones that share their input run as one grouped launch (self-attention:
// q, k, v; cross-attention: k, v).  ql == nullptr: K and V only (side-branch pre-pass).
void Engine::Impl::mha_project(size_t i, const Tensor& x, const Tensor* xq, Tensor* ql, Tensor& kl, Tensor& vl, int64_t Tka)
{
    Tensor xk = to_plain(in(i + 4, 0)), xv = to_plain(in(i + 9, 0));
    if (mha_stored(i, x, xk, xv)) {
        // W8A32: each projection on its uint8 weight as stored, one launch each
        const int64_t Tk = E.m_ops[i + 8].out[0].shape[2], C = kl.shape[1];
        if (Tka != Tk) {   // zero pad rows, as below
            ck(cudaMemsetAsync((char*)kl.mdata() + Tk * C * 4, 0, (Tka - Tk) * C * 4, st), "cudaMemsetAsync");
            ck(cudaMemsetAsync((char*)vl.mdata() + Tk * C * 4, 0, (Tka - Tk) * C * 4, st), "cudaMemsetAsync");
        }
        if (ql) project_stored(i, *xq, *ql);
        project_stored(i + 4, xk, kl);
        project_stored(i + 9, xv, vl);
        return;
    }
    Tensor wq = in(i, 1), wk = in(i + 4, 1), wv = in(i + 9, 1);
    const DType ty = x.type;
    if (xk.type != ty) xk = convert(xk, ty);
    if (xv.type != ty) xv = convert(xv, ty);
    if (wq.type != ty) wq = convert(wq, ty);
    if (wk.type != ty) wk = convert(wk, ty);
    if (wv.type != ty) wv = convert(wv, ty);
    auto& qs = E.m_ops[i + 3].out[0].shape; auto& kts = E.m_ops[i + 8].out[0].shape;
    const int64_t h = qs[0], T = qs[1], d = qs[2], Tk = kts[2], C = h * d;
    const size_t es = dtype_size(ty);
    if (Tka != Tk) {   // zero pad rows: they are read as extra (null) keys / values by the padded GEMMs
        ck(cudaMemsetAsync((char*)kl.mdata() + Tk * C * es, 0, (Tka - Tk) * C * es, st), "cudaMemsetAsync");
        ck(cudaMemsetAsync((char*)vl.mdata() + Tk * C * es, 0, (Tka - Tk) * C * es, st), "cudaMemsetAsync");
    }
    const bool kv_same = xk.data() == xv.data() && xk.shape == xv.shape && wk.shape == wv.shape;
    const bool qkv_same = ql && xq && kv_same && xq->data() == xk.data() && xq->shape == xk.shape && wq.shape == wk.shape && T == Tk;
    if (qkv_same) {
        const void* Bs[3] = { wq.data(), wk.data(), wv.data() };
        void* Cs[3] = { ql->mdata(), kl.mdata(), vl.mdata() };
        ck(osb_gemm_grouped(xq->data(), Bs, Cs, 3, T, C, xq->shape[2], 0, K(ty), E.gemm_impl, st), "osb_gemm_grouped(qkv)");
        return;
    }
    if (ql) ck(osb_gemm(xq->data(), wq.data(), ql->mdata(), nullptr, nullptr, 1, T, C, xq->shape[2], 0, 0, 0, 0, K(ty), E.gemm_impl, st), "osb_gemm(q)");
    if (kv_same) {
        const void* Bs[2] = { wk.data(), wv.data() };
        void* Cs[2] = { kl.mdata(), vl.mdata() };
        ck(osb_gemm_grouped(xk.data(), Bs, Cs, 2, Tk, C, xk.shape[2], 0, K(ty), E.gemm_impl, st), "osb_gemm_grouped(kv)");
    } else {
        ck(osb_gemm(xk.data(), wk.data(), kl.mdata(), nullptr, nullptr, 1, Tk, C, xk.shape[2], 0, 0, 0, 0, K(ty), E.gemm_impl, st), "osb_gemm(k)");
        ck(osb_gemm(xv.data(), wv.data(), vl.mdata(), nullptr, nullptr, 1, Tk, C, xv.shape[2], 0, 0, 0, 0, K(ty), E.gemm_impl, st), "osb_gemm(v)");
    }
}

// side-branch pre-pass of a cross-attention block: K / V projections of the (primary-independent) context, on the side stream
void Engine::Impl::mha_prepass(size_t si)
{
    const Step& s = plan.steps[si];
    const size_t i = s.first;
    cur_step = si; cur_b = 0; cur_B = 1;
    wcache.clear();
    Tensor xk = to_plain(in(i + 4, 0));
    const DType ty = act_dtype();
    if (xk.type != DType::f16 && xk.type != DType::f32) return;
    auto& qs = E.m_ops[i + 3].out[0].shape; auto& kts = E.m_ops[i + 8].out[0].shape;
    const int64_t h = qs[0], T = qs[1], d = qs[2], Tk = kts[2], C = h * d;
    float scale = scalar_of(in(i + 14, 1), E.m_ops[i + 14]);
    if (ty == DType::f16) scale = __half2float(__float2half_rn(scale));     // as fused_mha rounds it
    const bool use_flash = mha_flash(T, Tk, d, ty, scale);
    const int64_t Tka = use_flash ? Tk : ((Tk + 7) & ~(int64_t)7);
    Tensor proxy; proxy.type = ty; proxy.shape = E.m_ops[i].in[0].shape;     // the query side as the route rule sees it
    MhaKV kv;
    kv.kl = make(ty, { Tka, C }); kv.vl = make(ty, { Tka, C });
    mha_project(i, proxy, nullptr, nullptr, kv.kl, kv.vl, Tka);
    wcache.clear();
    mha_kv[si] = kv;
}

void Engine::Impl::fused_mha(const Step& s)
{
    size_t i = s.first;
    const OpDef& op = E.m_ops[i];
    Tensor x = to_plain(in(i, 0)), xk = to_plain(in(i + 4, 0)), xv = to_plain(in(i + 9, 0));
    // W8A32: the projections read their uint8 weights as stored (mha_project), so no fp32 copy is fetched here
    const bool u8p = mha_stored(i, x, xk, xv);
    Tensor wq, wk, wv;
    if (!u8p) { wq = in(i, 1); wk = in(i + 4, 1); wv = in(i + 9, 1); }
    for (size_t k : { (size_t)1, (size_t)3, (size_t)5, (size_t)7, (size_t)10, (size_t)12, (size_t)17, (size_t)19 }) (void)in(i + k, 1);   // shape constants: validated statically
    DType ty = x.type;
    if (ty != DType::f16 && ty != DType::f32) fail(op, "wrong data type of input 0.");
    if (xk.type != ty) xk = convert(xk, ty);
    if (xv.type != ty) xv = convert(xv, ty);
    if (!u8p && wq.type != ty) wq = convert(wq, ty);
    if (!u8p && wk.type != ty) wk = convert(wk, ty);
    if (!u8p && wv.type != ty) wv = convert(wv, ty);
    auto& qs = E.m_ops[i + 3].out[0].shape; auto& kts = E.m_ops[i + 8].out[0].shape;
    int64_t h = qs[0], T = qs[1], d = qs[2], Tk = kts[2], C = h * d;
    int64_t Tkp = (Tk + 7) & ~(int64_t)7;
    size_t es = dtype_size(ty);
    float scale = scalar_of(in(i + 14, 1), E.m_ops[i + 14]);
    if (ty == DType::f16) scale = __half2float(__float2half_rn(scale));
    if (x.shape[2] != op.in[1].shape[0] || xk.shape[2] != E.m_ops[i + 4].in[1].shape[0] || xv.shape[2] != E.m_ops[i + 9].in[1].shape[0]) throw std::runtime_error("XnnPack::matrix_multiply_fp32: invalid shape of inputs.");

    const bool use_flash = mha_flash(T, Tk, d, ty, scale);
    // the flash kernel reads K / V through tensor maps of exactly Tk rows (rows beyond are zero-filled by TMA): no padding needed
    const int64_t Tka = use_flash ? Tk : Tkp;
    Tensor ql = make(ty, { T, C }), kl, vl, out = make(ty, { 1, T, C });
    auto pre = mha_kv.find(cur_step);
    if (pre != mha_kv.end()) {
        // K / V projections of the text context were computed ahead on the side stream: only Q is projected here
        kl = pre->second.kl; vl = pre->second.vl;
        ck(cudaStreamWaitEvent(st, pre->second.ev, 0), "cudaStreamWaitEvent(main, side K/V)");
        mha_kv.erase(pre);
        if (u8p) project_stored(i, x, ql);
        else ck(osb_gemm(x.data(), wq.data(), ql.mdata(), nullptr, nullptr, 1, T, C, x.shape[2], 0, 0, 0, 0, K(ty), E.gemm_impl, st), "osb_gemm(q)");
    } else {
        kl = make(ty, { Tka, C }); vl = make(ty, { Tka, C });
        mha_project(i, x, &x, &ql, kl, vl, Tka);
    }

    if (use_flash) {
        // one kernel: QK^T -> online softmax -> PV with the score tile in registers
        if (ty == DType::f32) {
            // fp32: the launch first splits q, k, v into bf16 planes (6 bytes per element) in this scratch
            Tensor planes = make(DType::f16, { 3 * (T + 2 * Tk) * C });
            ck(osb_flash_attention_f32x(ql.data(), C, kl.data(), C, vl.data(), C, out.mdata(), C, h, T, Tk, d, scale, planes.mdata(), st), "osb_flash_attention_f32x");
        } else {
            ck(osb_flash_attention(ql.data(), C, kl.data(), C, vl.data(), C, out.mdata(), C, h, T, Tk, d, scale, st), "osb_flash_attention");
        }
        push(i + 19, 0, out);
        return;
    }
    int64_t per_head = T * Tkp * (int64_t)es;
    int64_t hc = std::max<int64_t>(1, std::min<int64_t>(h, ((int64_t)512 << 20) / std::max<int64_t>(per_head, 1)));
    for (int64_t h0 = 0; h0 < h; h0 += hc) {
        int64_t nh = std::min(hc, h - h0);
        Tensor S = make(ty, { nh, T, Tkp });
        const char* qp = (const char*)ql.data() + h0 * d * es;
        const char* kp = (const char*)kl.data() + h0 * d * es;
        const char* vp = (const char*)vl.data() + h0 * d * es;
        char* op_ = (char*)out.mdata() + h0 * d * es;
        // S[h] = Q[h] (T x d, rows C apart) * K[h]^T (K stored [Tkp x d], rows C apart => "B transposed")
        ck(osb_gemm_ld(qp, C, kp, C, S.mdata(), Tkp, nullptr, nullptr, nh, T, Tkp, d, d, d, T * Tkp, 1, K(ty), E.gemm_impl, st), "osb_gemm_ld(QK)");
        ck(osb_softmax_scaled_ld(S.data(), S.mdata(), K(ty), nh * T, Tk, Tkp, scale, nullptr, 1, st), "osb_softmax_scaled_ld");
        // O[:, h*d:(h+1)*d] = P[h] (T x Tkp) * V[h] (Tkp x d, rows C apart), written in place into the merged [T, C] layout
        ck(osb_gemm_ld(S.data(), Tkp, vp, C, op_, C, nullptr, nullptr, nh, T, d, Tkp, T * Tkp, d, d, 0, K(ty), E.gemm_impl, st), "osb_gemm_ld(PV)");
    }
    push(i + 19, 0, out);
}

// ScaledDotProductAttention (src/onnxstream.cpp:7767-7882): q [B,Hq,Tq,D], k [B,Hkv,Tk,D], v [B,Hkv,Tk,Dv], scale 1/s,
// additive mask [Tq,Tk] (or [1,1,Tq,Tk]); grouped KV heads supported.
void Engine::Impl::fused_sdpa(const Step& s)
{
    size_t i = s.first;
    const OpDef& op = E.m_ops[i];
    Tensor q = to_plain(in(i + 1, 0)), k = to_plain(in(i, 0)), sc = in(i + 2, 1), m = to_plain(in(i + 3, 1)), v = to_plain(in(i + 5, 1));
    if (q.shape.size() != 4) throw std::invalid_argument("ScaledDotProductAttention: invalid shape of query.");
    if (k.shape.size() != 4) throw std::invalid_argument("ScaledDotProductAttention: invalid shape of key.");
    if (v.shape.size() != 4) throw std::invalid_argument("ScaledDotProductAttention: invalid shape of value.");
    if (!(m.shape.size() == 2 || (m.shape.size() == 4 && m.shape[0] == 1 && m.shape[1] == 1)))
        throw std::invalid_argument("ScaledDotProductAttention: invalid shape of mask.");
    int64_t B = q.shape[0], Hq = q.shape[1], Tq = q.shape[2], D = q.shape[3], Hkv = k.shape[1], Tk = k.shape[2], Dv = v.shape[3];
    if (B != 1) throw std::invalid_argument("ScaledDotProductAttention: batch size != 1 (not implemented).");
    if (k.shape[3] != D || v.shape[1] != Hkv || v.shape[2] != Tk || Hkv == 0 || Hq % Hkv) throw std::runtime_error("XnnPack::scaled_dot_product_attention: invalid size of key.");
    if (m.numel() != Tq * Tk) throw std::runtime_error("XnnPack::scaled_dot_product_attention: invalid size of mask.");
    float sval = scalar_of(sc, op);
    float scale;
    if (q.type == DType::f16) { sval = __half2float(__float2half_rn(sval)); scale = __half2float(__float2half_rn(1.0f / sval)); }   // fp16 path rounds the scale (cpp:7849-7866)
    else scale = 1.0f / sval;
    if (k.type != q.type) k = convert(k, q.type);
    if (v.type != q.type) v = convert(v, q.type);
    if (m.type != q.type) m = convert(m, q.type);
    Tensor out = make(q.type, { B, Hq, Tq, Dv });
    Tensor q3 = q, k3 = k, v3 = v;
    q3.shape = { Hq, Tq, D }; k3.shape = { Hkv, Tk, D }; v3.shape = { Hkv, Tk, Dv };
    Tensor o3 = out; o3.shape = { Hq, Tq, Dv };
    // prompt prefill (more query rows than the decode kernels take): one fused wgmma kernel for all the grouped heads
    const bool aligned = ((((uintptr_t)q.data() | (uintptr_t)k.data() | (uintptr_t)v.data() | (uintptr_t)out.data()) & 15) == 0) && (((uintptr_t)m.data() & 3) == 0);
    if (q.type == DType::f16 && Tq > 16 && D == Dv && flash_on() && aligned && osb_sdpa_flash_ok(Hq, Hkv, Tq, Tk, D, Dv, K(q.type))) {
        ck(osb_sdpa_flash(q.data(), k.data(), v.data(), m.data(), out.mdata(), Hq, Hkv, Tq, Tk, D, scale, st), "osb_sdpa_flash");
        push(i + 5, 0, out);
        return;
    }
    // fp32 arithmetic: the same grouped-KV flash attention on the bf16 tensor cores at fp32 accuracy, for grouped and equal head counts
    // alike (instead of the per-row kernel, or the GEMM -> softmax -> GEMM chain and its fp32 [Hq, Tq, Tk] score buffer)
    if (q.type == DType::f32 && Tq > 16 && D == Dv && flash_on() && aligned && osb_sdpa_flash_f32x_ok(Hq, Hkv, Tq, Tk, D, Dv, K(q.type))) {
        // the launch splits q, k, v into bf16 planes (6 bytes per element) in this scratch
        Tensor planes = make(DType::f16, { 3 * (Hq * Tq + 2 * Hkv * Tk) * D });
        ck(osb_sdpa_flash_f32x(q.data(), k.data(), v.data(), m.data(), out.mdata(), Hq, Hkv, Tq, Tk, D, scale, planes.mdata(), st), "osb_sdpa_flash_f32x");
        push(i + 5, 0, out);
        return;
    }
    attention_core(q3, k3, v3, scale, false, &m, Hq / Hkv, o3);
    push(i + 5, 0, out);
}

void Engine::Impl::fused_groupnorm(const Step& s)
{
    size_t i = s.first;
    const OpDef& inrm = E.m_ops[i + 1];
    float eps = 1e-5f;
    for (auto& a : inrm.attrs) { if (a.first == "epsilon") eps = std::stof(a.second); else fail(inrm, "unrecognized attribute: " + a.first + "."); }
    Tensor x = in(i, 0);
    // statistics the producer step left in the current ring slot; whoever does not consume them must zero the slot again
    const bool pre = stats_ready_for == (long)cur_step;
    stats_ready_for = -1;
    auto drop_pre = [&] { if (pre) { ck(cudaMemsetAsync(gn_slot_ptr(gn_slot), 0, 1024, st), "cudaMemsetAsync(gn slot)"); gn_slot_used[gn_slot] = 0; } };
    (void)in(i, 1); (void)in(i + 2, 1);  // the two shape constants (validated statically by the matcher)
    Tensor gs = in(i + 1, 1), gb = in(i + 1, 2), gamma = in(i + 3, 1), beta = in(i + 4, 1);
    int64_t C = x.shape[1], HW = x.numel() / C;
    int G = (int)E.m_ops[i].out[0].shape[1];
    bool unit = gs.host_f32 && gb.host_f32;
    if (unit) { for (auto f : *gs.host_f32) if (f != 1.f) unit = false; for (auto f : *gb.host_f32) if (f != 0.f) unit = false; }
    if (!unit) {
        // non-trivial per-group affine: fold into per-channel gamma/beta on the host mirror is not possible for large C;
        // fall back to the unfused sequence for this group.
        drop_pre();
        exec_unfused(s);
        return;
    }
    if (x.type != DType::f16 && x.type != DType::f32) fail(inrm, "wrong data type of input.");
    if (gamma.type != x.type) gamma = convert(gamma, x.type);
    if (beta.type != x.type) beta = convert(beta, x.type);
    Tensor y = make(x.type, x.shape, x.layout);
    if (gn_split_enabled() && cur_B == 1 && gn_ring && gn_apply_ok(x, C, G)) {
        // statistics: already in the current ring slot (gathered by the producing conv / Add), or one atomics pass now; then ONE
        // streaming apply pass that also zeroes the other slot for the next producer -- no grid rendezvous, no co-residency assumption
        bool have = pre;
        if (!have) have = osb_channel_add_stats(x.data(), nullptr, nullptr, K(x.type), C, HW, G, gn_slot_ptr(gn_slot), st) == 0;
        if (have) {
            gn_slot_used[gn_slot] = std::max(gn_slot_used[gn_slot], 2 * G);
            ck(osb_group_norm_apply(x.data(), y.mdata(), K(x.type), C, HW, G, gamma.data(), beta.data(), eps, s.count == 7 ? 1 : 0,
                                    gn_slot_ptr(gn_slot), gn_slot_ptr(gn_slot ^ 1), st), "osb_group_norm_apply");
            int& other = gn_slot_used[gn_slot ^ 1];
            if (other > 2 * G)
                ck(cudaMemsetAsync(gn_slot_ptr(gn_slot ^ 1) + 2 * G, 0, (size_t)(other - 2 * G) * sizeof(double), st), "cudaMemsetAsync(gn slot tail)");
            other = 0;
            gn_slot ^= 1;
            push(s.first + s.count - 1, 0, y);
            return;
        }
    }
    drop_pre();
    if (!gn_stats) { gn_stats = E.m_pool.alloc(2048); ck(cudaMemsetAsync(gn_stats->ptr, 0, 2048, st), "cudaMemsetAsync(gn scratch)"); }
    ck(osb_group_norm(x.data(), y.mdata(), K(x.type), x.layout == Layout::nhwc ? 1 : 0, C, HW, G, gamma.data(), beta.data(), eps, s.count == 7 ? 1 : 0,
                      gn_stats->ptr, st), "osb_group_norm");
    push(s.first + s.count - 1, 0, y);
}

void Engine::Impl::fused_rmsnorm(const Step& s)
{
    const size_t i = s.first;
    const OpDef& pw = E.m_ops[i];
    // the kernel reads fp16 or fp32 and computes in fp32 either way: no up-cast copy of the input (in() would make one for an
    // m_requires_upcast op); quantised storage goes through in() as usual
    Tensor x = get_act(pw, pw.in[0].name);
    if (x.type != DType::f16 && x.type != DType::f32) x = in(i, 0);
    x = to_plain(x);
    const float two = scalar_of(in(i, 1), pw), eps = scalar_of(in(i + 2, 1), E.m_ops[i + 2]), one = scalar_of(in(i + 4, 0), E.m_ops[i + 4]);
    if (two != 2.f || one != 1.f || (x.type != DType::f16 && x.type != DType::f32)) { exec_unfused(s); return; }
    const OpDef& m2 = E.m_ops[i + 6];
    const size_t wi = is_float_weight(m2.in[0]) ? 0 : 1;
    Tensor w = in(i + 6, wi);
    // arithmetic class of the chain: fp32 when the ops are up-cast (m_requires_upcast) or the model runs fp32; the result type is what the
    // last Mul would have produced (push() then applies the storage rule)
    DType ot = (upcast_op(m2) || !E.use_fp16_arithmetic) ? DType::f32 : x.type;
    // push() would round an fp32 result to fp16 storage right away unless the next step is its only consumer: write those bits directly
    // (one rounding of the same fp32 value either way)
    if (ot == DType::f32 && E.use_fp16_arithmetic && !E.use_uint8_arithmetic && !E.use_uint8_qdq && !E.range_data_calibrate &&
        !next_is_sole_consumer(cur_step, m2.out[0].name)) ot = DType::f16;
    if (w.type != DType::f16 && w.type != DType::f32) { exec_unfused(s); return; }
    Tensor y = make(ot, x.shape);
    if (osb_rms_norm(x.data(), K(x.type), w.data(), K(w.type), y.mdata(), K(ot), x.numel() / x.shape.back(), x.shape.back(), eps, st) != 0) {
        // an unsupported type mix: the generic ops
        exec_unfused(s);
        return;
    }
    push(i + 6, 0, y);
}

void Engine::Impl::fused_rope(const Step& s)
{
    const size_t i = s.first;
    Tensor x = to_plain(in(i, 0));
    const int64_t D = x.shape.back(), nd = (int64_t)x.shape.size();
    // the Slice constants must really cut [0, D/2) and [D/2, D) of the last axis
    auto cut = [&](size_t oi, int64_t lo, int64_t hi) {
        Tensor st_ = in(oi, 1), en = in(oi, 2), ax = in(oi, 3), sp = in(oi, 4);
        if (st_.i64->size() != 1 || en.i64->size() != 1 || ax.i64->size() != 1 || sp.i64->size() != 1) return false;
        int64_t a = (*ax.i64)[0]; if (a < 0) a += nd;
        int64_t e = (*en.i64)[0]; if (e > D) e = D;
        return a == nd - 1 && (*sp.i64)[0] == 1 && (*st_.i64)[0] == lo && e == hi;
    };
    Tensor cs = to_plain(in(i + 4, 1)), sn = to_plain(in(i + 5, 1));
    // one table row for every x row, or one per position (x [.., T, D], table [T, D] broadcast over the leading dims)
    const int64_t T = nd >= 2 ? x.shape[nd - 2] : 1;
    const int64_t table_rows = cs.numel() / std::max<int64_t>(D, 1);
    const bool table_ok = (table_rows == 1 || table_rows == T) && cs.numel() == table_rows * D && sn.numel() == cs.numel();
    if (!cut(i, 0, D / 2) || !cut(i + 1, D / 2, D) || (x.type != DType::f16 && x.type != DType::f32) || !table_ok) { exec_unfused(s); return; }
    if (cs.type != x.type) cs = convert(cs, x.type);
    if (sn.type != x.type) sn = convert(sn, x.type);
    Tensor y = make(x.type, x.shape);
    ck(osb_rope(x.data(), cs.data(), sn.data(), y.mdata(), K(x.type), x.numel() / D, D, table_rows, st), "osb_rope");
    push(i + 6, 0, y);
}

// bf16 triple-split expansion of an fp32 operand for the tensor-core fp32 path (include/onnxstream_b200_kernels.h: osb_tc_gemm_f32x).
// by_rows: [K = rows][N = L] -> [6 K][N]; otherwise rows of length L -> rows of length 6 L.  A static weight of a resident model is expanded
// once and kept with the resident weights (cache_key non-empty).
Tensor Engine::Impl::f32x_operand(const Tensor& t, int64_t rows, int64_t L, bool by_rows, int b_side, const std::string& cache_key)
{
    const bool cache = E.resident_weights && !cache_key.empty();
    if (cache) { auto it = resident.find(cache_key); if (it != resident.end()) return it->second; }
    Tensor e = make(DType::f16, { rows, 6 * L });          // bfloat16 payload in a 2-byte container type
    if (by_rows) ck(osb_bf16x3_expand_rows(t.data(), e.mdata(), rows, L, b_side, st), "osb_bf16x3_expand_rows");
    else ck(osb_bf16x3_expand_cols(t.data(), e.mdata(), rows, L, L, b_side, st), "osb_bf16x3_expand_cols");
    if (cache) { resident[cache_key] = e; resident_bytes += (size_t)(rows * 6 * L) * 2; }
    return e;
}

// n (2 or 3) MatMul nodes x[rows <= 8, K] . W_g[K, N_g] sharing x: one grouped GEMV launch.  false = not expressible (the caller runs the
// nodes one by one); nothing has been pushed in that case.
bool Engine::Impl::gemv_group(const Tensor& a, const size_t* op_idx, int n, Tensor* outs)
{
    if (a.type != DType::f16 && a.type != DType::f32) return false;
    const int64_t rows = act_rows(a), Kd = a.shape.back();
    static const bool grouped = [] { const char* e = getenv("OSB_GEMV_GROUPED"); return !(e && e[0] == '0'); }();
    if (!grouped) return false;
    // one stored-blob GEMV for every member, or else the float GEMV on converted weights
    bool u8 = true, flt = true, f16w = true;
    for (int g = 0; g < n; g++) {
        const OpDef& op = E.m_ops[op_idx[g]];
        const TensorRef& wr = op.in[1];
        if (wr.shape[0] != Kd) return false;
        const WRoute r = weight_route(op, a);
        u8 = u8 && r == WRoute::u8_gemv;
        flt = flt && (wr.wtype != DType::u8 || !w8_gemv_on()) && wr.shape[1] % 8 == 0 && wr.shape[1] >= 256;
        f16w = f16w && r == WRoute::f16_gemv;
    }
    if (!u8 && !flt) return false;
    const void* B[3]; void* C[3]; int64_t N[3]; float ws[3]; int wz[3];
    Tensor wt[3];
    for (int g = 0; g < n; g++) {
        const OpDef& op = E.m_ops[op_idx[g]];
        wt[g] = (u8 || f16w) ? weight1(op_idx[g], true, false) : in(op_idx[g], 1);
        if (!u8 && !f16w && wt[g].type != a.type) wt[g] = convert(wt[g], a.type);
        std::vector<int64_t> os = a.shape; os.back() = op.in[1].shape[1];
        outs[g] = make(a.type, os);
        B[g] = wt[g].data(); C[g] = outs[g].mdata(); N[g] = op.in[1].shape[1]; ws[g] = wt[g].scale; wz[g] = wt[g].zero_point;
    }
    const int rc = osb_gemv_grouped(a.data(), B, C, N, ws, wz, n, rows, Kd, u8 ? OSB_U8 : (f16w ? OSB_F16 : K(a.type)), K(a.type), st);
    if (rc == (int)cudaErrorNotSupported) return false;
    ck(rc, "osb_gemv_grouped");
    return true;
}

void Engine::Impl::fused_gemv_group(const Step& s)
{
    Tensor a = to_plain(in(s.first, 0));
    size_t idx[3]; Tensor outs[3];
    for (size_t g = 0; g < s.count; g++) idx[g] = s.first + g;
    if (!gemv_group(a, idx, (int)s.count, outs)) {
        // every MatMul of the group has consumers outside it: run them one by one and keep all outputs (exec_unfused would drop the
        // "intermediates" of a fusion group)
        for (size_t g = 0; g < s.count; g++) exec_single(idx[g]);
        return;
    }
    for (size_t g = 0; g < s.count; g++) push(idx[g], 0, outs[g]);
}

void Engine::Impl::fused_swiglu(const Step& s)
{
    const size_t i = s.first;
    Tensor a = to_plain(in(i, 0));
    size_t idx[2] = { i, i + 3 }; Tensor outs[2];
    if (!gemv_group(a, idx, 2, outs)) { exec_unfused(s); return; }
    // silu(gate) * up in fp32, one rounding (the fused-step convention of this engine: GELU, GEGLU, SiLU behave the same way)
    Tensor y = make(a.type, outs[0].shape);
    const int64_t n = y.numel(), one = 1;
    ck(osb_binary(OSB_BIN_SILU_MUL, outs[0].data(), &one, outs[1].data(), &one, y.mdata(), &n, 1, K(a.type), st), "osb_binary(silu_mul)");
    push(i + 4, 0, y);
}

void Engine::Impl::fused_layernorm(const Step& s)
{
    size_t i = s.first;
    // the planner accepts any scalar exponent; only 2 is a LayerNorm: any other runs as the ops it is
    if (scalar_of(in(i + 2, 1), E.m_ops[i + 2]) != 2.f) { exec_unfused(s); return; }
    Tensor x = to_plain(in(i, 0));
    Tensor eps_t = in(i + 4, 1), gamma = in(i + 7, 1), beta = in(i + 8, 1);
    float eps = scalar_of(eps_t, E.m_ops[i + 4]);
    if (gamma.type != x.type) gamma = convert(gamma, x.type);
    if (beta.type != x.type) beta = convert(beta, x.type);
    Tensor y = make(x.type, x.shape);
    ck(osb_layer_norm(x.data(), y.mdata(), K(x.type), x.numel() / x.shape.back(), x.shape.back(), gamma.data(), beta.data(), eps, st), "osb_layer_norm");
    push(i + 8, 0, y);
}

void Engine::Impl::fused_gelu(const Step& s)
{
    size_t i = s.first;
    Tensor x = in(i, 0);
    float c0 = scalar_of(in(i, 1), E.m_ops[i]), c1 = scalar_of(in(i + 2, 1), E.m_ops[i + 2]), c2 = scalar_of(in(i + 4, 1), E.m_ops[i + 4]);
    if (std::fabs(c0 - 1.41421356f) > 1e-3f || c1 != 1.f || c2 != 0.5f) {
        exec_unfused(s);
        return;
    }
    if (s.count == 6) {
        Tensor a = in(i + 5, 0);
        push(i + 5, 0, binary(OSB_BIN_MUL_GELU, a, x));
    } else {
        Tensor y = make(x.type, x.shape, x.layout);
        ck(osb_unary(OSB_UN_GELU_ERF, x.data(), y.mdata(), K(x.type), (size_t)x.numel(), 0.f, st), "osb_unary(gelu)");
        push(i + 4, 0, y);
    }
}

void Engine::Impl::fused_geglu(const Step& s)
{
    // a 10-op step starts with the FF-in MatMul + bias Add (plan.cpp: geglu); the gate's 8 ops follow from op i
    const size_t lead = s.count == 10 ? 2 : 0, i = s.first + lead;
    // Slice op oi cuts [lo, hi) of the last axis of a rank-`rank` tensor whose last axis has n entries
    auto cuts = [&](size_t oi, int64_t rank, int64_t n, int64_t lo, int64_t hi) {
        Tensor st_ = in(oi, 1), en = in(oi, 2), ax = in(oi, 3), sp = in(oi, 4);
        if (!st_.i64 || !en.i64 || !ax.i64 || !sp.i64 || st_.i64->size() != 1 || en.i64->size() != 1 || ax.i64->size() != 1 || sp.i64->size() != 1) return false;
        int64_t a = (*ax.i64)[0], b = (*st_.i64)[0], e = (*en.i64)[0];
        if (a < 0) a += rank;
        if (b < 0) b += n;
        if (e < 0) e += n;
        return a == rank - 1 && (*sp.i64)[0] == 1 && b == lo && std::min(e, n) == hi;
    };
    // the halves of a rank-`rank` [.., n] tensor, and the constants of the erf GELU
    auto gate_ok = [&](int64_t rank, int64_t n) {
        float c0 = scalar_of(in(i + 2, 1), E.m_ops[i + 2]), c1 = scalar_of(in(i + 4, 1), E.m_ops[i + 4]), c2 = scalar_of(in(i + 6, 1), E.m_ops[i + 6]);
        return n >= 2 && n % 2 == 0 && cuts(i, rank, n, 0, n / 2) && cuts(i + 1, rank, n, n / 2, n) && std::fabs(c0 - 1.41421356f) <= 1e-3f && c1 == 1.f && c2 == 0.5f;
    };
    if (lead) {
        const size_t mm = s.first;
        Tensor a = to_plain(in(mm, 0)), bias = in(mm + 1, (size_t)s.bias_in);
        const TensorRef& wr = E.m_ops[mm].in[1];
        const int64_t Kd = wr.shape[0], inner = wr.shape[1] / 2, M = !a.shape.empty() && a.shape.back() == Kd && Kd > 0 ? act_rows(a) : 0;
        // not the two halves (or an unexpected constant): all ten ops by their own handlers, the bias Add included -- a bias in the GEMM
        // epilogue would round once where the MatMul and the Add round twice
        if (!gate_ok((int64_t)a.shape.size(), wr.shape[1])) { exec_unfused(s); return; }
        if (a.type == DType::f16 && E.gemm_impl != 1 && M > 0) {
            Tensor w = in(mm, 1);
            if (w.type != a.type) w = convert(w, a.type);
            if (bias.type != a.type) bias = convert(bias, a.type);
            std::vector<int64_t> os = a.shape; os.back() = inner;
            Tensor y = make(a.type, os);
            const int rc = osb_tc_gemm_geglu(a.data(), w.data(), y.mdata(), bias.data(), M, inner, Kd, st);
            if (rc != (int)cudaErrorNotSupported) {
                ck(rc, "osb_tc_gemm_geglu");
                push(i + 7, 0, y);
                return;
            }
        }
        op_matmul(mm, &bias, nullptr, mm + 1);     // the unfused chain: the bias GEMM, then the gate pass below
    }
    Tensor x = in(i, 0);
    const int64_t n2 = x.shape.empty() ? 0 : x.shape.back(), inner = n2 / 2;
    if (!((x.type == DType::f16 || x.type == DType::f32) && x.layout == Layout::plain && gate_ok((int64_t)x.shape.size(), n2))) {
        // not the two halves (or an unexpected constant): run the group with the ordinary handlers
        exec_unfused(s, lead);
        return;
    }
    std::vector<int64_t> os = x.shape; os.back() = inner;
    Tensor y = make(x.type, os);
    ck(osb_geglu(x.data(), y.mdata(), K(x.type), x.numel() / n2, inner, st), "osb_geglu");
    push(i + 7, 0, y);
    if (lead && cur_b + 1 == cur_B) {   // the GEMM's [.., 2 inner] result has no consumer outside the step
        const std::string& xn = E.m_ops[s.first + 1].out[0].name;
        store.erase(xn);
        order.erase(std::remove(order.begin(), order.end(), xn), order.end());
    }
}

void Engine::Impl::fused_silu(const Step& s)
{
    const std::string in_name = E.m_ops[s.first].in[0].name;
    Tensor x = in(s.first, 0);
    if (x.type != DType::f16 && x.type != DType::f32) fail(E.m_ops[s.first], "wrong data type of input.");
    // Every resnet block of a UNet applies SiLU to the same time embedding: tensor names are single-assignment, so the result
    // for (name, batch sibling) is computed once per run and aliased afterwards (small tensors only -- the cache pins memory).
    const bool cacheable = x.numel() <= 65536;
    const std::string key = in_name + "#" + std::to_string(cur_b);
    if (cacheable) {
        auto it = silu_cache.find(key);
        if (it != silu_cache.end() && it->second.type == x.type && it->second.shape == x.shape && it->second.layout == x.layout) {
            push(s.first + 1, 0, it->second);
            return;
        }
    }
    Tensor y = make(x.type, x.shape, x.layout);
    ck(osb_unary(OSB_UN_SILU, x.data(), y.mdata(), K(x.type), (size_t)x.numel(), 0.f, st), "osb_unary(silu)");
    if (cacheable) silu_cache[key] = y;
    push(s.first + 1, 0, y);
}

void Engine::Impl::fused_linear(const Step& s)
{
    const size_t last = s.first + s.count - 1;
    Tensor bias, res;
    if (s.bias_in >= 0) bias = in(s.first + 1, (size_t)s.bias_in);
    if (s.residual_in >= 0) res = in(last, (size_t)s.residual_in);
    op_matmul(s.first, s.bias_in >= 0 ? &bias : nullptr, s.residual_in >= 0 ? &res : nullptr, last);
}

void Engine::Impl::exec_single(size_t oi)
{
    const OpDef& op = E.m_ops[oi];
    const std::string& t = op.type;
    if (t == "Conv") op_conv(oi);
    else if (t == "MatMul") op_matmul(oi);
    else if (t == "Gemm") op_gemm(oi);
    else if (t == "Add") op_binary(oi, OSB_BIN_ADD);
    else if (t == "Sub") op_binary(oi, OSB_BIN_SUB);
    else if (t == "Mul") op_binary(oi, OSB_BIN_MUL);
    else if (t == "Div") op_binary(oi, OSB_BIN_DIV);
    else if (t == "Sigmoid") op_unary(oi, OSB_UN_SIGMOID);
    else if (t == "Erf") op_unary(oi, OSB_UN_ERF);
    else if (t == "Sqrt") op_unary(oi, OSB_UN_SQRT);
    else if (t == "Sin") op_unary(oi, OSB_UN_SIN);
    else if (t == "Cos") op_unary(oi, OSB_UN_COS);
    else if (t == "Neg") op_unary(oi, OSB_UN_NEG);
    else if (t == "Pow") {
        if (op.in.size() != 2) fail(op, "wrong number of inputs.");
        Tensor x = in(oi, 0), e = in(oi, 1);
        float ex = scalar_of(e, op);
        Tensor y = make(x.type, x.shape, x.layout);
        ck(osb_unary(OSB_UN_POW, x.data(), y.mdata(), K(x.type), (size_t)x.numel(), ex, st), "osb_unary(pow)");
        push(oi, 0, y);
    }
    else if (t == "Reshape" || t == "Unsqueeze" || t == "Squeeze" || t == "Flatten") op_reshape_like(oi);
    else if (t == "Transpose") op_transpose(oi);
    else if (t == "Concat") op_concat(oi);
    else if (t == "Split") op_split(oi);
    else if (t == "Slice") op_slice(oi);
    else if (t == "Resize") op_resize(oi);
    else if (t == "Softmax") op_softmax(oi);
    else if (t == "InstanceNormalization") op_instnorm(oi);
    else if (t == "ReduceMean") op_reduce_mean(oi);
    else if (t == "Gather") op_gather(oi);
    else op_misc_host(oi);
}

void Engine::Impl::exec_step(size_t si)
{
    const Step& s = plan.steps[si];
    cur_step = si;
    wcache.clear();
    // batch size of this step = number of siblings of its activation inputs (src/onnxstream.cpp:3817-3842)
    cur_B = 1;
    for (size_t oi = s.first; oi < s.first + s.count; oi++)
        for (auto& r : E.m_ops[oi].in) if (r.present && r.wtype == DType::none) {
            size_t b = batch_of(r.name);
            if (b > 1) { if (cur_B > 1 && cur_B != b) fail(E.m_ops[oi], "inconsistent m_batch.size() across two or more tensors."); cur_B = b; }
        }
    pump_weights();
    stats_want = -1;
    if (E.fuse_nodes && plan.stats_consumer[si] >= 0) {
        const Step& gs = plan.steps[(size_t)plan.stats_consumer[si]];
        stats_want = plan.stats_consumer[si];
        stats_groups = (int)E.m_ops[gs.first].out[0].shape[1];
    }
    if (E.ops_printf) for (size_t oi = s.first; oi < s.first + s.count; oi++) printf("#%zu) %s (%s)%s\n", oi, E.m_ops[oi].type.c_str(), E.m_ops[oi].name.c_str(), s.count > 1 ? " [fused]" : "");
    cudaEvent_t tev0 = nullptr, tev1 = nullptr;
    if (E.ops_times_printf) {
        // m_ops_times_printf (src/onnxstream.cpp:3812, 8199-8214): time per op TYPE; here the device time of the step's kernels
        // (cudaEvent pair on the compute stream; the step is attributed to its first op's type, fused groups to "<type>+")
        ck(cudaEventCreate(&tev0), "cudaEventCreate"); ck(cudaEventCreate(&tev1), "cudaEventCreate");
        ck(cudaEventRecord(tev0, st), "cudaEventRecord");
    }
    for (cur_b = 0; cur_b < cur_B; cur_b++) {
        switch (s.kind) {
        case SK_ATTENTION: fused_attention(s); break;
        case SK_GROUPNORM: fused_groupnorm(s); break;
        case SK_LAYERNORM: fused_layernorm(s); break;
        case SK_GELU: fused_gelu(s); break;
        case SK_GEGLU: fused_geglu(s); break;
        case SK_SILU: fused_silu(s); break;
        case SK_LINEAR: fused_linear(s); break;
        case SK_SDPA: fused_sdpa(s); break;
        case SK_MHA: fused_mha(s); break;
        case SK_RMSNORM: fused_rmsnorm(s); break;
        case SK_GEMV_GROUP: fused_gemv_group(s); break;
        case SK_SWIGLU: fused_swiglu(s); break;
        case SK_ROPE: fused_rope(s); break;
        case SK_CONV_ADD: { Tensor res = in(s.first + 1, (size_t)s.residual_in); op_conv(s.first, &res, s.first + 1); break; }
        default: exec_single(s.first); break;
        }
    }
    cur_b = 0;
    // release this step's weight slots (the consumer kernels are enqueued) and drop consumed activations
    if (E.m_streamer) {
        for (size_t oi = s.first; oi < s.first + s.count; oi++)
            for (size_t k = 0; k < E.m_ops[oi].in.size(); k++) staged.erase({ oi, k });
        auto sl = step_slot.find(si);
        if (sl != step_slot.end()) { E.m_streamer->release(sl->second, st); step_slot.erase(sl); }
    }
    if (tev0) {
        ck(cudaEventRecord(tev1, st), "cudaEventRecord");
        op_times.push_back({ E.m_ops[s.first].type + (s.count > 1 ? "+" : ""), tev0, tev1 });
    }
    wcache.clear();
    consume_inputs(s);
    E.m_stats.ops_executed += 1;
    E.m_stats.ops_fused_away += s.count - 1;
}

// ================================================================================================================
// Engine
// ================================================================================================================

Engine::Engine(int device)
{
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        throw std::runtime_error("onnxstream_b200: no CUDA device available -- this engine has no CPU fallback (" + std::string(cudaGetErrorString(e)) + ")");
    if (device < 0) { cudaGetDevice(&device); }
    m_device = device;
    check_cuda(cudaSetDevice(m_device), "cudaSetDevice");
    cudaStream_t s;
    check_cuda(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), "cudaStreamCreate");
    m_stream = s;
    m_impl = std::make_unique<Impl>(*this);
}

Engine::~Engine()
{
    cudaStreamSynchronize(m_stream);
    drop_graph();
    m_impl.reset();
    m_streamer.reset();
    osb_workspace_release(m_stream); cudaStreamDestroy(m_stream);
}

void Engine::set_weight_source(std::unique_ptr<WeightSource> src)
{
    if (m_source) throw std::invalid_argument("Model::set_weights_provider: weights provider already set.");
    m_source = std::move(src);
}

void Engine::read_file(const char* filename)
{
    FILE* f = fopen(filename, "rb");
    if (!f) throw std::runtime_error("read_file: unable to open file (" + std::string(filename) + ").");
    fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
    if (sz <= 0) { fclose(f); throw std::invalid_argument("read_file: invalid size of file."); }
    std::string text((size_t)sz, '\0');
    size_t got = fread(&text[0], 1, (size_t)sz, f);
    fclose(f);
    if (got != (size_t)sz) throw std::runtime_error("read_file: unable to read file.");
    m_text = std::move(text);
    m_path.clear();
    std::string fn(filename);
    size_t sep = fn.find_last_of("/\\");
    if (sep != std::string::npos) m_path = fn.substr(0, sep + 1);
    m_parsed = false;
    if (!m_source) m_source = make_disk_source(true);
    m_source->path = m_path;
}

void Engine::read_string(const char* text, const char* path_with_slash)
{
    m_text = text;
    m_path = path_with_slash;
    m_parsed = false;
    if (!m_source) m_source = make_disk_source(true);
    m_source->path = m_path;
}

void Engine::parse()
{
    if (m_parsed) return;
    m_ops = parse_model_text(m_text, support_dynamic_shapes);
    m_parsed = true;
    invalidate_plan();
}

// A different model text or different options: nothing derived from the old plan may survive -- the captured graph, the HBM weight
// cache (keyed by file name + dtype only), the step list and the per-run scratch.
void Engine::invalidate_plan()
{
    cudaStreamSynchronize(m_stream);
    drop_graph();
    m_first_run = true;
    m_refs_initial.clear();
    Impl& I = *m_impl;
    I.resident.clear(); I.resident_bytes = 0;
    I.plan = Plan{};
    I.staged.clear(); I.step_slot.clear();
    I.store.clear(); I.order.clear(); I.silu_cache.clear();
    I.runs_done = 0;
    m_streamer.reset();
}

// every knob that changes the plan, the dtype of a tensor or the set of outputs
std::string Engine::options_signature() const
{
    std::string s;
    auto b = [&](bool v) { s += v ? '1' : '0'; };
    b(use_fp16_arithmetic); b(use_uint8_qdq); b(use_uint8_arithmetic); b(fuse_ops_in_attention); b(force_fp16_storage);
    b(support_dynamic_shapes); b(use_scaled_dp_attn_op); b(use_nchw_convs); b(resident_weights); b(fuse_nodes); b(keep_nhwc); b(flash_attention);
    b((bool)requires_upcast); b(keep_inputs); b(drop_unconverted_outputs);
    s += std::to_string(gemm_impl); s += '|'; s += std::to_string(attention_fused_ops_parts); s += '|';
    for (auto& e : extra_outputs) { s += e; s += ','; }
    s += '|';
    for (auto& e : outputs_convert_set) { s += e; s += ','; }
    s += '|';
    for (auto& e : force_uint8_storage_set) { s += e; s += ','; }
    return s;
}

std::vector<std::pair<DType, std::string>> Engine::weights_names()
{
    auto ops = parse_model_text(m_text, true);
    std::vector<std::pair<DType, std::string>> out;
    for (auto& op : ops) for (auto& r : op.in) if (r.present && r.wtype != DType::none) {
        bool conv; out.emplace_back(r.wtype, Impl::weight_file(r, conv));
    }
    return out;
}

void* Engine::push_input(const std::string& name, DType type, const std::vector<size_t>& shape)
{
    HostTensor t;
    t.name = name; t.type = type; t.shape = shape;
    size_t n = 1; for (auto d : shape) n *= d;
    if (type != DType::f32 && type != DType::i64 && type != DType::f16) throw std::invalid_argument("Unsupported tensor data format.");
    t.count = n;
    t.buf = std::make_shared<PinnedBuf>(n * dtype_size(type));
    m_host_tensors.push_back(std::move(t));
    return m_host_tensors.back().buf->ptr;
}

void Engine::clear_tensors() { m_host_tensors.clear(); }

void Engine::set_comm(ncclComm* comm, int rank, int nranks) { m_comm = comm; m_rank = rank; m_nranks = nranks; }

void Engine::read_range_data(const char* filename)
{
    FILE* f = fopen(filename, "rb");
    if (!f) throw std::runtime_error("read_file: unable to open file (" + std::string(filename) + ").");
    char line[4096];
    range_data.clear();
    while (fgets(line, sizeof(line), f)) {
        std::string s(line);
        while (!s.empty() && (s.back() == '\n' || s.back() == '\r' || s.back() == ' ')) s.pop_back();
        if (s.empty()) continue;
        size_t c2 = s.rfind(','), c1 = c2 == std::string::npos ? c2 : s.rfind(',', c2 - 1);
        if (c1 == std::string::npos) { fclose(f); throw std::invalid_argument("Model::read_range_data: invalid format."); }
        range_data[s.substr(0, c1)] = { std::stof(s.substr(c1 + 1, c2 - c1 - 1)), std::stof(s.substr(c2 + 1)) };
    }
    fclose(f);
}

void Engine::write_range_data(const char* filename)
{
    FILE* f = fopen(filename, "wb");
    if (!f) throw std::runtime_error("write_file: unable to open file.");
    for (auto& kv : range_data) fprintf(f, "%s,%.9g,%.9g\n", kv.first.c_str(), kv.second.first, kv.second.second);
    fclose(f);
}

// ---- CUDA graph state (one captured run, replayed while the inputs keep their names and shapes) ----
struct GraphState {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    struct In { std::string name; std::vector<size_t> shape; DevPtr dev; size_t bytes; DType type; };
    struct Out { std::string name; std::vector<size_t> shape; DevPtr dev; size_t count; DType type; };
    std::vector<In> inputs;
    std::vector<Out> outputs;
    std::vector<DevPtr> keepalive;
    bool ready = false;
    bool failed = false;
};
static std::map<Engine*, GraphState> g_graphs;

void Engine::drop_graph()
{
    auto it = g_graphs.find(this);
    if (it == g_graphs.end()) return;
    if (it->second.exec) cudaGraphExecDestroy(it->second.exec);
    if (it->second.graph) cudaGraphDestroy(it->second.graph);
    g_graphs.erase(it);
}

bool Engine::try_replay()
{
    auto it = g_graphs.find(this);
    if (it == g_graphs.end() || !it->second.ready) return false;
    GraphState& G = it->second;
    // same inputs (names, shapes, order)?
    std::vector<HostTensor*> fins;
    for (auto& h : m_host_tensors) fins.push_back(&h);
    if (fins.size() != G.inputs.size()) { drop_graph(); return false; }
    for (size_t i = 0; i < fins.size(); i++)
        if (fins[i]->type != G.inputs[i].type || fins[i]->name != G.inputs[i].name || fins[i]->shape != G.inputs[i].shape) { drop_graph(); return false; }
    auto t0 = std::chrono::high_resolution_clock::now();
    cudaEvent_t ev0, ev1;
    check_cuda(cudaEventCreate(&ev0), "cudaEventCreate");
    check_cuda(cudaEventCreate(&ev1), "cudaEventCreate");
    check_cuda(cudaEventRecord(ev0, m_stream), "cudaEventRecord");
    m_stats.h2d_input_bytes = 0;
    for (size_t i = 0; i < fins.size(); i++) {
        check_cuda(cudaMemcpyAsync(G.inputs[i].dev->ptr, fins[i]->buf->ptr, G.inputs[i].bytes, cudaMemcpyHostToDevice, m_stream), "input H2D");
        m_stats.h2d_input_bytes += G.inputs[i].bytes;
    }
    check_cuda(cudaGraphLaunch(G.exec, m_stream), "cudaGraphLaunch");
    std::vector<HostTensor> outs;
    m_stats.d2h_output_bytes = 0;
    for (auto& o : G.outputs) {
        HostTensor h;
        h.name = o.name; h.type = o.type; h.shape = o.shape; h.count = o.count;
        const size_t ob = o.count * dtype_size(o.type);
        h.buf = std::make_shared<PinnedBuf>(ob);
        check_cuda(cudaMemcpyAsync(h.buf->ptr, o.dev->ptr, ob, cudaMemcpyDeviceToHost, m_stream), "output D2H");
        m_stats.d2h_output_bytes += ob;
        outs.push_back(std::move(h));
    }
    check_cuda(cudaEventRecord(ev1, m_stream), "cudaEventRecord");
    check_cuda(cudaStreamSynchronize(m_stream), "graph replay sync");
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0, ev1);
    cudaEventDestroy(ev0); cudaEventDestroy(ev1);
    m_host_tensors = std::move(outs);
    m_stats.last_gpu_ms = ms;
    m_stats.graph_replays++;
    m_stats.weight_bytes_streamed = 0;
    m_stats.last_run_ms = std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - t0).count();
    return true;
}

double Engine::run_resident(int steps)
{
    auto it = g_graphs.find(this);
    if (it == g_graphs.end() || !it->second.ready)
        throw std::runtime_error("run_resident: no captured graph (enable b200_cuda_graph + b200_resident_weights and call run() three times first)");
    GraphState& G = it->second;
    check_cuda(cudaSetDevice(m_device), "cudaSetDevice");
    cudaEvent_t ev0, ev1;
    check_cuda(cudaEventCreate(&ev0), "cudaEventCreate");
    check_cuda(cudaEventCreate(&ev1), "cudaEventCreate");
    check_cuda(cudaStreamSynchronize(m_stream), "sync");
    check_cuda(cudaEventRecord(ev0, m_stream), "cudaEventRecord");
    for (int i = 0; i < steps; i++) check_cuda(cudaGraphLaunch(G.exec, m_stream), "cudaGraphLaunch");
    check_cuda(cudaEventRecord(ev1, m_stream), "cudaEventRecord");
    check_cuda(cudaStreamSynchronize(m_stream), "sync");
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0, ev1);
    cudaEventDestroy(ev0); cudaEventDestroy(ev1);
    m_stats.graph_replays += steps;
    return ms;
}

void Engine::run()
{
    auto t0 = std::chrono::high_resolution_clock::now();
    check_cuda(cudaSetDevice(m_device), "cudaSetDevice");
    parse();
    Impl& I = *m_impl;
    {
        std::string sig = options_signature();
        if (sig != I.plan_signature) { if (!I.plan_signature.empty()) invalidate_plan(); I.plan_signature = sig; }
    }
    if (use_cuda_graph && try_replay()) return;
    osb_launch_count_reset();

    // init(): reference counts + weight schedule (src/onnxstream.cpp:3499-3548)
    if (m_refs_initial.empty() || I.plan.steps.empty()) {
        PlanOptions o;
        o.fuse_nodes = fuse_nodes; o.fuse_attention = fuse_ops_in_attention; o.sdpa_rewrite = use_scaled_dp_attn_op;
        o.uint8_arithmetic = use_uint8_arithmetic; o.uint8_qdq = use_uint8_qdq; o.fp16_arithmetic = use_fp16_arithmetic;
        o.requires_upcast = requires_upcast; o.extra_outputs = extra_outputs;
        I.plan = make_plan(m_ops, o);
        m_refs_initial = I.plan.uses;
        if (!m_source) m_source = make_disk_source(true);
        if (!source_on_init_done) for (auto& ws : I.plan.step_weights) for (auto& w : ws) { const TensorRef& r = m_ops[w.op].in[w.in]; m_source->on_init(r.wtype, r.name, w.bytes); }
        size_t cap = (size_t)((double)I.plan.largest_step_bytes * std::max(1.0, ring_factor)) + 4096;
        m_streamer = std::make_unique<WeightStreamer>(cap, !m_source->stable_pinned(), m_comm, m_rank, m_nranks);
        m_stats.weight_largest_node_bytes = I.plan.largest_step_bytes;
        m_stats.weight_ring_bytes = m_streamer->capacity();
        I.runs_done = 0;
    } else {
        m_first_run = false;
        m_source->on_restart();
    }
    I.refs = m_refs_initial;
    I.store.clear();
    I.order.clear();
    I.silu_cache.clear();
    I.staged.clear();
    I.step_slot.clear();
    I.next_stage = 0;
    m_stats.ops_executed = m_stats.ops_fused_away = 0;
    m_pool.reset_high_water();
    m_streamer->begin_run();

    // Capture on the third run: run 1 fills the resident weight cache, run 2 warms every lazily-grown scratch buffer with
    // the cache in place, run 3 records the graph (nothing allocates outside the pool any more).
    bool has_i64_input = false;
    for (auto& h : m_host_tensors) if (h.type == DType::i64) has_i64_input = true;
    GraphState* G = nullptr;
    // int64 inputs (token ids ...) are capturable when the previous eager run consumed their values only through device mirrors
    bool capturing = use_cuda_graph && resident_weights && (!has_i64_input || I.last_run_capture_safe) && I.runs_done >= 2 && m_nranks == 1;
    I.capture_unsafe = false;
    if (capturing) { auto& g = g_graphs[this]; if (g.failed) capturing = false; else G = &g; }

    cudaEvent_t ev0, ev1;
    check_cuda(cudaEventCreate(&ev0), "cudaEventCreate");
    check_cuda(cudaEventCreate(&ev1), "cudaEventCreate");
    check_cuda(cudaEventRecord(ev0, m_stream), "cudaEventRecord");

    // upload graph inputs (push_tensor semantics: same name pushed again => batch sibling, src/onnxstream.cpp:3040-3050)
    m_stats.h2d_input_bytes = 0;
    std::vector<std::pair<Tensor, bool>> uploaded;   // (device tensor, needs fp16 storage conversion)
    for (auto& h : m_host_tensors) {
        Tensor t;
        t.name = h.name;
        for (auto d : h.shape) t.shape.push_back((int64_t)d);
        if (h.type == DType::i64) {
            t.type = DType::i64;
            t.i64 = std::make_shared<std::vector<int64_t>>(h.i64(), h.i64() + h.count);
            t.tainted = true;
            t.i64_dev = m_pool.alloc(std::max<size_t>(h.count, 1) * 8);
            check_cuda(cudaMemcpyAsync(t.i64_dev->ptr, h.buf->ptr, h.count * 8, cudaMemcpyHostToDevice, m_stream), "input H2D (int64 mirror)");
            m_stats.h2d_input_bytes += h.count * 8;
            if (G) G->inputs.push_back({ h.name, h.shape, t.i64_dev, h.count * 8, DType::i64 });
            uploaded.emplace_back(t, false);
        } else {
            // float32, or float16 (the C++ adapter hands fp16 tensors -- e.g. a KV cache kept out of m_outputs_convert_set -- over as they are)
            const size_t esz = dtype_size(h.type);
            t.type = h.type;
            t.dev = m_pool.alloc(h.count * esz);
            check_cuda(cudaMemcpyAsync(t.dev->ptr, h.buf->ptr, h.count * esz, cudaMemcpyHostToDevice, m_stream), "input H2D");
            m_stats.h2d_input_bytes += h.count * esz;
            if (G) G->inputs.push_back({ h.name, h.shape, t.dev, h.count * esz, h.type });
            // storage rule of push_tensor for fp32 data (src/onnxstream.cpp:3006-3035), and m_force_fp16_storage (3764-3808)
            uploaded.emplace_back(t, h.type == DType::f32 && ((use_fp16_arithmetic && !use_uint8_arithmetic && !use_uint8_qdq) || force_fp16_storage));
        }
    }
    size_t n_fresh = (size_t)-1;
    if (keep_inputs) {
        // inputs pushed now replace their kept copies; kept copies of names NOT pushed this time are fed again from HBM
        for (auto& u : uploaded) {
            I.kept_inputs.erase(std::remove_if(I.kept_inputs.begin(), I.kept_inputs.end(), [&](const Tensor& k) { return k.name == u.first.name; }), I.kept_inputs.end());
        }
        n_fresh = uploaded.size();
        for (auto& k : I.kept_inputs) uploaded.emplace_back(k, false);      // already in their storage type
    }
    std::vector<HostTensor> pinned_inputs = std::move(m_host_tensors);   // keep the pinned sources alive until the copies ran
    m_host_tensors.clear();

    bool capture_open = false;
    std::vector<std::tuple<std::string, std::vector<size_t>, Tensor>> finals;   // outputs as f32 plain device tensors
    try {
        if (capturing) {
            check_cuda(cudaStreamSynchronize(m_stream), "pre-capture sync");
            check_cuda(cudaStreamBeginCapture(m_stream, cudaStreamCaptureModeRelaxed), "cudaStreamBeginCapture");
            capture_open = true;
        }
        for (size_t ui = 0; ui < uploaded.size(); ui++) {
            auto& u = uploaded[ui];
            Tensor t = u.first;
            if (ui >= n_fresh) { /* kept copy of an earlier run: stored as it was consumed then */ }
            else if ((use_uint8_qdq || use_uint8_arithmetic) && (t.type == DType::f32 || t.type == DType::f16)) { t = I.quantize_dynamic(t); t.name = u.first.name; }
            else if (u.second) { t = I.convert(t, DType::f16); t.name = u.first.name; }
            if (keep_inputs && ui < n_fresh && t.type != DType::i64) I.kept_inputs.push_back(t);
            auto& v = I.store[t.name];
            if (v.empty()) I.order.push_back(t.name);
            v.push_back(std::move(t));
        }
        if (!I.gn_ring) I.gn_ring = m_pool.alloc(2048);
        check_cuda(cudaMemsetAsync(I.gn_ring->ptr, 0, 2048, m_stream), "cudaMemsetAsync(gn ring)");    // both statistic slots zero: the invariant every producer relies on
        I.gn_slot = 0; I.gn_slot_used[0] = I.gn_slot_used[1] = 0; I.stats_ready_for = -1; I.stats_want = -1;
        I.mha_kv.clear();
        // side branch: steps off the critical path first, on their own stream and pool (see Impl::side_stream)
        bool hoist = !I.plan.is_side.empty() && resident_weights && !m_first_run && !has_i64_input && !ops_times_printf && !ops_printf && m_nranks == 1;
        if (hoist) { std::set<std::string> seen; for (auto& u : uploaded) if (!seen.insert(u.first.name).second) hoist = false; }   // batch siblings: sequential
        m_stats.side_steps = 0;
        if (hoist) {
            for (size_t si = 0; si < I.plan.steps.size(); si++) m_stats.side_steps += (I.plan.is_side[si] || (!I.plan.kv_side.empty() && I.plan.kv_side[si])) ? 1 : 0;
            if (!I.side_stream) check_cuda(cudaStreamCreateWithFlags(&I.side_stream, cudaStreamNonBlocking), "cudaStreamCreate(side)");
            if (I.side_events.size() != I.plan.steps.size() + 2) {
                for (auto e : I.side_events) if (e) cudaEventDestroy(e);
                I.side_events.assign(I.plan.steps.size() + 2, nullptr);
            }
            auto ev = [&](size_t k) -> cudaEvent_t& { if (!I.side_events[k]) check_cuda(cudaEventCreateWithFlags(&I.side_events[k], cudaEventDisableTiming), "cudaEventCreate"); return I.side_events[k]; };
            const size_t EV_IN = I.plan.steps.size(), EV_DONE = I.plan.steps.size() + 1;
            check_cuda(cudaEventRecord(ev(EV_IN), m_stream), "cudaEventRecord(inputs)");
            check_cuda(cudaStreamWaitEvent(I.side_stream, ev(EV_IN), 0), "cudaStreamWaitEvent(side, inputs)");     // (inside a capture: the side stream joins it here)
            I.on_side = true; I.st = I.side_stream;
            try {
                for (size_t si = 0; si < I.plan.steps.size(); si++) {
                    if (I.plan.is_side[si]) { I.exec_step(si); check_cuda(cudaEventRecord(ev(si), I.side_stream), "cudaEventRecord(side step)"); }
                    else if (!I.plan.kv_side.empty() && I.plan.kv_side[si]) {
                        I.mha_prepass(si);
                        auto it = I.mha_kv.find(si);
                        if (it != I.mha_kv.end()) { check_cuda(cudaEventRecord(ev(si), I.side_stream), "cudaEventRecord(side K/V)"); it->second.ev = ev(si); }
                    }
                }
                check_cuda(cudaEventRecord(ev(EV_DONE), I.side_stream), "cudaEventRecord(side done)");
            } catch (...) { I.on_side = false; I.st = m_stream; throw; }
            I.on_side = false; I.st = m_stream;
            for (size_t si = 0; si < I.plan.steps.size(); si++) {
                if (I.plan.is_side[si]) continue;
                for (size_t d : I.plan.side_deps[si]) check_cuda(cudaStreamWaitEvent(m_stream, ev(d), 0), "cudaStreamWaitEvent(main, side step)");
                I.exec_step(si);
            }
            check_cuda(cudaStreamWaitEvent(m_stream, ev(EV_DONE), 0), "cudaStreamWaitEvent(main, side done)");   // join (a capture must not end with a dangling branch)
        } else
        for (size_t si = 0; si < I.plan.steps.size(); si++) I.exec_step(si);
        m_streamer->end_run(m_stream);

        // epilogue: everything still referenced becomes f32 NCHW (src/onnxstream.cpp:8217-8263)
        for (auto& name : I.order) {
            auto it = I.store.find(name);
            if (it == I.store.end()) continue;
            for (auto& t0_ : it->second) {
                std::vector<size_t> shp;
                for (auto d : t0_.shape) shp.push_back((size_t)d);
                if (t0_.type == DType::i64) { finals.emplace_back(name, shp, t0_); continue; }
                Tensor t = I.to_plain(t0_);
                if (t.type == DType::u8) t = I.dequantize(t, DType::f32);     // src/onnxstream.cpp:8238-8241
                // m_outputs_convert_set (src/onnxstream.cpp:8234-8236): tensors outside a non-empty set keep their storage type
                // (fp16 stays fp16: half the D2H bytes, and llm.cpp feeds its KV cache straight back in)
                if (drop_unconverted_outputs && !outputs_convert_set.empty() && !outputs_convert_set.count(name)) continue;
                if (!outputs_convert_set.empty() && !outputs_convert_set.count(name) && t.type == DType::f16) {
                    if (!t.dev || (t.dev.get() == t0_.dev.get() && capturing)) {
                        Tensor c = I.make(DType::f16, t.shape);
                        check_cuda(cudaMemcpyAsync(c.mdata(), t.data(), (size_t)t.numel() * 2, cudaMemcpyDeviceToDevice, m_stream), "copy");
                        t = c;
                    }
                    finals.emplace_back(name, shp, t);
                    continue;
                }
                if (t.type == DType::f32 && !t.dev && t.dev_raw) { Tensor c = I.make(DType::f32, t.shape); check_cuda(cudaMemcpyAsync(c.mdata(), t.dev_raw, (size_t)t.numel() * 4, cudaMemcpyDeviceToDevice, m_stream), "copy"); t = c; }
                t = I.convert(t, DType::f32);
                if (t.dev.get() == t0_.dev.get() && capturing) {   // graph outputs need storage the graph owns exclusively
                    Tensor c = I.make(DType::f32, t.shape);
                    check_cuda(cudaMemcpyAsync(c.mdata(), t.data(), (size_t)t.numel() * 4, cudaMemcpyDeviceToDevice, m_stream), "copy");
                    t = c;
                }
                finals.emplace_back(name, shp, t);
            }
        }
        if (capturing) {
            if (I.capture_unsafe) throw std::runtime_error("an op read the values of an int64 graph input on the host: not capturable");
            for (auto& f : finals) if (std::get<2>(f).type == DType::i64) throw std::runtime_error("int64 graph outputs are host-evaluated: not capturable");
            capture_open = false;
            check_cuda(cudaStreamEndCapture(m_stream, &G->graph), "cudaStreamEndCapture");
            check_cuda(cudaGraphInstantiate(&G->exec, G->graph, 0), "cudaGraphInstantiate");
            for (auto& f : finals) if (std::get<2>(f).type != DType::i64) G->outputs.push_back({ std::get<0>(f), std::get<1>(f), std::get<2>(f).dev, (size_t)std::get<2>(f).numel(), std::get<2>(f).type });
            check_cuda(cudaGraphLaunch(G->exec, m_stream), "cudaGraphLaunch");   // capture does not execute: run it once now
            G->ready = true;
            m_pool.frozen = false;
        }
    } catch (...) {
        if (capture_open) { cudaGraph_t junk = nullptr; cudaStreamEndCapture(m_stream, &junk); if (junk) cudaGraphDestroy(junk); }
        if (capturing) { auto& g = g_graphs[this]; g.failed = true; g.inputs.clear(); g.outputs.clear(); }
        I.store.clear(); I.order.clear(); I.silu_cache.clear();
        cudaEventDestroy(ev0); cudaEventDestroy(ev1);
        if (capturing) {
            // the op list is not capture-safe (host round trips): fall back to eager execution for good
            cudaGetLastError();
            m_host_tensors = std::move(pinned_inputs);
            use_cuda_graph = false;
            run();
            return;
        }
        throw;
    }
    check_cuda(cudaEventRecord(ev1, m_stream), "cudaEventRecord");

    m_stats.d2h_output_bytes = 0;
    for (auto& f : finals) {
        HostTensor h;
        h.name = std::get<0>(f);
        h.shape = std::get<1>(f);
        Tensor& t = std::get<2>(f);
        h.count = (size_t)t.numel();
        if (t.type == DType::i64) {
            h.type = DType::i64;
            h.buf = std::make_shared<PinnedBuf>(h.count * 8);
            memcpy(h.buf->ptr, t.i64->data(), h.count * 8);
        } else {
            h.type = t.type;      // float32, or float16 for tensors outside m_outputs_convert_set
            const size_t ob = h.count * dtype_size(t.type);
            h.buf = std::make_shared<PinnedBuf>(ob);
            check_cuda(cudaMemcpyAsync(h.buf->ptr, t.data(), ob, cudaMemcpyDeviceToHost, m_stream), "output D2H");
            m_stats.d2h_output_bytes += ob;
        }
        m_host_tensors.push_back(std::move(h));
    }
    check_cuda(cudaStreamSynchronize(m_stream), "run sync");
    if (!I.op_times.empty()) {
        std::map<std::string, double> acc;
        for (auto& o : I.op_times) { float ms = 0.f; cudaEventElapsedTime(&ms, o.a, o.b); acc[o.type] += ms; cudaEventDestroy(o.a); cudaEventDestroy(o.b); }
        I.op_times.clear();
        printf("\033[7m > \033[0m");
        for (auto& e : acc) printf(" %s:%f,", e.first.c_str(), e.second);
        printf("\n");
    }
    I.store.clear();
    I.order.clear();
    I.silu_cache.clear();
    finals.clear();
    float ms = 0.f;
    if (!capturing) cudaEventElapsedTime(&ms, ev0, ev1);
    cudaEventDestroy(ev0); cudaEventDestroy(ev1);
    I.runs_done++;
    I.last_run_capture_safe = !I.capture_unsafe;
    m_stats.last_gpu_ms = ms;
    m_stats.kernel_launches = osb_launch_count();
    m_stats.tc_launches = osb_tc_launch_count();
    m_stats.act_high_water_bytes = m_pool.high_water();
    m_stats.weight_peak_live_bytes = m_streamer->peak_live();
    m_stats.weight_bytes_streamed = m_streamer->streamed();
    m_stats.weight_resident_bytes = I.resident_bytes;
    m_stats.last_run_ms = std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - t0).count();
}

}  // namespace osb
