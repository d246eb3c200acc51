// capi.cpp -- the drop-in C ABI: the 16 `model_*` entry points of the reference's FFI (src/exports.cpp:42-311) on top
// of the engine, plus `model_ext_*` / `model_b200_*` extensions for knobs the reference's apps set directly on
// public Model members (src/onnxstream.h:944-968).  Conventions are the reference's: opaque context pointer, borrowed
// NUL-terminated strings in, malloc'd strings/structs out (freed with model_free_buffer), raw pointers into
// engine-owned storage for tensor uploads, errors as malloc'd messages (model_read_file / model_run_2) or C++
// exceptions thrown across the boundary (model_run, model_set_option, model_add_tensor) exactly where the reference
// throws them.
#include "engine_impl.h"
#include "plan.h"
#include "../../include/onnxstream_b200.h"

#include <cuda_profiler_api.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

using namespace osb;

struct ModelContext {
    std::unique_ptr<Engine> engine;
    std::string def;
    std::string wp;
    std::vector<std::string> upcast_patterns;
    Engine& E()
    {
        if (!engine) throw std::runtime_error("onnxstream_b200: this model was created without a backend (threads_count < 0)");
        return *engine;
    }
};

static char* dup_cstr(const std::string& s)
{
    char* b = (char*)malloc(s.size() + 1);
    memcpy(b, s.c_str(), s.size() + 1);
    return b;
}

static std::unique_ptr<WeightSource> source_for(const char* wp)
{
    if (!strcmp(wp, "ram")) return make_ram_source(nullptr);
    if (!strcmp(wp, "nocache")) return make_disk_source(false);
    if (!strcmp(wp, "prefetch")) return make_disk_source(true);
    if (!strcmp(wp, "ram+nocache")) return make_ram_source(make_disk_source(false));
    if (!strcmp(wp, "ram+prefetch")) return make_ram_source(make_disk_source(true));
    return nullptr;
}

static ModelContext* new_ctx(int threads_count, const char* wp)
{
    auto src = source_for(wp);
    if (!src) return nullptr;
    auto* c = new ModelContext();
    c->wp = wp;
    if (threads_count >= 0) {   // threads_count < 0: no backend at all (src/onnxstream.cpp:2397)
        try {
            c->engine = std::make_unique<Engine>();
            c->engine->cpu_threads = threads_count;
            c->engine->set_weight_source(std::move(src));
        } catch (const std::exception& e) {   // no GPU: fail loudly, never fall back to a CPU path
            fprintf(stderr, "=== ERROR === %s\n", e.what());
            delete c;
            return nullptr;
        }
    }
    return c;
}

extern "C" {

ModelContext* model_new() { return new_ctx(0, "ram"); }

ModelContext* model_new_2(int threads_count, char* wp_name)
{
    return new_ctx(threads_count, wp_name);
}

void model_delete(ModelContext* obj) { delete obj; }

void model_read_string(ModelContext* obj, char* str)
{
    obj->def = str;
    obj->E().read_string(str);
}

char* model_read_file(ModelContext* obj, char* fn)
{
    try { obj->E().read_file(fn); return nullptr; }
    catch (const std::exception& e) { return dup_cstr(e.what()); }
}

char* model_get_weights_names(ModelContext* obj)
{
    std::string ret;
    for (auto& w : obj->E().weights_names()) {
        ret += dtype_name(w.first);
        ret += ":" + w.second + "|";
    }
    if (!ret.empty()) ret.pop_back();
    return dup_cstr(ret);
}

void* model_add_weights_file(ModelContext* obj, char* type, char* name, unsigned int size)
{
    if (obj->wp != "ram") return nullptr;
    if (strcmp(type, "uint8") && strcmp(type, "float16") && strcmp(type, "float32") && strcmp(type, "int64"))
        throw std::invalid_argument("Unsupported tensor data format.");
    return ram_source_add(obj->E().weight_source(), name, size);
}

void* model_add_tensor(ModelContext* obj, char* type, char* name, unsigned int dims_num, unsigned int* dims)
{
    std::vector<size_t> shape;
    for (unsigned i = 0; i < dims_num; i++) shape.push_back(dims[i]);
    DType t;
    if (!strcmp(type, "float32")) t = DType::f32;
    else if (!strcmp(type, "int64")) t = DType::i64;
    else throw std::invalid_argument("Unsupported tensor data format.");
    return obj->E().push_input(name, t, shape);
}

void* model_get_tensor(ModelContext* obj, char* name)
{
    HostTensor* t = nullptr;
    for (auto& h : obj->E().tensors()) if (h.name == name) { t = &h; break; }
    if (!t || t->type != DType::f32) return nullptr;
    struct ReturnLayout { size_t dims_num; size_t* dims; size_t data_num; float* data; };   // src/exports.cpp:217-223
    auto* r = (ReturnLayout*)malloc(sizeof(ReturnLayout));
    r->dims_num = t->shape.size();
    r->dims = t->shape.data();
    r->data_num = t->count;
    r->data = t->f32();
    return r;
}

char* model_get_all_tensor_names(ModelContext* obj)
{
    std::string ret;
    for (auto& h : obj->E().tensors()) ret += h.name + "|";
    if (!ret.empty()) ret.pop_back();
    return dup_cstr(ret);
}

void model_run(ModelContext* obj)
{
    try { obj->E().run(); }
    catch (const std::exception& e) { printf("=== ERROR === %s\n", e.what()); throw; }
}

char* model_run_2(ModelContext* obj)
{
    try { obj->E().run(); return nullptr; }
    catch (const std::exception& e) { return dup_cstr(e.what()); }
}

void model_clear_tensors(ModelContext* obj) { obj->E().clear_tensors(); }

void model_set_option(ModelContext* obj, char* name, unsigned int value)
{
    Engine& e = obj->E();
    bool v = value != 0, set = true;
#define OPT(O) if (!strcmp(name, #O)) e.O = v; else
    OPT(use_fp16_arithmetic) OPT(use_uint8_qdq) OPT(use_uint8_arithmetic) OPT(fuse_ops_in_attention) OPT(force_fp16_storage)
    OPT(support_dynamic_shapes) OPT(use_ops_cache) OPT(use_scaled_dp_attn_op) OPT(use_next_op_cache) OPT(ops_printf)
    OPT(ops_times_printf) OPT(use_nchw_convs)
#undef OPT
    if (!strcmp(name, "b200_resident_weights")) e.resident_weights = v;
    else if (!strcmp(name, "b200_cuda_graph")) e.use_cuda_graph = v;
    else if (!strcmp(name, "b200_fuse_nodes")) e.fuse_nodes = v;
    else if (!strcmp(name, "b200_keep_nhwc")) e.keep_nhwc = v;
    else if (!strcmp(name, "b200_gemm_impl")) e.gemm_impl = (int)value;
    else if (!strcmp(name, "b200_flash_attention")) e.flash_attention = v;
    else if (!strcmp(name, "b200_ring_factor_x100")) e.ring_factor = value / 100.0;
    else if (!strcmp(name, "b200_range_data_calibrate")) e.range_data_calibrate = v;
    else if (!strcmp(name, "b200_keep_inputs")) e.keep_inputs = v;
    else if (!strcmp(name, "b200_drop_unconverted_outputs")) e.drop_unconverted_outputs = v;
    else set = false;
    if (!set) {
        const char* err = "model_set_option: 'name' not found.";
        printf("=== ERROR === %s\n", err);
        throw std::invalid_argument(err);
    }
}

void model_add_extra_output(ModelContext* obj, char* name) { obj->E().extra_outputs.emplace_back(name); }

void model_free_buffer(void* ptr) { free(ptr); }

// ---- extensions -------------------------------------------------------------------------------------------------

void model_ext_set_attention_parts(ModelContext* obj, unsigned parts) { obj->E().attention_fused_ops_parts = parts; }

void model_ext_set_range(ModelContext* obj, const char* op_name, float mn, float mx) { obj->E().range_data[op_name] = { mn, mx }; }

char* model_ext_read_range_data(ModelContext* obj, const char* fn)
{
    try { obj->E().read_range_data(fn); return nullptr; }
    catch (const std::exception& e) { return dup_cstr(e.what()); }
}

char* model_ext_write_range_data(ModelContext* obj, const char* fn)
{
    try { obj->E().write_range_data(fn); return nullptr; }
    catch (const std::exception& e) { return dup_cstr(e.what()); }
}

void model_ext_add_upcast_pattern(ModelContext* obj, const char* pattern)
{
    obj->upcast_patterns.emplace_back(pattern);
    auto pats = obj->upcast_patterns;
    obj->E().requires_upcast = [pats](const std::string&, const std::string& name) {
        for (auto& p : pats) if (name.find(p) != std::string::npos) return true;
        return false;
    };
}

void model_ext_push_tensor(ModelContext* obj, const char* type, const char* name, unsigned dims_num, const unsigned* dims, const void* data)
{
    std::vector<size_t> shape;
    size_t n = 1;
    for (unsigned i = 0; i < dims_num; i++) { shape.push_back(dims[i]); n *= dims[i]; }
    bool f = !strcmp(type, "float32");
    if (!f && strcmp(type, "int64")) throw std::invalid_argument("Unsupported tensor data format.");
    void* dst = obj->E().push_input(name, f ? DType::f32 : DType::i64, shape);
    memcpy(dst, data, n * (f ? 4 : 8));
}

long long model_ext_get_tensor_i64(ModelContext* obj, const char* name, long long* dst, long long cap, size_t* dims, size_t* ndims)
{
    for (auto& h : obj->E().tensors())
        if (h.name == name) {
            if (h.type != DType::i64) return -1;
            for (size_t i = 0; i < h.count && (long long)i < cap; i++) dst[i] = h.i64()[i];
            *ndims = h.shape.size();
            for (size_t i = 0; i < h.shape.size() && i < 8; i++) dims[i] = h.shape[i];
            return (long long)h.count;
        }
    return -1;
}

// index-th tensor named `name` (batch siblings share a name, src/onnxstream.cpp:3040-3050); same return layout and ownership as
// model_get_tensor; NULL when absent or not float32
void* model_ext_get_tensor_at(ModelContext* obj, const char* name, unsigned int index)
{
    HostTensor* t = nullptr;
    unsigned int seen = 0;
    for (auto& h : obj->E().tensors()) if (h.name == name) { if (seen++ == index) { t = &h; break; } }
    if (!t || t->type != DType::f32) return nullptr;
    struct ReturnLayout { size_t dims_num; size_t* dims; size_t data_num; float* data; };
    auto* r = (ReturnLayout*)malloc(sizeof(ReturnLayout));
    r->dims_num = t->shape.size(); r->dims = t->shape.data(); r->data_num = t->count; r->data = t->f32();
    return r;
}

// m_outputs_convert_set (src/onnxstream.h:961): once a name is added, only listed outputs are converted to float32 at the end of run()
void model_ext_add_output_convert(ModelContext* obj, const char* name) { obj->E().outputs_convert_set.insert(name); }

int model_ext_get_tensor_type(ModelContext* obj, const char* name)
{
    for (auto& h : obj->E().tensors()) if (h.name == name) return (int)h.type;
    return -1;
}

char* model_b200_plan_summary(const char* model_text, int fp16_arithmetic, int fuse_nodes, int fuse_attention, int use_scaled_dp_attn_op)
{
    std::string r;
    try {
        r = osb::plan_summary(model_text ? model_text : "", fp16_arithmetic != 0, fuse_nodes != 0, fuse_attention != 0, use_scaled_dp_attn_op != 0);
    } catch (const std::exception& e) {
        r = std::string("=== ERROR === ") + e.what();
    }
    char* buf = (char*)malloc(r.size() + 1);
    if (buf) memcpy(buf, r.c_str(), r.size() + 1);
    return buf;
}

int model_b200_get_stats(ModelContext* obj, double* out, int n)
{
    const EngineStats& s = obj->E().stats();
    double v[] = { (double)s.weight_ring_bytes, (double)s.weight_peak_live_bytes, (double)s.weight_largest_node_bytes,
                   (double)s.weight_bytes_streamed, (double)s.weight_resident_bytes, (double)s.act_high_water_bytes,
                   (double)s.h2d_input_bytes, (double)s.d2h_output_bytes, (double)s.kernel_launches, (double)s.tc_launches,
                   (double)s.ops_executed, (double)s.ops_fused_away, s.last_run_ms, s.last_gpu_ms, (double)s.graph_replays, (double)s.side_steps };
    int m = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n && i < m; i++) out[i] = v[i];
    return m;
}

double model_b200_run_resident(ModelContext* obj, int steps)
{
    try { return obj->E().run_resident(steps); }
    catch (const std::exception& e) { fprintf(stderr, "=== ERROR === %s\n", e.what()); return -1.0; }
}

int model_b200_set_comm(ModelContext* obj, void* nccl_comm, int rank, int nranks)
{
    obj->E().set_comm((ncclComm*)nccl_comm, rank, nranks);
    return 0;
}

// cudaProfilerStart/Stop around a region of interest (profilers started with capture off)
void model_b200_profiler(int start)
{
    if (start) cudaProfilerStart(); else cudaProfilerStop();
}

const char* model_b200_version() { return "onnxstream_b200 0.1 (sm_90a)"; }

}  // extern "C"
