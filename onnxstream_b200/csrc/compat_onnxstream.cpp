// compat_onnxstream.cpp -- the C++ drop-in: defines every out-of-line `onnxstream::` symbol that the reference's
// own applications link against (measured with `nm -uC` on sd.o / llm.o / exports.o, SURVEY.md section 8b):
//
//     onnxstream::Model::Model(int)          ~Model()              read_file(const char*)     read_string(const char*, const char*)
//     onnxstream::Model::init()              run()                 push_tensor(Tensor&&)      read_range_data / write_range_data
//     onnxstream::Model::set_cuda_options(const CudaOptions&)      onnxstream::trim(std::string&)
//
// It is compiled against the reference's own, UNMODIFIED `onnxstream.h` where it lies (-I<reference>/src; the header is
// the ABI contract -- apps poke Model's public members directly -- and is never copied into this repository), and hides
// all GPU state behind the opaque `XnnPack* m_xnnpack` member (src/onnxstream.h:902,1036).  With this translation unit in
// place of the reference's onnxstream.cpp, src/sd.cpp, src/llm.cpp and src/exports.cpp compile and link unchanged
// (scripts/link_reference_apps.sh).
//
// Semantics kept: weights are requested from the app's WeightsProvider synchronously in strict graph order
// (on_init once per weight in order on the first init(), on_restart before later runs, src/onnxstream.cpp:3499-3548);
// tensors pushed twice under one name become m_batch siblings (src/onnxstream.cpp:3040-3050); after run() m_data holds the
// graph outputs and m_extra_outputs as float32 NCHW (src/onnxstream.cpp:8217-8263).
#include "onnxstream.h"   // the reference's header, found through -I<reference checkout>/src

#include "engine_impl.h"

#include <cstring>

namespace onnxstream {

// the opaque backend object behind Model::m_xnnpack
class XnnPack {
public:
    std::unique_ptr<osb::Engine> engine;
    CudaOptions cuda_options;
    bool source_installed = false;
};

namespace {

osb::DType to_osb(TensorDataType t)
{
    switch (t) {
    case TensorDataType::uint8: return osb::DType::u8;
    case TensorDataType::float16: return osb::DType::f16;
    case TensorDataType::float32: return osb::DType::f32;
    case TensorDataType::int64: return osb::DType::i64;
    default: return osb::DType::none;
    }
}
TensorDataType from_osb(osb::DType t)
{
    switch (t) {
    case osb::DType::u8: return TensorDataType::uint8;
    case osb::DType::f16: return TensorDataType::float16;
    case osb::DType::f32: return TensorDataType::float32;
    case osb::DType::i64: return TensorDataType::int64;
    default: return TensorDataType::none;
    }
}

// Engine-side view of the application's WeightsProvider (any subclass: DiskNoCache, DiskPrefetch, Ram<...>, custom).
class ProviderSource : public osb::WeightSource {
public:
    explicit ProviderSource(WeightsProvider* wp) : m_wp(wp) {}
    void on_init(osb::DType type, const std::string& name, size_t bytes) override { m_wp->on_init(from_osb(type), name, bytes); }
    void on_restart() override { m_wp->on_restart(); }
    const void* fetch(const std::string& name, osb::DType type, size_t bytes, void* dst) override
    {
        m_wp->m_path = path;
        auto put = [&](const void* src, size_t n) {
            if (n != bytes) throw std::invalid_argument("Model::get_tensor_data: mismatch between tensor shape and data size.");
            if (!dst) { m_tmp.assign((const char*)src, (const char*)src + n); return (const void*)m_tmp.data(); }
            std::memcpy(dst, src, n);
            return (const void*)dst;
        };
        bool ptr = m_wp->supports_getptr();
        switch (type) {
        case osb::DType::u8: { if (ptr) { auto p = m_wp->getptr_uint8(name); return put(p->data(), p->size()); } auto v = m_wp->get_uint8(name); return put(v.data(), v.size()); }
        case osb::DType::f16: { if (ptr) { auto p = m_wp->getptr_float16(name); return put(p->data(), p->size() * 2); } auto v = m_wp->get_float16(name); return put(v.data(), v.size() * 2); }
        case osb::DType::f32: { if (ptr) { auto p = m_wp->getptr_float32(name); return put(p->data(), p->size() * 4); } auto v = m_wp->get_float32(name); return put(v.data(), v.size() * 4); }
        case osb::DType::i64: { if (ptr) { auto p = m_wp->getptr_int64(name); return put(p->data(), p->size() * 8); } auto v = m_wp->get_int64(name); return put(v.data(), v.size() * 8); }
        default: throw std::invalid_argument("Model::get_tensor_data: unsupported tensor data format.");
        }
    }
    const char* kind() const override { return "WeightsProvider"; }
private:
    WeightsProvider* m_wp;
    std::vector<char> m_tmp;
};

}  // namespace

std::string& trim(std::string& s)
{
    const char* ws = " \t\n\r\f\v";
    s.erase(s.find_last_not_of(ws) + 1);
    s.erase(0, s.find_first_not_of(ws));
    return s;
}

Model::Model(int threads_count)
{
    if (threads_count >= 0) {   // negative: no backend at all (src/onnxstream.cpp:2397)
        m_xnnpack = new XnnPack();
        m_xnnpack->engine = std::make_unique<osb::Engine>();
        m_xnnpack->engine->cpu_threads = threads_count;
    }
}

Model::~Model()
{
    delete m_xnnpack;
}

void Model::set_cuda_options(const CudaOptions& options)
{
    // the reference budgets VRAM for resident cuBLAS weights (src/onnxstream.cpp:395-398); here a non-zero budget selects the
    // HBM-resident weight cache, zero keeps pure streaming.
    if (m_xnnpack) {
        m_xnnpack->cuda_options = options;
        m_xnnpack->engine->resident_weights = options.m_vram_to_use != 0;
    }
}

void Model::read_file(const char* filename)
{
    auto text = onnxstream::read_file<std::vector<char>>(filename);
    m_model = std::move(text);
    m_path = "";
    std::string fn(filename);
    auto sep = fn.find_last_of("/\\");
    if (sep != std::string::npos) m_path = fn.substr(0, sep + 1);
    get_wp()->m_path = m_path;
}

void Model::read_string(const char* string, const char* path_with_slash)
{
    m_model.assign(string, string + std::strlen(string));
    m_path = path_with_slash;
    get_wp()->m_path = m_path;
}

void Model::push_tensor(Tensor&& t)
{
    // app-side pushes happen outside run(): same name again => batch sibling (src/onnxstream.cpp:3040-3050)
    for (auto it = m_data.rbegin(); it != m_data.rend(); ++it)
        if (it->m_name == t.m_name) {
            if (it->m_batch == nullptr) it->m_batch = std::make_shared<std::vector<Tensor>>();
            it->m_batch->push_back(std::move(t));
            return;
        }
    m_data.push_back(std::move(t));
}

void Model::init()
{
    // First call: tell the provider every weight, in graph order (src/onnxstream.cpp:3505-3531).  Works without a backend
    // (threads_count < 0), which is how exports.cpp enumerates weight names (src/exports.cpp:111-148).
    if (m_intermediate_refs_copy.size() == 0) {
        std::string text(m_model.begin(), m_model.end());
        auto ops = osb::parse_model_text(text, m_support_dynamic_shapes);
        for (auto& op : ops)
            for (auto& in : op.in) {
                if (!in.present) continue;
                if (in.wtype == osb::DType::none) { m_intermediate_refs[in.name]++; continue; }
                size_t size = osb::dtype_size(in.wtype);
                for (auto d : in.shape) size *= (size_t)d;
                get_wp()->on_init(from_osb(in.wtype), in.name, size);
            }
        for (auto& name : m_extra_outputs) m_intermediate_refs[name]++;
        m_intermediate_refs_copy = m_intermediate_refs;
        if (m_intermediate_refs_copy.empty()) m_intermediate_refs_copy["<none>"] = 0;
    } else {
        m_first_run = false;
    }
}

void Model::run()
{
    if (!m_xnnpack) throw std::invalid_argument("Model::run: this model was created without a backend (threads_count < 0).");
    osb::Engine& e = *m_xnnpack->engine;

    // mirror the public knobs (src/onnxstream.h:944-968) into the engine
    e.use_fp16_arithmetic = m_use_fp16_arithmetic;
    e.use_uint8_qdq = m_use_uint8_qdq;
    e.use_uint8_arithmetic = m_use_uint8_arithmetic;
    e.fuse_ops_in_attention = m_fuse_ops_in_attention;
    e.attention_fused_ops_parts = m_attention_fused_ops_parts;
    e.extra_outputs = m_extra_outputs;
    e.force_fp16_storage = m_force_fp16_storage;
    e.support_dynamic_shapes = m_support_dynamic_shapes;
    e.use_ops_cache = m_use_ops_cache;
    if (m_use_ops_cache) e.resident_weights = true;   // "--ram"/llm: operators (and their weights) are kept after the first run
    e.requires_upcast = m_requires_upcast;
    e.use_scaled_dp_attn_op = m_use_scaled_dp_attn_op;
    e.outputs_convert_set = m_outputs_convert_set;
    e.force_uint8_storage_set = m_force_uint8_storage_set;
    e.use_nchw_convs = m_use_nchw_convs;
    e.ops_printf = m_ops_printf;
    e.ops_times_printf = m_ops_times_printf;
    e.range_data = m_range_data;
    e.range_data_calibrate = m_range_data_calibrate;

    if (!m_xnnpack->source_installed) {
        auto src = std::make_unique<ProviderSource>(get_wp());
        src->path = m_path;
        e.set_weight_source(std::move(src));
        std::string text(m_model.begin(), m_model.end());
        e.read_string(text.c_str(), m_path.c_str());
        m_xnnpack->source_installed = true;
    }

    // inputs: whatever the app pushed into m_data (float32 / float16 / int64), batch siblings included
    auto feed = [&](Tensor& t) {
        std::vector<size_t> shape(t.m_shape.begin(), t.m_shape.end());
        switch (t.m_type) {
        case TensorDataType::float32: { auto& v = t.get_vector<float>(); std::memcpy(e.push_input(t.m_name, osb::DType::f32, shape), v.data(), v.size() * 4); break; }
        case TensorDataType::int64: { auto& v = t.get_vector<int64_t>(); std::memcpy(e.push_input(t.m_name, osb::DType::i64, shape), v.data(), v.size() * 8); break; }
        case TensorDataType::float16: { auto& v = t.get_vector<uint16_t>(); std::memcpy(e.push_input(t.m_name, osb::DType::f16, shape), v.data(), v.size() * 2); break; }
        default: throw std::invalid_argument("Model::run: unsupported input tensor type.");
        }
    };
    e.clear_tensors();
    for (auto& t : m_data) {
        feed(t);
        if (t.m_batch) for (auto& u : *t.m_batch) feed(u);
    }
    m_data.clear();

    init();                          // first call announces every weight to the provider, in graph order
    e.source_on_init_done = true;    // ... so the engine must not announce them again
    e.run();

    // outputs back into m_data, siblings regrouped under the first tensor of each name
    for (auto& h : e.tensors()) {
        Tensor t;
        t.m_name = h.name;
        t.m_shape.assign(h.shape.begin(), h.shape.end());
        if (h.type == osb::DType::i64) { tensor_vector<int64_t> v(h.i64(), h.i64() + h.count); t.set_vector(std::move(v)); }
        else if (h.type == osb::DType::f16) { tensor_vector<uint16_t> v(h.f16(), h.f16() + h.count); t.set_vector(std::move(v)); }   // outside m_outputs_convert_set
        else { tensor_vector<float> v(h.f32(), h.f32() + h.count); t.set_vector(std::move(v)); }
        push_tensor(std::move(t));
    }
    e.clear_tensors();
    m_range_data = e.range_data;
}

void Model::read_range_data(const char* filename)
{
    osb::Engine* e = m_xnnpack ? m_xnnpack->engine.get() : nullptr;
    if (!e) throw std::invalid_argument("Model::read_range_data: no backend.");
    e->read_range_data(filename);
    m_range_data = e->range_data;
}

void Model::write_range_data(const char* filename)
{
    osb::Engine* e = m_xnnpack ? m_xnnpack->engine.get() : nullptr;
    if (!e) throw std::invalid_argument("Model::write_range_data: no backend.");
    e->range_data = m_range_data;
    e->write_range_data(filename);
}

}  // namespace onnxstream
