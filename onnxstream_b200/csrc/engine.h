// engine.h -- H100-native per-node execution engine behind OnnxStream's Model / WeightsProvider surface.
//
// The reference executes a text graph op by op on the CPU (Model::run, src/onnxstream.cpp:3550-8269), fetching each
// node's weights from a WeightsProvider (src/onnxstream.h:266-900) right before use.  This engine keeps exactly that
// contract -- same file format, same per-op semantics, same ref-counted tensor store, same "weights in strict graph
// order" streaming -- but every float tensor lives in HBM, every op is a CUDA kernel launch on one compute stream,
// and weights flow pinned-host -> HBM ring on a copy stream overlapped with the previous node's kernels.
//
// Not a port: the reference re-parses the text file on every run and allocates per op; here the graph is parsed once,
// activations come from a stream-ordered pool, fusions (GroupNorm+SiLU, LayerNorm, GELU/GEGLU, attention, bias /
// residual epilogues, NHWC relabelling instead of transposes) are decided on the parsed op list, and a whole run can
// be captured into a CUDA graph.
#pragma once

#include <cstdint>
#include <cstddef>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

struct CUstream_st;
struct CUevent_st;
struct ncclComm;

namespace osb {

enum class DType : int { none = 0, u8 = 1, f16 = 2, f32 = 3, i64 = 4 };  // src/onnxstream.h:147-154
enum class Layout : int { plain = 0, nhwc = 1 };                          // src/onnxstream.h:156-160

size_t dtype_size(DType t);
const char* dtype_name(DType t);

// ---- device memory ------------------------------------------------------------------------------------------
class DevicePool;
struct DevBlock {
    void* ptr = nullptr;
    size_t bytes = 0;
    DevicePool* pool = nullptr;
    ~DevBlock();
};
using DevPtr = std::shared_ptr<DevBlock>;

// Stream-ordered best-fit pool over large cudaMalloc slabs.  All users run on the single compute stream, so a block
// can be handed out again as soon as it is released (stream order keeps the previous kernel ahead of the next).
class DevicePool {
public:
    ~DevicePool();
    DevPtr alloc(size_t bytes);
    void release(void* ptr, size_t bytes);
    size_t bytes_in_use() const { return m_in_use; }
    size_t high_water() const { return m_high_water; }
    size_t reserved() const { return m_reserved; }
    void reset_high_water() { m_high_water = m_in_use; }
    bool frozen = false;  // set while a CUDA graph owns the addresses: growing is an error
private:
    struct Slab { void* base; size_t bytes; };
    std::vector<Slab> m_slabs;
    std::map<uintptr_t, size_t> m_free;  // address -> bytes, coalesced
    size_t m_in_use = 0, m_high_water = 0, m_reserved = 0;
    void add_slab(size_t min_bytes);
};

// ---- tensors -------------------------------------------------------------------------------------------------
struct Tensor {
    std::string name;
    DType type = DType::none;
    std::vector<int64_t> shape;       // logical shape (NCHW for images, like the reference)
    Layout layout = Layout::plain;    // nhwc: memory order is [H, W, C] for logical [1, C, H, W]
    DevPtr dev;                       // device payload for u8 / f16 / f32
    const void* dev_raw = nullptr;    // non-owning device payload (weight ring / resident weight cache)
    std::shared_ptr<std::vector<int64_t>> i64;  // host payload for int64 tensors (shape arithmetic stays on the host)
    DevPtr i64_dev;                   // device mirror of an int64 GRAPH INPUT (token ids, positions, masks): refreshed before every run / graph
                                      // replay, read by the ops whose result depends on the VALUES (Gather indices, Cast to float)
    bool tainted = false;             // int64 values that come from a graph input: reading them on the host bakes them into a captured graph
    std::shared_ptr<std::vector<float>> host_f32;  // host mirror of small float constants (scalars, Resize scales)
    float scale = 0.f;
    int zero_point = 0;
    bool is_weight = false;

    int64_t numel() const { int64_t n = 1; for (auto d : shape) n *= d; return n; }
    const void* data() const { return dev ? dev->ptr : dev_raw; }
    void* mdata() { return dev ? dev->ptr : nullptr; }
    bool on_device() const { return dev != nullptr || dev_raw != nullptr; }
};

struct TensorRef {                    // a tensor mention inside model.txt (src/onnxstream.cpp:2540-2616)
    std::string name;
    DType wtype = DType::none;        // != none: static weight whose file name is `name`
    std::vector<int64_t> shape;
    float scale = 0.f;
    int zero_point = 0;
    bool present = false;
};

struct OpDef {                        // src/onnxstream.h:253-264
    std::string name, type;
    std::vector<TensorRef> in, out;
    std::vector<std::pair<std::string, std::string>> attrs;
    const std::string* attr(const char* key) const;
};

// ---- weights -------------------------------------------------------------------------------------------------
// Host-side source of weight bytes.  Mirrors the WeightsProvider contract (src/onnxstream.h:266-291): `on_init` once
// per weight in graph order, `on_restart` at the start of every later run, `fetch` synchronously in graph order.
class WeightSource {
public:
    virtual ~WeightSource() {}
    std::string path;
    virtual void on_init(DType type, const std::string& name, size_t bytes) {}
    virtual void on_restart() {}
    // Copies (or exposes) `bytes` bytes of weight `name`.  If the source owns stable pinned memory it returns a pointer
    // and leaves `dst` untouched; otherwise it fills `dst` (pinned staging provided by the streamer) and returns dst.
    virtual const void* fetch(const std::string& name, DType type, size_t bytes, void* dst) = 0;
    virtual bool stable_pinned() const { return false; }
    virtual const char* kind() const = 0;
};

std::unique_ptr<WeightSource> make_disk_source(bool prefetch_thread);           // "nocache" / "prefetch"
std::unique_ptr<WeightSource> make_ram_source(std::unique_ptr<WeightSource> inner);  // "ram", "ram+nocache", "ram+prefetch"
void* ram_source_add(WeightSource* ram, const std::string& name, size_t bytes);   // model_add_weights_file

// Double-buffered HBM arena fed from pinned host memory on a side stream (the CUDA WeightsProvider of the north star).
class WeightStreamer;

struct EngineStats {
    size_t weight_ring_bytes = 0;        // capacity of the HBM weight ring
    size_t weight_peak_live_bytes = 0;   // high-water mark of streamed weight bytes resident in HBM at once
    size_t weight_largest_node_bytes = 0;
    size_t weight_bytes_streamed = 0;    // H2D weight traffic of the last run
    size_t weight_resident_bytes = 0;    // HBM-resident (cached) weight bytes in "hbm" mode
    size_t act_high_water_bytes = 0;
    size_t h2d_input_bytes = 0, d2h_output_bytes = 0;
    uint64_t kernel_launches = 0, tc_launches = 0;
    uint64_t ops_executed = 0, ops_fused_away = 0;
    double last_run_ms = 0.0;            // wall time of the last run() on the host, including the final sync
    double last_gpu_ms = 0.0;            // CUDA-event time of the last run on the compute stream
    int graph_replays = 0;
    int side_steps = 0;                  // steps of the last run that were enqueued on the side stream (0: sequential run)
};

struct PinnedBuf {                    // page-locked host memory (cudaHostAlloc): H2D/D2H copies run at full PCIe rate
    void* ptr = nullptr;
    size_t bytes = 0;
    explicit PinnedBuf(size_t n);
    ~PinnedBuf();
};

struct HostTensor {                   // what is left in the model's tensor list after run(): f32 NCHW, int64, or f16 (outside m_outputs_convert_set)
    std::string name;
    DType type = DType::none;
    std::vector<size_t> shape;
    std::shared_ptr<PinnedBuf> buf;
    size_t count = 0;
    float* f32() const { return (float*)buf->ptr; }
    uint16_t* f16() const { return (uint16_t*)buf->ptr; }
    int64_t* i64() const { return (int64_t*)buf->ptr; }
};

struct EngineNoDevice {};   // tag: construct the host-side planner only

class Engine {
public:
    explicit Engine(EngineNoDevice);
    explicit Engine(int device = -1);
    ~Engine();
    // Host-only planning (no CUDA device needed): parse `model_text`, run the fusion matchers, return one line per execution step
    // ("KIND ops first_op_type first_op_name") followed by a "#summary" line.  Used by the CPU test-suite to pin the planner.
    static std::string plan_summary(const std::string& model_text, bool fp16_arithmetic, bool fuse_nodes, bool fuse_attention, bool use_sdpa_rewrite = false);

    // --- the reference's public knobs (src/onnxstream.h:944-968) ---
    bool use_fp16_arithmetic = false;
    bool use_uint8_qdq = false;
    bool use_uint8_arithmetic = false;
    bool fuse_ops_in_attention = false;
    size_t attention_fused_ops_parts = 2;   // accepted, no effect: the fused kernel never materialises more than a tile
    std::vector<std::string> extra_outputs;
    bool force_fp16_storage = false;
    bool support_dynamic_shapes = false;
    bool use_ops_cache = false;
    std::function<bool(const std::string&, const std::string&)> requires_upcast;
    bool use_scaled_dp_attn_op = false;
    std::set<std::string> outputs_convert_set;
    std::set<std::string> force_uint8_storage_set;
    bool use_next_op_cache = false;
    bool use_nchw_convs = false;
    bool ops_printf = false;
    bool ops_times_printf = false;
    std::map<std::string, std::pair<float, float>> range_data;
    bool range_data_calibrate = false;     // m_range_data_calibrate (src/onnxstream.h:964): record every op output's percentile range
    int cpu_threads = 0;                   // the reference's pool size (Model(threads_count)): it partitions the percentile chunks

    // --- engine-specific knobs (set through model_set_option("b200_*")) ---
    bool resident_weights = false;   // keep converted weights in HBM after the first run (upper bound; "--ram" analogue)
    bool use_cuda_graph = false;     // capture run() once and replay
    bool fuse_nodes = true;          // GroupNorm/LayerNorm/GELU/SiLU/bias/residual fusions
    bool keep_nhwc = true;           // keep conv trunks channel-last instead of transposing around every Conv
    int gemm_impl = 0;               // 0 auto, 1 force CUDA-core kernels, 2 force the tensor-core kernel
    bool flash_attention = true;     // fused wgmma attention for d <= 64 (else two GEMMs around a softmax)
    double ring_factor = 1.0;        // weight ring capacity = ring_factor * largest node footprint
    bool keep_inputs = false;        // graph inputs stay in HBM after a run; a later run that does not push a name again reuses the device copy
                                     // (a device-resident KV cache for fixed-shape decode steps: only the new token's ids cross PCIe)
    bool drop_unconverted_outputs = false;   // with a non-empty outputs_convert_set: tensors outside it are not copied back at all
    bool source_on_init_done = false;  // set by the C++ adapter when it already announced every weight to the provider

    void set_weight_source(std::unique_ptr<WeightSource> src);
    WeightSource* weight_source() { return m_source.get(); }

    void read_file(const char* filename);
    void read_string(const char* text, const char* path_with_slash = "./");
    bool is_model_empty() const { return m_text.empty(); }
    std::vector<std::pair<DType, std::string>> weights_names();   // model_get_weights_names

    // inputs are copied to pinned host staging here and uploaded at the start of run()
    void* push_input(const std::string& name, DType type, const std::vector<size_t>& shape);  // returns host buffer to fill
    void run();
    // Replays the captured CUDA graph `steps` times on the device-resident inputs of the last run (no H2D / D2H);
    // returns the CUDA-event time in ms.  Requires b200_cuda_graph + b200_resident_weights and one completed run().
    double run_resident(int steps);
    std::vector<HostTensor>& tensors() { return m_host_tensors; }   // inputs before run(), outputs after
    void clear_tensors();

    void read_range_data(const char* filename);
    void write_range_data(const char* filename);

    // multi-GPU: every rank streams the same weights; rank `root` does the H2D and broadcasts each block over NCCL.
    void set_comm(ncclComm* comm, int rank, int nranks);

    const EngineStats& stats() const { return m_stats; }
    int device() const { return m_device; }
    CUstream_st* compute_stream() const { return m_stream; }

private:
    friend struct OpCtx;
    int m_device = 0;
    CUstream_st* m_stream = nullptr;
    std::string m_text, m_path;
    std::vector<OpDef> m_ops;
    bool m_parsed = false;
    std::map<std::string, int> m_refs_initial;
    bool m_first_run = true;

    std::unique_ptr<WeightSource> m_source;
    std::unique_ptr<WeightStreamer> m_streamer;
    DevicePool m_pool;
    EngineStats m_stats;
    std::vector<HostTensor> m_host_tensors;

    ncclComm* m_comm = nullptr;
    int m_rank = 0, m_nranks = 1;

    void parse();
    void invalidate_plan();
    std::string options_signature() const;
    void run_body(bool capturing);
    bool try_replay();
    void drop_graph();
    struct Impl;
    std::unique_ptr<Impl> m_impl;
};

void check_cuda(int err, const char* what);
void* pinned_alloc(size_t bytes, const char* what);   // page-locked host memory on the NUMA node local to the current device

}  // namespace osb
