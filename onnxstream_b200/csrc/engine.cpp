// engine.cpp -- infrastructure of the engine: device pool, model.txt parser, weight sources, the streaming
// HBM weight ring.  The op interpreter lives in engine_run.cpp.
#include "engine_impl.h"

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <cctype>
#include <cstdio>
#include <cstring>

#include <algorithm>
#include <map>
#include <mutex>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <stdexcept>

namespace osb {

void check_cuda(int err, const char* what)
{
    if (err != 0) {
        const char* s = cudaGetErrorString((cudaError_t)err);
        throw std::runtime_error(std::string(what) + ": CUDA error " + std::to_string(err) + " (" + (s ? s : "?") + ")");
    }
}

size_t dtype_size(DType t)
{
    switch (t) {
    case DType::u8: return 1;
    case DType::f16: return 2;
    case DType::f32: return 4;
    case DType::i64: return 8;
    default: return 0;
    }
}

const char* dtype_name(DType t)
{
    switch (t) {
    case DType::u8: return "uint8";
    case DType::f16: return "float16";
    case DType::f32: return "float32";
    case DType::i64: return "int64";
    default: return "none";
    }
}

// ================================================================================================================
// NUMA-local pinned memory
// ================================================================================================================
// On a two-socket host a pinned buffer that lands on the socket the GPU is NOT attached to streams markedly slower over PCIe
// (and the whole streaming step is PCIe-bound).
// Pages are allocated on the node of the thread that calls cudaHostAlloc, so the call runs with the thread temporarily bound
// to the CPUs local to the current device (/sys/bus/pci/devices/<bdf>/local_cpulist); the previous affinity is restored on
// scope exit.  OSB_NUMA_BIND=0 disables it; any failure degrades to a plain allocation.
namespace {
struct LocalCpuGuard {
    cpu_set_t old_set;
    bool active = false;
    bool policy_set = false;
    // set_mempolicy(2) without libnuma: MPOL_BIND = 2 to the GPU's node while the allocation runs, MPOL_DEFAULT = 0 afterwards
    static long set_policy(int mode, const unsigned long* mask, unsigned long maxnode)
    {
#ifdef SYS_set_mempolicy
        return syscall(SYS_set_mempolicy, mode, mask, maxnode);
#else
        return -1;
#endif
    }
    void bind_memory_to_node_of(const std::string& bdf)
    {
        FILE* f = fopen(("/sys/bus/pci/devices/" + bdf + "/numa_node").c_str(), "r");
        if (!f) return;
        int node = -1;
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
        if (node < 0 || node >= 1024) return;
        unsigned long mask[16] = { 0 };
        mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
        if (set_policy(2 /* MPOL_BIND */, mask, 1024 + 1) == 0) policy_set = true;
    }
    LocalCpuGuard()
    {
        static const bool enabled = [] { const char* e = getenv("OSB_NUMA_BIND"); return !(e && e[0] == '0'); }();
        if (!enabled) return;
        int dev = 0;
        char bdf[32] = { 0 };
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetPCIBusId(bdf, sizeof bdf, dev) != cudaSuccess) return;
        for (char* c = bdf; *c; c++) *c = (char)tolower((unsigned char)*c);
        static const bool policy = [] { const char* e = getenv("OSB_NUMA_POLICY"); return !(e && e[0] == '0'); }();
        if (policy) bind_memory_to_node_of(bdf);     // memory policy first: it holds even when the CPU mask cannot be narrowed
        std::string path = std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist";
        FILE* f = fopen(path.c_str(), "r");
        if (!f) return;
        char line[4096] = { 0 };
        bool got = fgets(line, sizeof line, f) != nullptr;
        fclose(f);
        if (!got) return;
        cpu_set_t local;
        CPU_ZERO(&local);
        for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int a = 0, b = 0;
            int n = sscanf(tok, "%d-%d", &a, &b);
            if (n == 1) b = a;
            if (n < 1) continue;
            for (int c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET(c, &local);
        }
        if (sched_getaffinity(0, sizeof old_set, &old_set) != 0) return;
        cpu_set_t want;
        CPU_AND(&want, &local, &old_set);          // never widen what the process was given
        if (CPU_COUNT(&want) == 0 || CPU_EQUAL(&want, &old_set)) return;
        if (sched_setaffinity(0, sizeof want, &want) == 0) active = true;
    }
    ~LocalCpuGuard()
    {
        if (policy_set) set_policy(0 /* MPOL_DEFAULT */, nullptr, 0);
        if (active) sched_setaffinity(0, sizeof old_set, &old_set);
    }
};
}  // namespace

void* pinned_alloc(size_t bytes, const char* what)
{
    LocalCpuGuard guard;
    void* p = nullptr;
    check_cuda(cudaHostAlloc(&p, std::max<size_t>(bytes, 16), cudaHostAllocDefault), what);
    // cudaHostAlloc populates and pins the pages before it returns, in this thread's context: they follow the MPOL_BIND policy and
    // the CPU mask the guard installed (both restored on scope exit)
    return p;
}

// Host tensors (graph inputs / outputs) are re-created on every run with the same few sizes: cudaHostAlloc / cudaFreeHost cost
// 0.1-1 ms each (driver ioctl + GPU mapping), so freed buffers are parked in a small size-keyed free list instead.
namespace {
std::mutex g_pin_mu;
std::multimap<size_t, void*> g_pin_free;
size_t g_pin_free_bytes = 0;
constexpr size_t PIN_POOL_MAX = (size_t)512 << 20;
}  // namespace

PinnedBuf::PinnedBuf(size_t n) : bytes(n)
{
    {
        std::lock_guard<std::mutex> lock(g_pin_mu);
        auto it = g_pin_free.find(std::max<size_t>(n, 16));
        if (it != g_pin_free.end()) { ptr = it->second; g_pin_free_bytes -= it->first; g_pin_free.erase(it); return; }
    }
    ptr = pinned_alloc(n, "cudaHostAlloc(host tensor)");
}
PinnedBuf::~PinnedBuf()
{
    if (!ptr) return;
    const size_t key = std::max<size_t>(bytes, 16);
    {
        std::lock_guard<std::mutex> lock(g_pin_mu);
        if (g_pin_free_bytes + key <= PIN_POOL_MAX) { g_pin_free.emplace(key, ptr); g_pin_free_bytes += key; return; }
    }
    cudaFreeHost(ptr);
}

// ================================================================================================================
// DevicePool
// ================================================================================================================

DevBlock::~DevBlock() { if (pool && ptr) pool->release(ptr, bytes); }

DevicePool::~DevicePool()
{
    for (auto& s : m_slabs) cudaFree(s.base);
}

void DevicePool::add_slab(size_t min_bytes)
{
    if (frozen) throw std::runtime_error("DevicePool: cannot grow while a CUDA graph owns the pool addresses");
    size_t bytes = std::max<size_t>(min_bytes, m_slabs.empty() ? (size_t)256 << 20 : (size_t)512 << 20);
    bytes = (bytes + ((size_t)2 << 20) - 1) & ~(((size_t)2 << 20) - 1);
    void* p = nullptr;
    check_cuda(cudaMalloc(&p, bytes), "DevicePool cudaMalloc");
    m_slabs.push_back({ p, bytes });
    m_reserved += bytes;
    m_in_use += bytes;  // release() subtracts (clamped at zero: adding after it would count the slab as in use whenever it exceeds m_in_use)
    release(p, bytes);
}

DevPtr DevicePool::alloc(size_t bytes)
{
    if (bytes == 0) bytes = 256;
    bytes = (bytes + 255) & ~(size_t)255;
    for (int attempt = 0; attempt < 2; attempt++) {
        // best fit
        auto best = m_free.end();
        for (auto it = m_free.begin(); it != m_free.end(); ++it)
            if (it->second >= bytes && (best == m_free.end() || it->second < best->second)) best = it;
        if (best != m_free.end()) {
            uintptr_t addr = best->first;
            size_t sz = best->second;
            m_free.erase(best);
            if (sz > bytes) m_free[addr + bytes] = sz - bytes;
            m_in_use += bytes;
            m_high_water = std::max(m_high_water, m_in_use);
            auto blk = std::make_shared<DevBlock>();
            blk->ptr = (void*)addr; blk->bytes = bytes; blk->pool = this;
            return blk;
        }
        add_slab(bytes);
    }
    throw std::runtime_error("DevicePool: allocation failed");
}

void DevicePool::release(void* ptr, size_t bytes)
{
    uintptr_t addr = (uintptr_t)ptr;
    m_in_use -= std::min(m_in_use, bytes);
    auto next = m_free.lower_bound(addr);
    // never merge across slab boundaries
    auto same_slab = [&](uintptr_t a, uintptr_t b) {
        for (auto& s : m_slabs) {
            uintptr_t lo = (uintptr_t)s.base, hi = lo + s.bytes;
            if (a >= lo && a < hi) return b >= lo && b < hi;
        }
        return false;
    };
    if (next != m_free.end() && addr + bytes == next->first && same_slab(addr, next->first)) {
        bytes += next->second;
        next = m_free.erase(next);
    }
    if (next != m_free.begin()) {
        auto prev = std::prev(next);
        if (prev->first + prev->second == addr && same_slab(prev->first, addr)) {
            prev->second += bytes;
            return;
        }
    }
    m_free[addr] = bytes;
}

// ================================================================================================================
// parser (format: src/onnxstream.cpp:2445-2616; SURVEY Appendix A)
// ================================================================================================================

static std::vector<std::string> split(const std::string& s, char delim)
{
    std::vector<std::string> out;
    size_t start = 0;
    while (true) {
        size_t pos = s.find(delim, start);
        if (pos == std::string::npos) { out.push_back(s.substr(start)); break; }
        out.push_back(s.substr(start, pos - start));
        start = pos + 1;
    }
    return out;
}

const std::string* OpDef::attr(const char* key) const
{
    for (auto& a : attrs) if (a.first == key) return &a.second;
    return nullptr;
}

static TensorRef parse_tensor(const std::string& str, bool dynamic_shapes)
{
    TensorRef t;
    if (str.empty()) return t;
    size_t open = str.find('(');
    if (open == std::string::npos || open == 0 || str.back() != ')' || str.find('(', open + 1) != std::string::npos)
        throw std::invalid_argument("Model::parse_tensor_string: invalid tensor format.");
    t.present = true;
    t.name = str.substr(0, open);
    std::string inner = str.substr(open + 1, str.size() - open - 2);
    std::string shape;
    size_t colon = inner.find(':');
    if (colon == std::string::npos) {
        shape = inner;
    } else {
        if (inner.find(':', colon + 1) != std::string::npos) throw std::invalid_argument("Model::parse_tensor_string: invalid tensor format.");
        std::string ty = inner.substr(0, colon);
        shape = inner.substr(colon + 1);
        if (ty.rfind("uint8[", 0) == 0 && ty.back() == ']') {
            auto rv = split(ty.substr(6, ty.size() - 7), ',');
            if (rv.size() != 2) throw std::invalid_argument("Model::parse_tensor_string: invalid uint8 range.");
            t.wtype = DType::u8;
            t.scale = (float)std::stod(rv[0]);
            t.zero_point = std::stoi(rv[1]);
        } else if (ty == "float16") t.wtype = DType::f16;
        else if (ty == "float32") t.wtype = DType::f32;
        else if (ty == "int64") t.wtype = DType::i64;
        else throw std::invalid_argument("Model::parse_tensor_string: unsupported tensor data format.");
    }
    if (!shape.empty()) {
        for (auto& d : split(shape, ',')) {
            int v = std::stoi(d);
            if (v < 0) throw std::invalid_argument("Model::parse_tensor_string: invalid shape (dim < 0).");
            if (v == 0 && !dynamic_shapes) throw std::invalid_argument("Model::parse_tensor_string: invalid shape (dim == 0).");
            t.shape.push_back(v);
        }
    }
    return t;
}

std::vector<OpDef> parse_model_text(const std::string& text, bool dynamic_shapes)
{
    std::vector<OpDef> ops;
    size_t pos = 0, n = text.size();
    while (pos < n) {
        size_t end = pos;
        while (end < n && text[end] != '\n' && text[end] != '\r') end++;
        std::string line = text.substr(pos, end - pos);
        size_t line_pos = pos;
        pos = end;
        while (pos < n && (text[pos] == '\n' || text[pos] == '\r')) pos++;
        if (line.empty()) continue;
        auto sections = split(line, '*');
        if (sections.size() != 3 && sections.size() != 4) throw std::invalid_argument("Model::next_op: invalid format of model line.");
        OpDef op;
        auto first = split(sections[0], ':');
        if (first.size() != 2) throw std::invalid_argument("Model::next_op: invalid format of model line.");
        op.name = first[0];
        op.type = first[1];
        if (op.name.empty()) op.name = "onnxstream_fallback_name_" + std::to_string(line_pos);
        if (sections[1].rfind("input:", 0) != 0 || sections[2].rfind("output:", 0) != 0)
            throw std::invalid_argument("Model::next_op: invalid format of model line.");
        for (auto& s : split(sections[1].substr(6), ';')) op.in.push_back(parse_tensor(s, dynamic_shapes));
        for (auto& s : split(sections[2].substr(7), ';')) op.out.push_back(parse_tensor(s, dynamic_shapes));
        if (sections.size() == 4) {
            for (auto& kv : split(sections[3], ';')) {
                auto p = split(kv, ':');
                if (p.size() != 2) throw std::invalid_argument("Model::next_op: invalid format of model line.");
                op.attrs.emplace_back(p[0], p[1]);
            }
        }
        ops.push_back(std::move(op));
    }
    return ops;
}

// ================================================================================================================
// weight sources
// ================================================================================================================

static void read_blob(const std::string& fn, void* dst, size_t bytes)
{
    FILE* f = fopen(fn.c_str(), "rb");
    if (!f) throw std::runtime_error("read_file: unable to open file (" + fn + ").");
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (sz < 0 || (size_t)sz != bytes) { fclose(f); throw std::invalid_argument("Model::get_tensor_data: mismatch between tensor shape and data size (" + fn + ")."); }
    size_t got = bytes ? fread(dst, 1, bytes, f) : 0;
    fclose(f);
    if (got != bytes) throw std::runtime_error("read_file: unable to read file.");
}

namespace {

// DiskNoCacheWeightsProvider analogue (src/onnxstream.h:331-354): one read per request, straight into pinned staging.
class DiskSource : public WeightSource {
public:
    const void* fetch(const std::string& name, DType, size_t bytes, void* dst) override
    {
        read_blob(path + name, dst, bytes);
        return dst;
    }
    const char* kind() const override { return "nocache"; }
};

// RamWeightsProvider analogue (src/onnxstream.h:666-900): blobs stay in *pinned* host memory after the first load so
// every later run streams them to HBM with cudaMemcpyAsync at full PCIe rate.
class RamSource : public WeightSource {
public:
    explicit RamSource(std::unique_ptr<WeightSource> inner) : m_inner(std::move(inner)) {}
    ~RamSource() override { for (auto& c : m_chunks) cudaFreeHost(c.base); }
    struct Blob { void* ptr; size_t bytes; };
    std::unordered_map<std::string, Blob> m_blobs;
    std::unique_ptr<WeightSource> m_inner;

    // Blobs are bump-allocated, 256-byte aligned, from large pinned chunks in the order they are first requested (= graph
    // order).  A node's weights therefore sit back to back in host memory with exactly the layout the HBM ring gives them, and
    // the streamer can move a whole node with ONE cudaMemcpyAsync (and one NCCL broadcast) instead of one per blob.
    struct Chunk { char* base; size_t cap, used; };
    std::vector<Chunk> m_chunks;

    void* arena_alloc(size_t bytes)
    {
        size_t need = (std::max<size_t>(bytes, 16) + 255) & ~(size_t)255;
        if (m_chunks.empty() || m_chunks.back().used + need > m_chunks.back().cap) {
            size_t cap = std::max<size_t>(need, (size_t)128 << 20);
            void* p = pinned_alloc(cap, "cudaHostAlloc(weights)");
            m_chunks.push_back({ (char*)p, cap, 0 });
        }
        Chunk& c = m_chunks.back();
        void* p = c.base + c.used;
        c.used += need;
        return p;
    }

    void* add(const std::string& name, size_t bytes)
    {
        auto it = m_blobs.find(name);
        if (it != m_blobs.end() && it->second.bytes >= bytes) { it->second.bytes = bytes; return it->second.ptr; }
        void* p = arena_alloc(bytes);
        m_blobs[name] = { p, bytes };
        return p;
    }
    const void* fetch(const std::string& name, DType type, size_t bytes, void* dst) override
    {
        auto it = m_blobs.find(name);
        if (it == m_blobs.end()) {
            if (!m_inner) throw std::invalid_argument("RamWeightsProvider: weights not found: " + name);
            m_inner->path = path;
            void* p = add(name, bytes);
            m_inner->fetch(name, type, bytes, p);
            it = m_blobs.find(name);
        }
        if (it->second.bytes != bytes) throw std::invalid_argument("Model::get_tensor_data: mismatch between tensor shape and data size (" + name + ").");
        return it->second.ptr;
    }
    bool stable_pinned() const override { return true; }
    const char* kind() const override { return "ram"; }
};

}  // namespace

std::unique_ptr<WeightSource> make_disk_source(bool) { return std::make_unique<DiskSource>(); }
std::unique_ptr<WeightSource> make_ram_source(std::unique_ptr<WeightSource> inner) { return std::make_unique<RamSource>(std::move(inner)); }
void* ram_source_add(WeightSource* ram, const std::string& name, size_t bytes)
{
    auto* r = dynamic_cast<RamSource*>(ram);
    if (!r) return nullptr;
    return r->add(name, bytes);
}

// ================================================================================================================
// WeightStreamer: pinned host -> HBM ring on the copy stream
// ================================================================================================================

WeightStreamer::WeightStreamer(size_t capacity, bool host_mirror, ncclComm* comm, int rank, int nranks)
    : m_cap(((capacity + 255) & ~(size_t)255) + (nranks > 1 ? (size_t)256 * nranks : 0)), m_comm(comm), m_rank(rank), m_nranks(nranks)
{
    // (N > 1: room for the per-rank chunk padding of the sharded upload)
    m_sharded = nranks > 1;
    if (const char* e = getenv("OSB_SHARDED_H2D")) m_sharded = e[0] != '0' && nranks > 1;
    check_cuda(cudaStreamCreateWithFlags(&m_copy, cudaStreamNonBlocking), "cudaStreamCreate(copy)");
    if (nranks > 1) check_cuda(cudaStreamCreateWithFlags(&m_coll, cudaStreamNonBlocking), "cudaStreamCreate(collective)");
    check_cuda(cudaMalloc(&m_ring, m_cap), "cudaMalloc(weight ring)");
    if (host_mirror) m_host = (char*)pinned_alloc(m_cap, "cudaHostAlloc(weight staging)");
}

WeightStreamer::~WeightStreamer()
{
    cudaStreamSynchronize(m_copy);
    if (m_coll) cudaStreamSynchronize(m_coll);
    for (auto& s : m_slots) { if (s.ready) cudaEventDestroy(s.ready); if (s.released_ev) cudaEventDestroy(s.released_ev); if (s.h2d_ev) cudaEventDestroy(s.h2d_ev); }
    for (auto e : m_event_pool) cudaEventDestroy(e);
    if (m_ring) cudaFree(m_ring);
    if (m_host) cudaFreeHost(m_host);
    cudaStreamDestroy(m_copy);
    if (m_coll) cudaStreamDestroy(m_coll);
}

cudaEvent_t WeightStreamer::get_event()
{
    if (!m_event_pool.empty()) { auto e = m_event_pool.back(); m_event_pool.pop_back(); return e; }
    cudaEvent_t e;
    check_cuda(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate");
    return e;
}

void WeightStreamer::begin_run()
{
    m_streamed = 0;   // m_live keeps counting slots that are still queued from the previous run
}

// Reserve [off, off+bytes) in the ring.  Slots are FIFO in graph order; a slot can be overwritten once its consumer
// has been *enqueued* (release event recorded) -- the copy stream then waits on that event, so the host never blocks
// on the GPU except when it must overwrite the pinned host mirror of a slot whose H2D has not finished (disk modes).
bool WeightStreamer::try_reserve(size_t bytes, size_t& off)
{
    if (bytes > m_cap) throw std::runtime_error("WeightStreamer: node footprint exceeds ring capacity");
    size_t cand = m_head;
    if (cand + bytes > m_cap) cand = 0;  // wrap; the tail remainder is skipped
    auto overlaps = [&](const Slot& s) { return s.off < cand + bytes && cand < s.off + s.bytes; };
    while (true) {
        bool any = false;
        for (auto& s : m_slots) if (overlaps(s)) { any = true; break; }
        if (!any) break;
        Slot& f = m_slots.front();
        if (!f.released) return false;
        check_cuda(cudaStreamWaitEvent(m_copy, f.released_ev, 0), "cudaStreamWaitEvent(copy, released)");
        if (m_host) check_cuda(cudaEventSynchronize(f.ready), "cudaEventSynchronize(h2d done)");
        m_live -= f.bytes;
        m_event_pool.push_back(f.ready);
        m_event_pool.push_back(f.released_ev);
        if (f.h2d_ev) m_event_pool.push_back(f.h2d_ev);
        m_slots.pop_front();
    }
    off = cand;
    m_head = cand + bytes;
    return true;
}

WeightStreamer::Slot* WeightStreamer::stage(WeightSource& src, const std::vector<Request>& node, bool must)
{
    size_t total = 0;
    for (auto& r : node) total += (r.bytes + 255) & ~(size_t)255;
    if (total == 0) total = 256;
    // sharded upload: the slot is nranks equal chunks (the last ones may be padding)
    const size_t chunk = m_sharded ? ((((total + m_nranks - 1) / m_nranks) + 255) & ~(size_t)255) : 0;
    if (m_sharded) total = std::max(total, chunk * (size_t)m_nranks);
    size_t off = 0;
    if (!try_reserve(total, off)) {
        if (must) throw std::runtime_error("WeightStreamer: ring full although all previous nodes were released");
        return nullptr;
    }
    m_slots.emplace_back();
    Slot& s = m_slots.back();
    s.off = off;
    s.bytes = total;
    s.ready = get_event();
    s.released_ev = get_event();
    s.released = false;
    s.h2d_ev = nullptr;
    // N > 1: the collective of this slot runs on m_coll after this rank's upload (event), so the copy stream is free to start the
    // next slot's upload while NVLink completes this one
    auto after_upload = [&]() -> cudaStream_t {
        if (!m_coll) return m_copy;
        if (!s.h2d_ev) s.h2d_ev = get_event();
        check_cuda(cudaEventRecord(s.h2d_ev, m_copy), "cudaEventRecord(h2d)");
        check_cuda(cudaStreamWaitEvent(m_coll, s.h2d_ev, 0), "cudaStreamWaitEvent(collective, h2d)");
        return m_coll;
    };
    bool do_h2d = (m_nranks == 1) || (m_rank == 0);
    size_t cur = off;
    for (auto& r : node) {
        Blob b;
        b.dev = (char*)m_ring + cur;
        b.bytes = r.bytes;
        // every rank reads the host bytes (small constants are evaluated on the host); only the root uploads them
        b.host = src.fetch(r.name, r.type, r.bytes, m_host ? (char*)m_host + cur : nullptr);
        s.blobs.push_back(b);
        cur += (r.bytes + 255) & ~(size_t)255;
    }
    // one transfer per node when the host copies are laid out exactly like the ring slot (pinned arena of the "ram" sources,
    // or the pinned mirror of the disk sources); otherwise one per blob
    bool contiguous = !s.blobs.empty();
    for (size_t k = 0; k + 1 < s.blobs.size() && contiguous; k++)
        contiguous = (const char*)s.blobs[k + 1].host == (const char*)s.blobs[k].host + ((s.blobs[k].bytes + 255) & ~(size_t)255);
    if (contiguous) {
        size_t span = ((const char*)s.blobs.back().host - (const char*)s.blobs.front().host) + s.blobs.back().bytes;
        if (m_sharded) {
            // every rank holds the same host bytes: upload slice [rank * chunk, (rank + 1) * chunk) of the node, gather the rest over NVLink
            size_t lo = std::min(span, (size_t)m_rank * chunk), hi = std::min(span, lo + chunk);
            if (hi > lo) check_cuda(cudaMemcpyAsync((char*)s.blobs.front().dev + lo, (const char*)s.blobs.front().host + lo, hi - lo, cudaMemcpyHostToDevice, m_copy), "cudaMemcpyAsync(node shard H2D)");
            nccl_allgather_inplace(s.blobs.front().dev, chunk, after_upload());
            m_streamed += hi - lo;     // bytes this rank moved over PCIe
        } else {
            if (do_h2d) check_cuda(cudaMemcpyAsync(s.blobs.front().dev, s.blobs.front().host, span, cudaMemcpyHostToDevice, m_copy), "cudaMemcpyAsync(node H2D)");
            if (m_nranks > 1) nccl_broadcast(s.blobs.front().dev, span, after_upload());
            for (size_t k = 0; k < node.size(); k++) if (node[k].type != DType::i64) m_streamed += node[k].bytes;
        }
    } else {
        for (size_t k = 0; k < node.size(); k++) {
            const Blob& b = s.blobs[k];
            if (!b.bytes || node[k].type == DType::i64) continue;
            if (do_h2d) check_cuda(cudaMemcpyAsync(b.dev, b.host, b.bytes, cudaMemcpyHostToDevice, m_copy), "cudaMemcpyAsync(weights H2D)");
            if (m_nranks > 1) nccl_broadcast(b.dev, b.bytes, after_upload());
            m_streamed += b.bytes;
        }
    }
    check_cuda(cudaEventRecord(s.ready, m_coll ? m_coll : m_copy), "cudaEventRecord(ready)");
    m_live += s.bytes;
    m_peak_live = std::max(m_peak_live, m_live);
    return &s;
}

void WeightStreamer::release(Slot* s, cudaStream_t compute)
{
    check_cuda(cudaEventRecord(s->released_ev, compute), "cudaEventRecord(released)");
    s->released = true;
}

void WeightStreamer::end_run(cudaStream_t compute)
{
    // everything staged must have been consumed; keep slots (their events order the next run's copies)
    for (auto& s : m_slots) if (!s.released) { check_cuda(cudaEventRecord(s.released_ev, compute), "cudaEventRecord"); s.released = true; }
}

}  // namespace osb
