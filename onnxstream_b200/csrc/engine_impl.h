// engine_impl.h -- private declarations shared by engine.cpp / engine_run.cpp / capi.cpp.
#pragma once

#include "engine.h"
#include "../../include/onnxstream_b200_kernels.h"

#include <cuda_runtime.h>
#include <deque>
#include <string>
#include <vector>

namespace osb {

// Pinned host -> HBM ring on a side stream.  One slot per streamed weight blob; slots are FIFO in graph order.
class WeightStreamer {
public:
    struct Blob {
        void* dev = nullptr;
        const void* host = nullptr;      // host bytes of the blob (valid until the slot is recycled)
        size_t bytes = 0;
    };
    struct Slot {                        // one node's weights: a contiguous reservation in the ring
        size_t off = 0, bytes = 0;
        std::vector<Blob> blobs;
        cudaEvent_t ready = nullptr;     // recorded on the copy stream after the H2D (+ broadcast) of every blob
        cudaEvent_t released_ev = nullptr;  // recorded on the compute stream after the consuming kernels
        cudaEvent_t h2d_ev = nullptr;       // N > 1: recorded on the copy stream after this rank's upload; the collective stream waits on it
        bool released = false;
    };
    struct Request { std::string name; DType type; size_t bytes; };

    WeightStreamer(size_t capacity, bool host_mirror, ncclComm* comm, int rank, int nranks);
    ~WeightStreamer();

    void begin_run();
    Slot* stage(WeightSource& src, const std::vector<Request>& node, bool must);
    void release(Slot* s, cudaStream_t compute);
    void end_run(cudaStream_t compute);

    size_t capacity() const { return m_cap; }
    size_t peak_live() const { return m_peak_live; }
    size_t streamed() const { return m_streamed; }
    cudaStream_t copy_stream() const { return m_copy; }
    // N > 1 only: every rank uploads 1/N of each node over its own PCIe link and an in-place ncclAllGather completes the slot
    // (N x the aggregate host->device bandwidth of a root upload + ncclBroadcast).  Default at N > 1; OSB_SHARDED_H2D=0 selects the
    // root-upload + broadcast variant.
    void set_sharded_upload(bool on) { m_sharded = on && m_nranks > 1; }

private:
    size_t m_cap = 0, m_head = 0, m_live = 0, m_peak_live = 0, m_streamed = 0;
    void* m_ring = nullptr;
    void* m_host = nullptr;
    cudaStream_t m_copy = nullptr;
    cudaStream_t m_coll = nullptr;       // N > 1: NCCL collectives run here, so the upload of slot k+1 overlaps the gather of slot k
    std::deque<Slot> m_slots;
    std::vector<cudaEvent_t> m_event_pool;
    ncclComm* m_comm = nullptr;
    int m_rank = 0, m_nranks = 1;
    bool m_sharded = false;

    bool try_reserve(size_t bytes, size_t& off);
    cudaEvent_t get_event();
    void nccl_broadcast(void* dev, size_t bytes, cudaStream_t st);
    void nccl_allgather_inplace(void* dev, size_t chunk_bytes, cudaStream_t st);
};

}  // namespace osb
