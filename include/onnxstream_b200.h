/* onnxstream_b200.h -- the drop-in boundary: C ABI of libonnxstream_b200.so.
 *
 * Part 1 is, entry point for entry point, the reference's FFI (vitoplantamura/OnnxStream src/exports.cpp:42-311), i.e.
 * exactly what its bindings.py / bindings.cs / wasm.js bind.  A maintainer switches by pointing `library_path` at this
 * library; see INTEGRATION.md for the binding stub.  Conventions (unchanged): opaque ModelContext*; strings in are
 * borrowed NUL-terminated char*; strings / structs out are malloc'd and freed with model_free_buffer; model_add_tensor and
 * model_add_weights_file return a raw pointer INTO engine-owned (pinned) host storage that the caller fills;
 * model_get_tensor returns {size_t dims_num; size_t* dims; size_t data_num; float* data;} pointing at live engine memory
 * (float32 tensors only); model_read_file / model_run_2 return a malloc'd error message or NULL; model_run,
 * model_set_option and model_add_tensor throw C++ exceptions across the boundary on error, as the reference does.
 *
 * Part 2 (model_ext_*, model_b200_*) covers Model members the reference's apps poke directly (src/onnxstream.h:944-968)
 * and engine-specific controls; none of them is needed by existing bindings.
 */
#ifndef ONNXSTREAM_B200_H
#define ONNXSTREAM_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ModelContext ModelContext;

/* ---- Part 1: the reference's 16 entry points -------------------------------------------------------------------- */
ModelContext* model_new(void);                                                  /* src/exports.cpp:42-60   ("ram" provider) */
ModelContext* model_new_2(int threads_count, char* wp_name);                    /* src/exports.cpp:62-85   wp_name: ram | nocache | prefetch | ram+nocache | ram+prefetch; threads_count < 0: no backend */
void  model_delete(ModelContext* obj);                                          /* src/exports.cpp:87-90 */
void  model_read_string(ModelContext* obj, char* str);                          /* src/exports.cpp:92-96 */
char* model_read_file(ModelContext* obj, char* fn);                             /* src/exports.cpp:98-109 */
char* model_get_weights_names(ModelContext* obj);                               /* src/exports.cpp:111-148 "dtype:file|dtype:file|..." */
void* model_add_weights_file(ModelContext* obj, char* type, char* name, unsigned int size);   /* src/exports.cpp:150-167 */
void* model_add_tensor(ModelContext* obj, char* type, char* name, unsigned int dims_num, unsigned int* dims); /* src/exports.cpp:169-203 */
void* model_get_tensor(ModelContext* obj, char* name);                          /* src/exports.cpp:205-233 */
char* model_get_all_tensor_names(ModelContext* obj);                            /* src/exports.cpp:235-243 */
void  model_run(ModelContext* obj);                                             /* src/exports.cpp:245-256 */
char* model_run_2(ModelContext* obj);                                           /* src/exports.cpp:258-269 */
void  model_clear_tensors(ModelContext* obj);                                   /* src/exports.cpp:271-274 */
void  model_set_option(ModelContext* obj, char* name, unsigned int value);      /* src/exports.cpp:276-301 (+ "b200_*" names) */
void  model_add_extra_output(ModelContext* obj, char* name);                    /* src/exports.cpp:303-306 */
void  model_free_buffer(void* ptr);                                             /* src/exports.cpp:308-311 */

/* ---- Part 2: extensions ------------------------------------------------------------------------------------------ */
void  model_ext_set_attention_parts(ModelContext* obj, unsigned parts);         /* Model::m_attention_fused_ops_parts (src/onnxstream.h:953) */
void  model_ext_set_range(ModelContext* obj, const char* op_name, float mn, float mx);  /* Model::m_range_data (src/onnxstream.h:946) */
char* model_ext_read_range_data(ModelContext* obj, const char* fn);             /* Model::read_range_data (src/onnxstream.cpp:3436-3479) */
char* model_ext_write_range_data(ModelContext* obj, const char* fn);            /* Model::write_range_data (src/onnxstream.cpp:3481-3497); ranges come from option b200_range_data_calibrate = Model::m_range_data_calibrate */
void  model_ext_add_upcast_pattern(ModelContext* obj, const char* pattern);     /* Model::m_requires_upcast as installed by src/llm.cpp:385-389 */
void  model_ext_push_tensor(ModelContext* obj, const char* type, const char* name, unsigned dims_num, const unsigned* dims, const void* data); /* Model::push_tensor as sd.cpp calls it (src/sd.cpp:1488-1516): copies `data` */
long long model_ext_get_tensor_i64(ModelContext* obj, const char* name, long long* dst, long long cap, size_t* dims, size_t* ndims);
int   model_ext_get_tensor_type(ModelContext* obj, const char* name);           /* TensorDataType value, -1 if absent */
void* model_ext_get_tensor_at(ModelContext* obj, const char* name, unsigned int index);   /* index-th batch sibling of `name` (src/onnxstream.cpp:3040-3050); as model_get_tensor */
void  model_ext_add_output_convert(ModelContext* obj, const char* name);        /* Model::m_outputs_convert_set (src/onnxstream.h:961) */

/* Host-only (works without a CUDA device): parse a model.txt text, run the engine's fusion planner and return a malloc'd report, one
 * line per execution step "KIND n_ops first_op_type first_op_name" plus a final "#summary ..." line (free with model_free_buffer).
 * The planner restates the reference's lookahead fusion (src/onnxstream.cpp:3576-3755) on the whole op list. */
char* model_b200_plan_summary(const char* model_text, int fp16_arithmetic, int fuse_nodes, int fuse_attention, int use_scaled_dp_attn_op);

/* stats: [0] weight ring bytes, [1] peak live streamed weight bytes, [2] largest node footprint, [3] weight bytes streamed in the
 * last run, [4] HBM-resident cached weight bytes, [5] activation pool high-water, [6] input H2D bytes, [7] output D2H bytes,
 * [8] kernel launches, [9] tensor-core launches, [10] steps executed, [11] ops fused away, [12] last run wall ms, [13] last run GPU ms,
 * [14] CUDA-graph replays.  Returns the number of fields available. */
int   model_b200_get_stats(ModelContext* obj, double* out, int n);
double model_b200_run_resident(ModelContext* obj, int steps);   /* replay the captured graph on device-resident inputs; CUDA-event ms, < 0 on error */
int   model_b200_set_comm(ModelContext* obj, void* nccl_comm, int rank, int nranks);  /* weights: rank 0 uploads, NCCL broadcast to the rest */
void  model_b200_profiler(int start);                          /* cudaProfilerStart / cudaProfilerStop */
const char* model_b200_version(void);

/* NCCL bootstrap helpers (the unique id travels over whatever out-of-band channel the host uses, e.g. torch.distributed). */
int   osb_comm_unique_id(char* out128);
void* osb_comm_init(int nranks, int rank, const char* id128);
void  osb_comm_destroy(void* comm);

#ifdef __cplusplus
}
#endif
#endif
