// common.cuh — internals shared by the sm_90a engine's translation units.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <map>
#include <unordered_map>
#include <vector>

#include "../../include/dfgpu.h"

namespace dfgpu {

// ---------------------------------------------------------------------------------------------
// errors: C++ exception inside the library, converted to (code, thread-local message) at the ABI.
// ---------------------------------------------------------------------------------------------
struct Error {
  int code;
  std::string msg;
};
[[noreturn]] inline void fail(int code, const std::string& m) { throw Error{code, m}; }

void set_last_error(const std::string& m);

#define DF_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      ::dfgpu::fail(_e == cudaErrorMemoryAllocation ? DFGPU_ERR_OOM : DFGPU_ERR_CUDA,              \
                    std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" + \
                        std::to_string(__LINE__) + " (" #expr ")");                                \
  } while (0)

template <class Fn>
int guarded(Fn&& fn) {
  try {
    fn();
    return DFGPU_OK;
  } catch (const Error& e) {
    set_last_error(e.msg);
    return e.code;
  } catch (const std::exception& e) {
    set_last_error(std::string("internal: ") + e.what());
    return DFGPU_ERR_INTERNAL;
  }
}

const char* dtype_name(int dt);
int dtype_width(int dt);  // bytes; 0 for bool/utf8
inline bool is_signed_int(int dt) { return dt >= DFGPU_INT8 && dt <= DFGPU_INT64; }
inline bool is_unsigned_int(int dt) { return dt >= DFGPU_UINT8 && dt <= DFGPU_UINT64; }
inline bool is_int(int dt) { return dt >= DFGPU_INT8 && dt <= DFGPU_UINT64; }
inline bool is_float(int dt) { return dt == DFGPU_FLOAT32 || dt == DFGPU_FLOAT64; }
inline bool is_numeric(int dt) { return dt >= DFGPU_INT8 && dt <= DFGPU_FLOAT64; }
// operand types of the interpreter-free kernels: 8-byte numeric, and 4- or 8-byte numeric
inline bool is_numeric8(int dt) { return dt == DFGPU_FLOAT64 || dt == DFGPU_INT64 || dt == DFGPU_UINT64; }
inline bool is_numeric4or8(int dt) { return is_numeric8(dt) || dt == DFGPU_FLOAT32 || dt == DFGPU_INT32 || dt == DFGPU_UINT32; }

}  // namespace dfgpu

// ---------------------------------------------------------------------------------------------
// opaque handle definitions
// ---------------------------------------------------------------------------------------------
struct dfgpu_ctx {
  int device = 0;
  int sm_count = 132;
  size_t device_mem_bytes = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  int64_t launches = 0;
  bool force_direct_kernel = false;  // DFGPU_FP_KERNEL=direct: bypass the TMA pipeline (A/B testing)
  void* flush_buf = nullptr;
  size_t flush_bytes = 0;
  // scratch words shared by the operators, laid out by the SCR_* ranges below
  unsigned long long* d_scratch = nullptr;
  unsigned long long* h_scratch = nullptr;  // pinned
  // pinned staging ring for uploads from pageable memory
  void* stage[2] = {nullptr, nullptr};
  cudaEvent_t stage_ev[2] = {nullptr, nullptr};
  size_t stage_bytes = 0;
  // per-kernel profiling (dfgpu_profile_*): ring of event pairs around the dominant kernels
  static constexpr int kProfRing = 32;
  bool prof_on = false;
  cudaEvent_t prof_ev[kProfRing][2] = {};
  bool prof_pending[kProfRing] = {};
  int prof_next = 0;
  double prof_ms = 0.0;
  int64_t prof_n = 0;
  int prof_begin();          // returns ring slot or -1
  void prof_end(int slot);
  void prof_drain();
  // streamed host->host operators: copy-in / copy-out streams and a cache of pinned result buffers
  cudaStream_t stream_in = nullptr, stream_out = nullptr;
  struct HostBlock { void* p; size_t bytes; bool used; };
  std::vector<HostBlock> host_blocks;
  void* host_alloc(size_t bytes);   // pinned, cached
  void host_release(void* p);
  // multi-GPU
  int rank = 0, world = 1;
  void* nccl_comm = nullptr;

  // Stream-ordered filter/project results (filter_project.cu): each result whose row count is not read yet owns one
  // slot, a pinned [row count, DivideByZero flag] word pair its kernel writes and an event recorded after that kernel.
  // A slot is handed out again only after its event has been observed complete; the slab grows instead of waiting.
  struct FpSlot {
    unsigned long long* words = nullptr;
    cudaEvent_t done = nullptr;
    dfgpu_result* owner = nullptr;  // the pending result, or null
  };
  static constexpr int kFpSlab = 64;  // slots added per growth
  std::vector<FpSlot> fp_slots;
  std::vector<void*> fp_slabs;  // pinned blocks behind fp_slots[].words
  std::vector<int> fp_free;     // slots ready for a new result
  std::vector<int> fp_retired;  // slots of results freed while their kernel could still be running
  int fp_acquire(dfgpu_result* owner);
  void fp_retire(int slot);

  // kernels whose per-device function attributes (dynamic shared memory limit) were set through this
  // ctx: the attribute belongs to the device, so it is tracked per ctx and not per process
  std::vector<const void*> configured_kernels;
  bool first_use(const void* kernel) {
    for (const void* k : configured_kernels)
      if (k == kernel) return false;
    configured_kernels.push_back(kernel);
    return true;
  }

  // device memory: see api.cu
  static constexpr size_t kBigBlock = 256u << 10;
  std::map<size_t, std::vector<void*>> big_free;  // size class -> cached blocks
  std::unordered_map<void*, size_t> big_live;     // block -> size class
  size_t big_cached_bytes = 0;
  void release_cached();
  void* alloc(size_t bytes);
  void free(void* p);
  void use();  // cudaSetDevice(device)
};

struct DevColumn {
  int dtype = 0;
  void* values = nullptr;        // device
  size_t values_bytes = 0;
  uint8_t* validity = nullptr;   // device, bit 0 = row 0 (re-based to offset 0), or null
  int32_t* offsets = nullptr;    // utf8: device i32 offsets (re-based view keeps original values)
  int64_t null_count = 0;
};

namespace dfgpu {
// collectives over the ctx's NCCL communicator (api.cu); counts and offsets in u64 words, all on ctx->stream
void comm_allgather_u64(dfgpu_ctx* ctx, const unsigned long long* send, unsigned long long* recv, size_t count);
void comm_exchange_v(dfgpu_ctx* ctx, const unsigned long long* send, const size_t* send_off, const size_t* send_cnt,
                     unsigned long long* recv, const size_t* recv_off, const size_t* recv_cnt);
void comm_allgather_v(dfgpu_ctx* ctx, const unsigned long long* send, unsigned long long* recv, const size_t* off, const size_t* cnt);
void comm_allgather_bytes_v(dfgpu_ctx* ctx, const void* send, void* recv, const size_t* off, const size_t* cnt);
void comm_allreduce_aggs(dfgpu_ctx* ctx, int naggs, const int* funcs, const int* mtypes, unsigned long long* d_vals, unsigned long long* d_nonnull,
                         unsigned long long* d_rows);
// one Utf8 column on the device (arrow 0.12 BinaryArray): the unit of the multi-source string gather
struct Utf8Source {
  const int* off;
  const unsigned char* bytes;
};
constexpr int UTF8_SRC_SHIFT = 40;  // gather index = (source << 40) | row

// DFGPU_TRACE=1: print host-side phase timings of an operator (each phase synchronised)
struct Trace {
  bool on;
  dfgpu_ctx* ctx;
  double t0;
  explicit Trace(dfgpu_ctx* c);
  void mark(const char* what);
};
// DFGPU_TRACE: name each kernel as it is launched, template arguments included, so that a run shows which
// instantiation the dispatch chose (the kernel tests assert it)
void trace_launch(const char* kernel);

// ceil(work_items / per_block) CTAs, at least 1 and at most per_sm per SM
int grid_for(const dfgpu_ctx* ctx, long long work_items, int per_block, int per_sm);

struct LaunchOpts {
  size_t smem = 0;           // dynamic shared memory bytes
  bool profiled = false;     // timed in the profile ring (dfgpu_profile_get), where the benchmark's kernel times come from
  bool cooperative = false;  // cudaLaunchCooperativeKernel: every CTA of the grid resident at once
};
constexpr LaunchOpts PROFILED{0, true, false};

// Every kernel launch of the library: on ctx->stream, checked, named under DFGPU_TRACE, timed when opts.profiled and
// counted in ctx->launches (dfgpu_kernel_launches).  The arguments must have the kernel's exact parameter types.
template <class... P>
void launch(dfgpu_ctx* ctx, const char* name, void (*kernel)(P...), int grid, int block, const LaunchOpts& opts, const P&... args) {
  const int ps = opts.profiled ? ctx->prof_begin() : -1;
  if (opts.cooperative) {
    void* argv[] = {(void*)&args...};
    DF_CUDA(cudaLaunchCooperativeKernel((const void*)kernel, dim3(grid), dim3(block), argv, opts.smem, ctx->stream));
  } else {
    kernel<<<grid, block, opts.smem, ctx->stream>>>(args...);
  }
  DF_CUDA(cudaGetLastError());
  trace_launch(name);
  ctx->prof_end(ps);
  ctx->launches++;
}

// The words of ctx->h_scratch (pinned) and ctx->d_scratch (device), kScratchWords u64 each, as ranges of one user each,
// so that no user overwrites words another's copy or kernel may still read.
struct ScratchRange {
  int at, words;
};
constexpr ScratchRange SCR_FP_ROWS{0, 1};       // filter/project: the row count its kernel writes to h_scratch (zero-copy)
constexpr ScratchRange SCR_FP_DIV0{1, 1};       // filter/project: its DivideByZero flag, likewise
constexpr ScratchRange SCR_FP_NULLS{2, 24};     // filter/project: null count per program, in d_scratch, copied to h_scratch
constexpr ScratchRange SCR_AGG_HEADER{26, 16};  // aggregate: multi-GPU header record, built in h_scratch and uploaded
constexpr ScratchRange SCR_AGG_NONNULL{42, 8};  // aggregate: the CTR_NONNULL counters, written in h_scratch and uploaded
constexpr ScratchRange SCR_AGG_ROWS{50, 1};     // aggregate: CTR_ROWS, likewise
constexpr ScratchRange SCR_STAGE{64, 64};       // read_words: staging of one synchronous read, free again when it returns
constexpr int kScratchWords = 128;
constexpr ScratchRange kScratchLayout[] = {SCR_FP_ROWS, SCR_FP_DIV0, SCR_FP_NULLS, SCR_AGG_HEADER, SCR_AGG_NONNULL, SCR_AGG_ROWS, SCR_STAGE};
constexpr bool scratch_layout_ok() {
  int end = 0;
  for (const ScratchRange& r : kScratchLayout) {
    if (r.at < end || r.words < 1) return false;
    end = r.at + r.words;
  }
  return end <= kScratchWords;
}
static_assert(scratch_layout_ok(), "the scratch ranges overlap or overflow the scratch buffers");

// Synchronous device -> host copy of `bytes` (at most SCR_STAGE's) through the pinned staging range: copies on ctx->stream,
// synchronises it and copies the words out to `host`.
void read_words(dfgpu_ctx* ctx, const void* dev, size_t bytes, void* host);
unsigned long long read_word(dfgpu_ctx* ctx, const unsigned long long* dev);

// Device blocks that go back to the ctx pool at scope exit (stream-ordered, see dfgpu_ctx::free).
struct DevBufs {
  dfgpu_ctx* ctx;
  std::vector<void*> blocks;
  explicit DevBufs(dfgpu_ctx* c) : ctx(c) {}
  DevBufs(const DevBufs&) = delete;
  DevBufs& operator=(const DevBufs&) = delete;
  ~DevBufs() {
    for (void* q : blocks) ctx->free(q);
  }
  template <class T = unsigned long long>
  T* alloc(size_t bytes) {
    void* q = ctx->alloc(bytes);
    blocks.push_back(q);
    return static_cast<T*>(q);
  }
};

// Returns a column's values, validity and offsets to the ctx pool and nulls them.
void free_column(dfgpu_ctx* ctx, DevColumn& c);
// Sets a column's null count, and frees its bitmap when it has no null: a column without nulls carries no bitmap.
void set_null_count(dfgpu_ctx* ctx, DevColumn& c, int64_t nulls);
}  // namespace dfgpu

struct dfgpu_batch {
  dfgpu_ctx* ctx = nullptr;
  int64_t nrows = 0;
  std::vector<DevColumn> cols;
  bool owns = true;  // false: a view into buffers owned elsewhere (chunks of dfgpu_aggregate_update_host)
  ~dfgpu_batch();  // returns the column buffers to the ctx pool
};

struct dfgpu_result {
  dfgpu_ctx* ctx = nullptr;
  // A stream-ordered filter/project result learns its row count when its kernel has completed: until
  // dfgpu::resolve has run, `pending` is its ctx->fp_slots index and nrows is not valid.
  mutable int64_t nrows = 0;
  mutable int pending = -1;
  mutable bool div_by_zero = false;
  std::vector<DevColumn> cols;
  bool on_host = false;  // columns live in pinned host memory (dfgpu_filter_project_host)
  ~dfgpu_result();
};

namespace dfgpu {
// Makes a result's shape readable: waits for a pending result's kernel, reads its row count, and fails with
// DivideByZero when the kernel raised it (api.cu).  Every entry point that reports a result's shape or data calls it.
void resolve(const dfgpu_result* r);
}  // namespace dfgpu
