// api.cu — context, memory, batch upload, result download, timing and the NCCL communicator of the
// C ABI declared in include/dfgpu.h.
#include <dlfcn.h>
#include <nccl.h>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <memory>

#include "common.cuh"

namespace dfgpu {

static thread_local std::string g_last_error;
void set_last_error(const std::string& m) { g_last_error = m; }

const char* dtype_name(int dt) {
  switch (dt) {
    case DFGPU_BOOL: return "Boolean";
    case DFGPU_INT8: return "Int8";
    case DFGPU_INT16: return "Int16";
    case DFGPU_INT32: return "Int32";
    case DFGPU_INT64: return "Int64";
    case DFGPU_UINT8: return "UInt8";
    case DFGPU_UINT16: return "UInt16";
    case DFGPU_UINT32: return "UInt32";
    case DFGPU_UINT64: return "UInt64";
    case DFGPU_FLOAT32: return "Float32";
    case DFGPU_FLOAT64: return "Float64";
    case DFGPU_UTF8: return "Utf8";
  }
  return "?";
}

int dtype_width(int dt) {
  switch (dt) {
    case DFGPU_INT8: case DFGPU_UINT8: return 1;
    case DFGPU_INT16: case DFGPU_UINT16: return 2;
    case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: return 4;
    case DFGPU_INT64: case DFGPU_UINT64: case DFGPU_FLOAT64: return 8;
  }
  return 0;
}

static double now_ms() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

Trace::Trace(dfgpu_ctx* c) : on(getenv("DFGPU_TRACE") != nullptr), ctx(c), t0(0) {
  if (on) { cudaStreamSynchronize(ctx->stream); t0 = now_ms(); }
}

void Trace::mark(const char* what) {
  if (!on) return;
  cudaStreamSynchronize(ctx->stream);
  const double t = now_ms();
  fprintf(stderr, "[dfgpu trace] %-28s %8.3f ms\n", what, t - t0);
  t0 = t;
}

void trace_launch(const char* kernel) {
  if (getenv("DFGPU_TRACE")) fprintf(stderr, "[dfgpu trace] launch %s\n", kernel);
}

int grid_for(const dfgpu_ctx* ctx, long long work_items, int per_block, int per_sm) {
  const long long g = (work_items + per_block - 1) / per_block;
  return int(std::max(1ll, std::min(g, (long long)ctx->sm_count * per_sm)));
}

void read_words(dfgpu_ctx* ctx, const void* dev, size_t bytes, void* host) {
  if (bytes > size_t(SCR_STAGE.words) * 8) fail(DFGPU_ERR_INTERNAL, "read_words: " + std::to_string(bytes) + " bytes exceed the staging range");
  unsigned long long* stage = ctx->h_scratch + SCR_STAGE.at;
  DF_CUDA(cudaMemcpyAsync(stage, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(host, stage, bytes);
}

unsigned long long read_word(dfgpu_ctx* ctx, const unsigned long long* dev) {
  unsigned long long v = 0;
  read_words(ctx, dev, 8, &v);
  return v;
}

void free_column(dfgpu_ctx* ctx, DevColumn& c) {
  ctx->free(c.values);
  ctx->free(c.validity);
  ctx->free(c.offsets);
  c.values = nullptr;
  c.validity = nullptr;
  c.offsets = nullptr;
}

void set_null_count(dfgpu_ctx* ctx, DevColumn& c, int64_t nulls) {
  c.null_count = nulls;
  if (nulls == 0) {
    ctx->free(c.validity);
    c.validity = nullptr;
  }
}

}  // namespace dfgpu

using namespace dfgpu;

namespace dfgpu {
void rebase_offsets(dfgpu_ctx* ctx, int* d_off, long long n, int lo);  // utf8_gather.cu
}

// ---------------------------------------------------------------------------------------------
// ctx
// ---------------------------------------------------------------------------------------------
void dfgpu_ctx::use() { DF_CUDA(cudaSetDevice(device)); }

// Device memory.  Small blocks come from CUDA's stream-ordered pool.  Blocks of 256 KiB and more (column
// buffers, hash tables, overflow lists: hundreds of MB each) are kept in a per-ctx cache by size class
// (8 classes per power of two, <= 12.5 % padding) and handed out again without a driver call: the
// stream-ordered pool splits and re-merges big blocks, and a request it cannot serve from a cached
// block maps new physical memory, which takes milliseconds for a table of a few hundred MB.
// Every consumer of these blocks is ordered on ctx->stream (or synchronises its side stream before
// freeing), so immediate reuse is safe.
static size_t big_class(size_t bytes) {
  int lg = 63 - __builtin_clzll((unsigned long long)bytes);
  const size_t step = size_t(1) << (lg - 3);
  return (bytes + step - 1) / step * step;
}

void* dfgpu_ctx::alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0) bytes = 8;
  if (bytes < kBigBlock) {
    DF_CUDA(cudaMallocAsync(&p, bytes, stream));
    return p;
  }
  const size_t cls = big_class(bytes);
  auto it = big_free.find(cls);
  if (it != big_free.end() && !it->second.empty()) {
    p = it->second.back();
    it->second.pop_back();
    big_cached_bytes -= cls;
  } else {
    cudaError_t e = cudaMallocAsync(&p, cls, stream);
    if (e == cudaErrorMemoryAllocation) {  // give the cache back and retry once
      cudaGetLastError();
      release_cached();
      e = cudaMallocAsync(&p, cls, stream);
    }
    DF_CUDA(e);
  }
  big_live[p] = cls;
  return p;
}

void dfgpu_ctx::free(void* p) {
  if (!p) return;
  auto it = big_live.find(p);
  if (it == big_live.end()) {
    cudaFreeAsync(p, stream);
    return;
  }
  big_free[it->second].push_back(p);
  big_cached_bytes += it->second;
  big_live.erase(it);
}

void dfgpu_ctx::release_cached() {
  for (auto& kv : big_free)
    for (void* q : kv.second) cudaFreeAsync(q, stream);
  big_free.clear();
  big_cached_bytes = 0;
  cudaStreamSynchronize(stream);
}

int dfgpu_ctx::prof_begin() {
  if (!prof_on) return -1;
  const int s = prof_next;
  prof_next = (prof_next + 1) % kProfRing;
  if (!prof_ev[s][0]) {
    DF_CUDA(cudaEventCreate(&prof_ev[s][0]));
    DF_CUDA(cudaEventCreate(&prof_ev[s][1]));
  }
  if (prof_pending[s]) {  // slot reuse: fold the old measurement in first (long finished)
    float ms = 0;
    DF_CUDA(cudaEventSynchronize(prof_ev[s][1]));
    DF_CUDA(cudaEventElapsedTime(&ms, prof_ev[s][0], prof_ev[s][1]));
    prof_ms += ms;
    prof_n++;
    prof_pending[s] = false;
  }
  DF_CUDA(cudaEventRecord(prof_ev[s][0], stream));
  return s;
}
void dfgpu_ctx::prof_end(int s) {
  if (s < 0) return;
  DF_CUDA(cudaEventRecord(prof_ev[s][1], stream));
  prof_pending[s] = true;
}
void dfgpu_ctx::prof_drain() {
  for (int s = 0; s < kProfRing; s++) {
    if (!prof_pending[s]) continue;
    float ms = 0;
    DF_CUDA(cudaEventSynchronize(prof_ev[s][1]));
    DF_CUDA(cudaEventElapsedTime(&ms, prof_ev[s][0], prof_ev[s][1]));
    prof_ms += ms;
    prof_n++;
    prof_pending[s] = false;
  }
}

extern "C" int dfgpu_profile_enable(dfgpu_ctx* ctx, int on) {
  return guarded([&] {
    ctx->use();
    ctx->prof_drain();
    ctx->prof_on = on != 0;
    ctx->prof_ms = 0.0;
    ctx->prof_n = 0;
  });
}
extern "C" int dfgpu_profile_get(dfgpu_ctx* ctx, double* kernel_ms, int64_t* launches) {
  return guarded([&] {
    ctx->use();
    ctx->prof_drain();
    *kernel_ms = ctx->prof_ms;
    *launches = ctx->prof_n;
  });
}

int dfgpu_ctx::fp_acquire(dfgpu_result* owner) {
  if (fp_free.empty()) {  // take back the retired slots whose kernel has completed
    for (size_t i = 0; i < fp_retired.size();) {
      const cudaError_t e = cudaEventQuery(fp_slots[size_t(fp_retired[i])].done);
      if (e == cudaErrorNotReady) {
        cudaGetLastError();  // not an error: keep it out of the next launch check
        i++;
        continue;
      }
      DF_CUDA(e);
      fp_free.push_back(fp_retired[i]);
      fp_retired[i] = fp_retired.back();
      fp_retired.pop_back();
    }
  }
  if (fp_free.empty()) {  // all slots in flight: grow rather than wait
    unsigned long long* words = nullptr;
    DF_CUDA(cudaMallocHost(&words, size_t(kFpSlab) * 2 * 8));
    fp_slabs.push_back(words);
    for (int i = 0; i < kFpSlab; i++) {
      FpSlot s;
      s.words = words + 2 * i;
      DF_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
      fp_free.push_back(int(fp_slots.size()));
      fp_slots.push_back(s);
    }
  }
  const int s = fp_free.back();
  fp_free.pop_back();
  FpSlot& slot = fp_slots[size_t(s)];
  slot.words[0] = 0;
  slot.words[1] = 0;
  slot.owner = owner;
  return s;
}

void dfgpu_ctx::fp_retire(int s) {
  fp_slots[size_t(s)].owner = nullptr;
  fp_retired.push_back(s);
}

namespace dfgpu {

// A pending result's kernel has completed (or is waited for here): take its row count and flag, free its slot.
static void settle(const dfgpu_result* r) {
  dfgpu_ctx* ctx = r->ctx;
  dfgpu_ctx::FpSlot& s = ctx->fp_slots[size_t(r->pending)];
  DF_CUDA(cudaEventSynchronize(s.done));
  r->nrows = (int64_t)s.words[0];
  r->div_by_zero = s.words[1] != 0;
  s.owner = nullptr;
  ctx->fp_free.push_back(r->pending);
  r->pending = -1;
}

void resolve(const dfgpu_result* r) {
  if (r->pending >= 0) {
    r->ctx->use();
    settle(r);
  }
  if (r->div_by_zero) fail(DFGPU_ERR_ARROW, "DivideByZero");
}

}  // namespace dfgpu

dfgpu_batch::~dfgpu_batch() {
  if (!ctx || !owns) return;
  cudaSetDevice(ctx->device);
  for (auto& c : cols) free_column(ctx, c);
}
void* dfgpu_ctx::host_alloc(size_t bytes) {
  if (bytes == 0) bytes = 8;
  HostBlock* best = nullptr;
  for (auto& b : host_blocks)
    if (!b.used && b.bytes >= bytes && b.bytes <= 2 * bytes + (1 << 20) && (!best || b.bytes < best->bytes)) best = &b;
  if (best) {
    best->used = true;
    return best->p;
  }
  void* p = nullptr;
  DF_CUDA(cudaMallocHost(&p, bytes));
  host_blocks.push_back(HostBlock{p, bytes, true});
  return p;
}
void dfgpu_ctx::host_release(void* p) {
  for (auto& b : host_blocks)
    if (b.p == p) b.used = false;
}

dfgpu_result::~dfgpu_result() {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  // never waits: the slot returns once its kernel is seen complete, the buffers below go back in stream order
  if (pending >= 0) ctx->fp_retire(pending);
  if (on_host) {
    for (auto& c : cols) ctx->host_release(c.values);
    return;
  }
  for (auto& c : cols) free_column(ctx, c);
}

extern "C" int dfgpu_abi_version(void) { return DFGPU_ABI_VERSION; }
extern "C" const char* dfgpu_last_error(void) { return g_last_error.c_str(); }

extern "C" int dfgpu_device_count(int* out) {
  return guarded([&] {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
      cudaGetLastError();
      n = 0;
    }
    *out = n;
  });
}

// One process (host thread) per GPU: keep that thread and the memory it allocates next — numpy / Arrow buffers,
// cudaMallocHost staging — on the NUMA node the GPU hangs off.  On 2-socket hosts with 8 GPUs, half the GPUs sit
// on each node, and ranks whose pinned buffers the OS places on the far node pay for it in every H2D / D2H
// copy.  Opt out with DFGPU_NUMA=0.  Best effort: silently does
// nothing when sysfs does not expose the topology.
static void bind_to_gpu_numa_node(int device) {
  if (const char* e = getenv("DFGPU_NUMA")) if (atoi(e) == 0) return;
  char bus[64] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return; }
  for (char* c = bus; *c; c++) *c = char(tolower((unsigned char)*c));
  int node = -1;
  {
    FILE* f = fopen((std::string("/sys/bus/pci/devices/") + bus + "/numa_node").c_str(), "r");
    if (!f) return;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
  }
  if (node < 0) {
    if (getenv("DFGPU_TRACE")) fprintf(stderr, "[dfgpu trace] device %d (%s): sysfs reports no NUMA node\n", device, bus);
    return;
  }
  FILE* f = fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r");
  if (!f) return;
  char list[4096] = {0};
  const bool got = fgets(list, sizeof(list), f) != nullptr;
  fclose(f);
  if (!got) return;
  cpu_set_t set;
  CPU_ZERO(&set);
  int ncpu = 0;
  for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    const int k = sscanf(tok, "%d-%d", &a, &b);
    if (k == 1) b = a;
    if (k < 1) continue;
    for (int c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET(c, &set); ncpu++; }
  }
  if (ncpu == 0) return;
  const int rc_aff = sched_setaffinity(0, sizeof(set), &set);
  if (getenv("DFGPU_TRACE")) fprintf(stderr, "[dfgpu trace] device %d (%s) -> NUMA node %d, %d cpus, sched_setaffinity rc=%d\n", device, bus, node, ncpu, rc_aff);
  // set_mempolicy(MPOL_PREFERRED, {node}): later allocations of this thread come from the GPU's node
  unsigned long mask[16] = {0};
  if (node < int(sizeof(mask) * 8)) {
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, 1 /*MPOL_PREFERRED*/, mask, sizeof(mask) * 8);
  }
}

extern "C" int dfgpu_init(int device, dfgpu_ctx** out) {
  return guarded([&] {
    if (!out) fail(DFGPU_ERR_GENERAL, "dfgpu_init: null out");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
      cudaGetLastError();
      fail(DFGPU_ERR_CUDA, "no CUDA device available: this engine has no CPU fallback");
    }
    if (device < 0 || device >= n) fail(DFGPU_ERR_CUDA, "device ordinal " + std::to_string(device) + " out of range");
    auto ctx = std::make_unique<dfgpu_ctx>();
    ctx->device = device;
    ctx->use();
    bind_to_gpu_numa_node(device);
    cudaDeviceProp prop;
    DF_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
      fail(DFGPU_ERR_CUDA, std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major * 10 + prop.minor) +
                               "; this library is built for sm_90a (H100) only");
    ctx->sm_count = prop.multiProcessorCount;
    ctx->device_mem_bytes = prop.totalGlobalMem;
    if (const char* e = getenv("DFGPU_FP_KERNEL")) ctx->force_direct_kernel = std::string(e) == "direct";
    DF_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    DF_CUDA(cudaStreamCreateWithFlags(&ctx->stream_in, cudaStreamNonBlocking));
    DF_CUDA(cudaStreamCreateWithFlags(&ctx->stream_out, cudaStreamNonBlocking));
    DF_CUDA(cudaEventCreate(&ctx->ev_start));
    DF_CUDA(cudaEventCreate(&ctx->ev_stop));
    // keep freed blocks cached in the stream-ordered pool
    cudaMemPool_t pool;
    DF_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thresh = ~0ull;
    DF_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
    DF_CUDA(cudaMalloc(&ctx->d_scratch, kScratchWords * 8));
    DF_CUDA(cudaMemset(ctx->d_scratch, 0, kScratchWords * 8));
    DF_CUDA(cudaMallocHost(&ctx->h_scratch, kScratchWords * 8));
    *out = ctx.release();
  });
}

extern "C" int dfgpu_comm_destroy(dfgpu_ctx* ctx);

extern "C" int dfgpu_shutdown(dfgpu_ctx* ctx) {
  return guarded([&] {
    if (!ctx) return;
    ctx->use();
    cudaStreamSynchronize(ctx->stream);
    // results still pending keep their row count: they outlive the slots that hold it
    for (auto& s : ctx->fp_slots)
      if (s.owner) settle(s.owner);
    for (auto& s : ctx->fp_slots) cudaEventDestroy(s.done);
    for (void* w : ctx->fp_slabs) cudaFreeHost(w);
    dfgpu_comm_destroy(ctx);
    ctx->release_cached();
    if (ctx->flush_buf) cudaFree(ctx->flush_buf);
    for (int i = 0; i < 2; i++) {
      if (ctx->stage[i]) cudaFreeHost(ctx->stage[i]);
      if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
    }
    for (int i = 0; i < dfgpu_ctx::kProfRing; i++)
      for (int j = 0; j < 2; j++)
        if (ctx->prof_ev[i][j]) cudaEventDestroy(ctx->prof_ev[i][j]);
    for (auto& b : ctx->host_blocks) cudaFreeHost(b.p);
    cudaStreamDestroy(ctx->stream_in);
    cudaStreamDestroy(ctx->stream_out);
    cudaFree(ctx->d_scratch);
    cudaFreeHost(ctx->h_scratch);
    cudaEventDestroy(ctx->ev_start);
    cudaEventDestroy(ctx->ev_stop);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
  });
}

extern "C" int dfgpu_sync(dfgpu_ctx* ctx) {
  return guarded([&] {
    ctx->use();
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
  });
}

extern "C" int dfgpu_host_alloc(size_t bytes, void** out) {
  return guarded([&] { DF_CUDA(cudaMallocHost(out, bytes ? bytes : 8)); });
}
extern "C" int dfgpu_host_free(void* p) {
  return guarded([&] {
    if (p) DF_CUDA(cudaFreeHost(p));
  });
}

extern "C" int dfgpu_timer_start(dfgpu_ctx* ctx) {
  return guarded([&] {
    ctx->use();
    DF_CUDA(cudaEventRecord(ctx->ev_start, ctx->stream));
  });
}
extern "C" int dfgpu_timer_stop(dfgpu_ctx* ctx, float* ms) {
  return guarded([&] {
    ctx->use();
    DF_CUDA(cudaEventRecord(ctx->ev_stop, ctx->stream));
    DF_CUDA(cudaEventSynchronize(ctx->ev_stop));
    DF_CUDA(cudaEventElapsedTime(ms, ctx->ev_start, ctx->ev_stop));
  });
}

extern "C" int dfgpu_flush_l2(dfgpu_ctx* ctx) {
  return guarded([&] {
    ctx->use();
    if (!ctx->flush_buf) {
      ctx->flush_bytes = size_t(128) << 20;  // > 2x the 50 MB L2
      DF_CUDA(cudaMalloc(&ctx->flush_buf, ctx->flush_bytes));
    }
    DF_CUDA(cudaMemsetAsync(ctx->flush_buf, 0x5a, ctx->flush_bytes, ctx->stream));
  });
}

extern "C" int dfgpu_kernel_launches(const dfgpu_ctx* ctx, int64_t* out) {
  *out = ctx->launches;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// upload
// ---------------------------------------------------------------------------------------------
namespace {

bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

// host -> device.  Pinned sources are one DMA; pageable sources are pipelined through two pinned
// staging buffers (memcpy of chunk i+1 overlaps the DMA of chunk i).
void h2d(dfgpu_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return;
  if (is_pinned(src)) {
    DF_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return;
  }
  if (!ctx->stage[0]) {
    ctx->stage_bytes = size_t(32) << 20;
    for (int i = 0; i < 2; i++) {
      DF_CUDA(cudaMallocHost(&ctx->stage[i], ctx->stage_bytes));
      DF_CUDA(cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming));
    }
  }
  size_t off = 0;
  int i = 0;
  while (off < bytes) {
    size_t n = std::min(ctx->stage_bytes, bytes - off);
    DF_CUDA(cudaEventSynchronize(ctx->stage_ev[i]));  // previous DMA out of this buffer is done
    memcpy(ctx->stage[i], static_cast<const uint8_t*>(src) + off, n);
    DF_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(dst) + off, ctx->stage[i], n, cudaMemcpyHostToDevice, ctx->stream));
    DF_CUDA(cudaEventRecord(ctx->stage_ev[i], ctx->stream));
    off += n;
    i ^= 1;
  }
}

// copy `len` bits starting at bit `offset` into a fresh byte vector whose bit 0 is the first one
std::vector<uint8_t> rebase_bits(const uint8_t* bits, int64_t offset, int64_t len) {
  std::vector<uint8_t> out(size_t((len + 7) / 8), 0);
  if ((offset & 7) == 0) {
    memcpy(out.data(), bits + (offset >> 3), out.size());
  } else {
    for (int64_t i = 0; i < len; i++)
      if ((bits[(offset + i) >> 3] >> ((offset + i) & 7)) & 1) out[size_t(i >> 3)] |= uint8_t(1u << (i & 7));
  }
  if (len & 7) out.back() &= uint8_t((1u << (len & 7)) - 1u);
  return out;
}

}  // namespace

extern "C" int dfgpu_batch_upload(dfgpu_ctx* ctx, const dfgpu_col* cols, int ncols, dfgpu_batch** out) {
  return guarded([&] {
    if (!ctx || !out || (ncols > 0 && !cols)) fail(DFGPU_ERR_GENERAL, "dfgpu_batch_upload: null argument");
    ctx->use();
    auto b = std::make_unique<dfgpu_batch>();
    b->ctx = ctx;
    b->nrows = ncols > 0 ? cols[0].len : 0;
    for (int i = 0; i < ncols; i++) {
      const dfgpu_col& c = cols[i];
      if (c.len != b->nrows) fail(DFGPU_ERR_GENERAL, "all columns of a RecordBatch must have the same length");
      if (c.len < 0 || c.offset < 0) fail(DFGPU_ERR_GENERAL, "negative length/offset");
      DevColumn d;
      d.dtype = c.dtype;
      std::vector<uint8_t> tmp;
      if (c.validity && c.len > 0) {
        tmp = rebase_bits(c.validity, c.offset, c.len);
        int64_t valid = 0;
        for (uint8_t byte : tmp) valid += __builtin_popcount(byte);
        d.null_count = c.len - valid;
        if (d.null_count > 0) {
          d.validity = (uint8_t*)ctx->alloc(tmp.size());
          // tmp is pageable and short-lived: synchronous-safe copy through the staging path
          h2d(ctx, d.validity, tmp.data(), tmp.size());
          DF_CUDA(cudaStreamSynchronize(ctx->stream));
        }
      }
      const int w = dtype_width(c.dtype);
      if (w > 0) {
        d.values_bytes = size_t(c.len) * size_t(w);
        d.values = ctx->alloc(d.values_bytes);
        if (c.len > 0) {
          if (!c.values) fail(DFGPU_ERR_GENERAL, "null values buffer");
          h2d(ctx, d.values, static_cast<const uint8_t*>(c.values) + size_t(c.offset) * size_t(w), d.values_bytes);
        }
      } else if (c.dtype == DFGPU_BOOL) {
        std::vector<uint8_t> bits = c.len > 0 ? rebase_bits(static_cast<const uint8_t*>(c.values), c.offset, c.len) : std::vector<uint8_t>();
        d.values_bytes = bits.size();
        d.values = ctx->alloc(d.values_bytes);
        if (!bits.empty()) {
          h2d(ctx, d.values, bits.data(), bits.size());
          DF_CUDA(cudaStreamSynchronize(ctx->stream));
        }
      } else if (c.dtype == DFGPU_UTF8) {
        if (!c.offsets) fail(DFGPU_ERR_GENERAL, "Utf8 column without offsets buffer");
        d.offsets = (int32_t*)ctx->alloc(size_t(c.len + 1) * 4);
        h2d(ctx, d.offsets, c.offsets + c.offset, size_t(c.len + 1) * 4);
        const int32_t lo = c.offsets[c.offset], hi = c.offsets[c.offset + c.len];
        if (hi < lo || hi > c.values_bytes) fail(DFGPU_ERR_GENERAL, "corrupt Utf8 offsets");
        // only this batch's bytes [lo, hi) travel (a batch is often a slice of a long column: copying the
        // prefix [0, hi) for every batch is quadratic over a table); the device offsets are rebased by -lo
        d.values_bytes = size_t(hi - lo);
        // whole 16-byte words: the string predicates read aligned 16-byte words (utf8_predicate.cu)
        d.values = ctx->alloc((d.values_bytes + 15) & ~size_t(15));
        if (hi > lo) h2d(ctx, d.values, static_cast<const uint8_t*>(c.values) + lo, size_t(hi - lo));
        rebase_offsets(ctx, d.offsets, c.len + 1, lo);
      } else {
        fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("unsupported column type ") + std::to_string(c.dtype));
      }
      b->cols.push_back(d);
    }
    // the call borrows the host buffers only for its duration
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = b.release();
  });
}

extern "C" int dfgpu_batch_rows(const dfgpu_batch* b, int64_t* nrows) {
  *nrows = b->nrows;
  return 0;
}
extern "C" int dfgpu_batch_free(dfgpu_batch* b) {
  return guarded([&] { delete b; });
}

// ---------------------------------------------------------------------------------------------
// results
// ---------------------------------------------------------------------------------------------
extern "C" int dfgpu_result_shape(const dfgpu_result* r, int64_t* nrows, int* ncols) {
  return guarded([&] {
    resolve(r);
    *nrows = r->nrows;
    *ncols = int(r->cols.size());
  });
}
extern "C" int dfgpu_result_col_dtype(const dfgpu_result* r, int i, int32_t* dtype) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    *dtype = r->cols[size_t(i)].dtype;
  });
}
extern "C" int dfgpu_result_col_bytes(const dfgpu_result* r, int i, int64_t* nbytes) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    resolve(r);
    const DevColumn& c = r->cols[size_t(i)];
    const int w = dtype_width(c.dtype);
    *nbytes = w ? r->nrows * w : int64_t(c.values_bytes);
  });
}
extern "C" int dfgpu_result_col_nulls(const dfgpu_result* r, int i, int64_t* nulls) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    resolve(r);
    *nulls = r->cols[size_t(i)].null_count;
  });
}
extern "C" int dfgpu_result_copy_col(const dfgpu_result* r, int i, void* dst_values, uint8_t* dst_validity, int32_t* dst_offsets) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    resolve(r);
    dfgpu_ctx* ctx = r->ctx;
    ctx->use();
    const DevColumn& c = r->cols[size_t(i)];
    const int w = dtype_width(c.dtype);
    const size_t nb = w ? size_t(r->nrows) * size_t(w) : c.values_bytes;
    if (r->on_host) {
      if (nb && dst_values) memcpy(dst_values, c.values, nb);
      if (dst_validity) memset(dst_validity, 0xff, size_t(r->nrows + 7) / 8);
      return;
    }
    if (nb && dst_values) DF_CUDA(cudaMemcpyAsync(dst_values, c.values, nb, cudaMemcpyDeviceToHost, ctx->stream));
    if (dst_validity) {
      const size_t vb = size_t(r->nrows + 7) / 8;
      if (c.validity) DF_CUDA(cudaMemcpyAsync(dst_validity, c.validity, vb, cudaMemcpyDeviceToHost, ctx->stream));
      else memset(dst_validity, 0xff, vb);
    }
    if (dst_offsets && c.offsets)
      DF_CUDA(cudaMemcpyAsync(dst_offsets, c.offsets, size_t(r->nrows + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
  });
}
extern "C" int dfgpu_result_col_device_ptr(const dfgpu_result* r, int i, const void** dptr) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    if (r->on_host) fail(DFGPU_ERR_GENERAL, "result lives in host memory: use dfgpu_result_col_host_ptr");
    resolve(r);
    *dptr = r->cols[size_t(i)].values;
  });
}
extern "C" int dfgpu_result_on_host(const dfgpu_result* r, int* on_host) {
  return guarded([&] {
    if (!r || !on_host) fail(DFGPU_ERR_GENERAL, "dfgpu_result_on_host: null argument");
    *on_host = r->on_host ? 1 : 0;
  });
}
extern "C" int dfgpu_result_col_host_ptr(const dfgpu_result* r, int i, const void** hptr) {
  return guarded([&] {
    if (i < 0 || size_t(i) >= r->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "result column out of range");
    if (!r->on_host) fail(DFGPU_ERR_GENERAL, "result lives in device memory: use dfgpu_result_copy_col");
    resolve(r);
    *hptr = r->cols[size_t(i)].values;
  });
}
extern "C" int dfgpu_result_free(dfgpu_result* r) {
  return guarded([&] { delete r; });
}

// ---------------------------------------------------------------------------------------------
// communicator: NCCL (loaded lazily so single-GPU use has no libnccl dependency)
// ---------------------------------------------------------------------------------------------
namespace {

struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi& nccl() {
  static NcclApi api;
  if (api.h) return api;
  // RTLD_NOLOAD first: reuse the copy a host application (e.g. torch) already mapped
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW);
  if (!h) fail(DFGPU_ERR_CUDA, std::string("cannot load libnccl: ") + dlerror());
#define LOAD(N)                                                     \
  *(void**)(&api.N) = dlsym(h, "nccl" #N);                          \
  if (!api.N) fail(DFGPU_ERR_CUDA, "libnccl is missing symbol nccl" #N);
  LOAD(GetUniqueId) LOAD(CommInitRank) LOAD(CommDestroy) LOAD(AllGather) LOAD(AllReduce) LOAD(GroupStart) LOAD(GroupEnd)
  LOAD(Send) LOAD(Recv) LOAD(Broadcast)
  LOAD(GetErrorString)
#undef LOAD
  api.h = h;
  return api;
}

#define DF_NCCL(expr)                                                                                        \
  do {                                                                                                       \
    ncclResult_t _r = (expr);                                                                                \
    if (_r != ncclSuccess) fail(DFGPU_ERR_CUDA, std::string("NCCL error: ") + nccl().GetErrorString(_r) + " (" #expr ")"); \
  } while (0)

}  // namespace

extern "C" int dfgpu_comm_unique_id(uint8_t out_id[128]) {
  return guarded([&] {
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
    ncclUniqueId id;
    DF_NCCL(nccl().GetUniqueId(&id));
    memcpy(out_id, &id, 128);
  });
}

extern "C" int dfgpu_comm_init(dfgpu_ctx* ctx, int rank, int world, const uint8_t nccl_unique_id[128]) {
  return guarded([&] {
    if (!ctx) fail(DFGPU_ERR_GENERAL, "dfgpu_comm_init: null ctx");
    if (world < 1 || rank < 0 || rank >= world) fail(DFGPU_ERR_GENERAL, "bad rank/world");
    ctx->use();
    if (ctx->nccl_comm) fail(DFGPU_ERR_GENERAL, "communicator already initialised");
    ctx->rank = rank;
    ctx->world = world;
    if (world == 1) return;
    ncclUniqueId id;
    memcpy(&id, nccl_unique_id, 128);
    ncclComm_t comm;
    DF_NCCL(nccl().CommInitRank(&comm, world, id, rank));
    ctx->nccl_comm = comm;
  });
}

extern "C" int dfgpu_comm_world(const dfgpu_ctx* ctx, int64_t* world) {
  *world = ctx ? ctx->world : 1;
  return 0;
}

extern "C" int dfgpu_comm_destroy(dfgpu_ctx* ctx) {
  return guarded([&] {
    if (ctx && ctx->nccl_comm) {
      ctx->use();
      nccl().CommDestroy((ncclComm_t)ctx->nccl_comm);
      ctx->nccl_comm = nullptr;
    }
    if (ctx) {
      ctx->world = 1;
      ctx->rank = 0;
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Collectives used by the partial-aggregate merge (aggregate.cu: agg_exchange_groups; SURVEY.md §8e).
// All traffic is u64 words on ctx->stream; counts / offsets are in words.
//   comm_allgather_u64 : fixed-size all-gather (headers, counts)
//   comm_exchange_v    : personalised all-to-all — one grouped ncclSend / ncclRecv pair per peer (the
//                        owner-partitioned exchange of partial aggregates); the self segment is copied locally
//   comm_allgather_v   : every rank's final segment to every rank (one grouped ncclBroadcast per root)
//   comm_allreduce_aggs: no-GROUP-BY accumulators: one ncclAllReduce each (ncclSum on f64/u64, ncclMin/ncclMax
//                        on the order-preserving u64 encoding)
// ---------------------------------------------------------------------------------------------
namespace dfgpu {

static ncclComm_t comm_of(dfgpu_ctx* ctx) {
  if (!ctx->nccl_comm) fail(DFGPU_ERR_GENERAL, "world > 1 but no communicator");
  return (ncclComm_t)ctx->nccl_comm;
}

void comm_allgather_u64(dfgpu_ctx* ctx, const unsigned long long* send, unsigned long long* recv, size_t count) {
  DF_NCCL(nccl().AllGather(send, recv, count, ncclUint64, comm_of(ctx), ctx->stream));
}

void comm_exchange_v(dfgpu_ctx* ctx, const unsigned long long* send, const size_t* send_off, const size_t* send_cnt,
                     unsigned long long* recv, const size_t* recv_off, const size_t* recv_cnt) {
  NcclApi& N = nccl();
  ncclComm_t comm = comm_of(ctx);
  const int W = ctx->world, me = ctx->rank;
  if (send_cnt[me])
    DF_CUDA(cudaMemcpyAsync(recv + recv_off[me], send + send_off[me], send_cnt[me] * 8, cudaMemcpyDeviceToDevice, ctx->stream));
  DF_NCCL(N.GroupStart());
  for (int r = 0; r < W; r++) {
    if (r == me) continue;
    if (send_cnt[r]) DF_NCCL(N.Send(send + send_off[r], send_cnt[r], ncclUint64, r, comm, ctx->stream));
    if (recv_cnt[r]) DF_NCCL(N.Recv(recv + recv_off[r], recv_cnt[r], ncclUint64, r, comm, ctx->stream));
  }
  DF_NCCL(N.GroupEnd());
}

void comm_allgather_v(dfgpu_ctx* ctx, const unsigned long long* send, unsigned long long* recv, const size_t* off, const size_t* cnt) {
  NcclApi& N = nccl();
  ncclComm_t comm = comm_of(ctx);
  const int W = ctx->world, me = ctx->rank;
  DF_NCCL(N.GroupStart());
  for (int r = 0; r < W; r++) {
    if (!cnt[r]) continue;
    DF_NCCL(N.Broadcast(r == me ? (const void*)send : (const void*)(recv + off[r]), recv + off[r], cnt[r], ncclUint64, r, comm, ctx->stream));
  }
  DF_NCCL(N.GroupEnd());
}

// byte-granular all-gather of segments of different sizes (one grouped ncclBroadcast per root): the regroup merge of
// Utf8 / wide-key aggregates ships whole result columns
void comm_allgather_bytes_v(dfgpu_ctx* ctx, const void* send, void* recv, const size_t* off, const size_t* cnt) {
  NcclApi& N = nccl();
  ncclComm_t comm = comm_of(ctx);
  const int W = ctx->world, me = ctx->rank;
  DF_NCCL(N.GroupStart());
  for (int r = 0; r < W; r++) {
    if (!cnt[r]) continue;
    char* dst = static_cast<char*>(recv) + off[r];
    DF_NCCL(N.Broadcast(r == me ? send : (const void*)dst, dst, cnt[r], ncclInt8, r, comm, ctx->stream));
  }
  DF_NCCL(N.GroupEnd());
}

void comm_allreduce_aggs(dfgpu_ctx* ctx, int naggs, const int* funcs, const int* mtypes, unsigned long long* d_vals, unsigned long long* d_nonnull,
                         unsigned long long* d_rows /* [1] rows seen, summed */) {
  NcclApi& N = nccl();
  ncclComm_t comm = comm_of(ctx);
  DF_NCCL(N.GroupStart());
  for (int a = 0; a < naggs; a++) {
    ncclDataType_t dt = ncclUint64;
    ncclRedOp_t op = ncclSum;
    if (funcs[a] == DFGPU_AGG_MIN) op = ncclMin;
    else if (funcs[a] == DFGPU_AGG_MAX) op = ncclMax;
    else if (funcs[a] == DFGPU_AGG_SUM && mtypes[a] == 1 /*MT_F64*/) dt = ncclFloat64;
    else if (funcs[a] == DFGPU_AGG_SUM && mtypes[a] == 2 /*MT_F32*/) dt = ncclFloat32;
    // f32 accumulators occupy the low 4 bytes of their 8-byte cell
    DF_NCCL(N.AllReduce(d_vals + a, d_vals + a, 1, dt, op, comm, ctx->stream));
  }
  // non-null input counts per aggregate (an aggregate that saw none anywhere is null) and the row count
  DF_NCCL(N.AllReduce(d_nonnull, d_nonnull, 8, ncclUint64, ncclSum, comm, ctx->stream));
  DF_NCCL(N.AllReduce(d_rows, d_rows, 1, ncclUint64, ncclSum, comm, ctx->stream));
  DF_NCCL(N.GroupEnd());
}

}  // namespace dfgpu
