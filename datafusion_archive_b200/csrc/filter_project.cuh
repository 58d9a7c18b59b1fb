// filter_project.cuh — parameter block and chained-scan helpers shared by the two filter/project
// kernels (filter_project.cu: direct-load kernel; filter_project_tma.cu: TMA-staged pipeline).
#pragma once
#include "expr_vm.cuh"

namespace dfgpu {

constexpr int FP_THREADS = 256;
constexpr int FP_WARPS = FP_THREADS / 32;
constexpr int FP_R = 4;       // rows per interpreter pass (per thread)
constexpr int FP_CHUNKS = 2;  // interpreter passes per tile
constexpr int FP_ITEMS = FP_R * FP_CHUNKS;
constexpr int FP_TILE = FP_THREADS * FP_ITEMS;

struct FPParams {
  ProgramSet ps;  // program 0 = predicate when has_pred, projections follow
  void* out[kMaxProgs];
  // no-predicate queries over nullable inputs: per-projection validity bitmap (32 rows per word) and
  // null counter; null when the projection cannot produce nulls
  unsigned* out_valid[kMaxProgs];
  unsigned long long* null_counts;  // [kMaxProgs]
  long long nrows;
  int ntiles;
  int has_pred;
  int nproj;
  unsigned long long* tile_status;  // [ntiles], zeroed per launch
  unsigned* ticket;                 // zeroed per launch
  unsigned long long* out_count;
  unsigned* err_flag;
  // TMA-staged kernel only: layout of the two shared-memory rings.  Ring A stages hold the column
  // slices the predicate reads, ring B stages the slices the projections read (-1 = not in ring).
  int col_offA[kMaxCols];
  int col_offB[kMaxCols];
  int col_w[kMaxCols];  // element width of column slot s
  int stage_bytesA, stage_bytesB;
  int nstagesA, nstagesB;
  int lag;    // tiles between the predicate pass and the projection pass
  int delay;  // waves between publishing a tile's count and resolving the offsets of its wave (1 <= delay <= lag)
  // "fast shapes" (Leaf, as ProgramBuilder::add recognised them): the TMA kernel runs them without the interpreter
  LeafChain pred_fast;  // the predicate as a comparison chain
  Leaf proj_fast[kMaxProgs];
  // queries with a predicate whose projection can hold a CASE-made null (direct kernel, extended interpreter only): one
  // validity byte per selected row, in output order; null for every other projection
  unsigned char* out_vbytes[kMaxProgs];
};

constexpr unsigned long long ST_AGG = 1ull << 62, ST_INCL = 2ull << 62, ST_MASK = (1ull << 62) - 1;

__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}


// filter_project_tma.cu: persistent warp-specialised kernel fed by cp.async.bulk (TMA) through a
// shared-memory ring.  Returns false when the shape does not fit it (caller uses the direct kernel).
bool launch_fp_tma(dfgpu_ctx* ctx, FPParams& p);

}  // namespace dfgpu
