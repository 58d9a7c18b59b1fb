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

struct FastOp {
  int kind;  // 0 = use the interpreter, 1 = copy column a, 2 = a op column b, 3 = a op imm
  int op;    // VOp
  int a, b;  // column slots
  int ty;    // operand dtype: Float64 / Int64 / UInt64 / Float32 / Int32 / UInt32
  int _pad;
  unsigned long long imm;  // raw bits, widened like DevInsn::imm
};

// predicate fast shape: up to 4 Float64 comparisons chained left to right with AND / OR
//   t0 [conn1 t1 [conn2 t2 [conn3 t3]]]   (each term: COL cmp COL | COL cmp IMM)
struct FastPred {
  int nterms;  // 0 = use the interpreter
  int conn[4]; // conn[i] joins the running result with term i: 0 = AND, 1 = OR
  FastOp term[4];
};

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
  // "fast shapes": single-operation programs over 4- and 8-byte numeric columns are recognised on the host and executed by
  // straight-line code instead of the interpreter (same arithmetic, no decode in the inner loop).
  //   predicate : chain of (COL cmp COL | COL cmp IMM) joined by AND / OR
  //   projection: COL | COL op COL | COL op IMM          (op in + - * /)
  FastPred pred_fast;
  FastOp proj_fast[kMaxProgs];
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
