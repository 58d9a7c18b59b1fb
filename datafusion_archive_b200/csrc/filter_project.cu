// filter_project.cu — FilterRelation + ProjectRelation as ONE order-preserving stream-compaction
// kernel (K1 predicate-eval + K2 filter-gather + K3 fused expr/project of SURVEY.md §2b).
//
// Reference path replaced (per batch): predicate closure -> BooleanArray (src/execution/filter.rs:50),
// per-column builder gather of EVERY input column (filter.rs:55-57,79-110), then one closure pass
// per projection expression (src/execution/projection.rs:49-50).  Here: one pass over the referenced
// columns only; the predicate lives in registers as ballot masks, never in HBM; projected values are
// computed in registers and written straight to their compacted position.
//
// Order preservation (filter.rs:86-90 appends in row order) = single-pass chained scan with
// decoupled look-back across tiles; tiles are claimed through an atomic ticket so that a tile's
// predecessors are always resident (forward progress without any grid-wide barrier).
#include <memory>

#include "filter_project.cuh"

namespace dfgpu {

// NULLS: some referenced column has a validity bitmap.  The predicate is evaluated with arrow's null
// semantics (a null And/Or result reads as false, like `filter.value(i)` in filter.rs:86).  With a
// predicate the projections then see null-free arrays, exactly like the reference: `fn filter` copies
// values and drops the bitmap (filter.rs:83-91) before ProjectRelation runs.  Without a predicate the
// projections run on the original arrays and their validity is written out (32 rows per ballot word).  A CASE-made null
// is a null under a predicate too: the extended interpreter writes the validity of such a projection as one byte per
// selected row (out_vbytes), packed after the kernel.
template <int DEPTH, bool NULLS>
__global__ void __launch_bounds__(FP_THREADS) k_filter_project(const __grid_constant__ FPParams p) {
  __shared__ int s_tile;
  __shared__ unsigned s_wcount[FP_ITEMS * FP_WARPS];
  __shared__ unsigned s_woff[FP_ITEMS * FP_WARPS];
  __shared__ unsigned long long s_prefix;
  static_assert(FP_ITEMS * FP_WARPS == 64, "scan below assumes 64 (item,warp) counters = 2 per lane");

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;

  for (;;) {
    if (tid == 0) s_tile = (int)atomicAdd(p.ticket, 1u);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= p.ntiles) break;
    const long long base = (long long)tile * FP_TILE;

    // ---- phase 1: predicate -> per-thread flag bits (bit j = row base + j*THREADS + tid) ----
    unsigned flags = 0;
    bool bad = false;
#pragma unroll 1
    for (int c = 0; c < FP_CHUNKS; c++) {
      GlobalRows<FP_R> src;
      src.valid = 0;
#pragma unroll
      for (int r = 0; r < FP_R; r++) {
        long long row = base + (long long)(c * FP_R + r) * FP_THREADS + tid;
        src.rows[r] = row < p.nrows ? row : -1;
        if (row < p.nrows) src.valid |= 1u << r;
      }
      if (p.has_pred) {
        unsigned long long v[FP_R];
        unsigned ov;
        unsigned b = eval_program_n<DEPTH, FP_R, false, NULLS>(p.ps, 0, src, v, ov);
        bad = bad || (b != 0);
#pragma unroll
        for (int r = 0; r < FP_R; r++)
          if (((src.valid >> r) & 1u) && (v[r] & 1ull)) flags |= 1u << (c * FP_R + r);
      } else {
        flags |= src.valid << (c * FP_R);
      }
    }
#pragma unroll
    for (int j = 0; j < FP_ITEMS; j++) {
      unsigned b = __ballot_sync(0xffffffffu, (flags >> j) & 1u);
      if (lane == 0) s_wcount[j * FP_WARPS + warp] = __popc(b);
    }
    __syncthreads();

    // ---- warp 0: scan the 64 (item,warp) counts, then chain to the preceding tiles ----
    if (warp == 0) {
      unsigned c0 = s_wcount[2 * lane], c1 = s_wcount[2 * lane + 1];
      unsigned incl = c0 + c1;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      unsigned excl = incl - (c0 + c1);
      s_woff[2 * lane] = excl;
      s_woff[2 * lane + 1] = excl + c0;
      const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);

      unsigned long long prefix = 0;
      if (!p.has_pred) {
        prefix = (unsigned long long)base;  // nothing is dropped: positions are known without chaining
      } else if (tile == 0) {
        if (lane == 0) st_relaxed(&p.tile_status[0], ST_INCL | total);
      } else {
        if (lane == 0) st_relaxed(&p.tile_status[tile], ST_AGG | total);
        long long look = (long long)tile - 1;
        unsigned long long run = 0;
        for (;;) {
          const long long idx = look - lane;
          unsigned long long s = idx >= 0 ? ld_relaxed(&p.tile_status[idx]) : ST_INCL;  // before tile 0: inclusive 0
          while (__any_sync(0xffffffffu, (s >> 62) == 0)) {
            if ((s >> 62) == 0) s = ld_relaxed(&p.tile_status[idx]);
          }
          const unsigned incl_mask = __ballot_sync(0xffffffffu, (s >> 62) == 2);
          if (incl_mask) {
            const int first = __ffs(incl_mask) - 1;  // nearest predecessor holding an inclusive prefix
            run += warp_sum64(lane <= first ? (s & ST_MASK) : 0ull);
            break;
          }
          run += warp_sum64(s & ST_MASK);
          look -= 32;
        }
        prefix = run;
        if (lane == 0) st_relaxed(&p.tile_status[tile], ST_INCL | (prefix + total));
      }
      if (lane == 0) {
        s_prefix = prefix;
        if (tile == p.ntiles - 1) *p.out_count = prefix + total;
      }
    }
    __syncthreads();

    // ---- phase 2: evaluate the projections, write selected rows at their compacted position ----
    const unsigned long long prefix = s_prefix;
    for (int q = 0; q < p.nproj; q++) {
      const int prog = q + p.has_pred;
      const int odt = p.ps.out_dtype[prog];
      void* o = p.out[q];
#pragma unroll 1
      for (int c = 0; c < FP_CHUNKS; c++) {
        GlobalRows<FP_R> src;
        src.valid = 0;
#pragma unroll
        for (int r = 0; r < FP_R; r++) {
          long long row = base + (long long)(c * FP_R + r) * FP_THREADS + tid;
          src.rows[r] = row < p.nrows ? row : -1;
          if (row < p.nrows) src.valid |= 1u << r;
        }
        unsigned long long v[FP_R];
        unsigned ov = (1u << FP_R) - 1u;
        unsigned b;
        if (NULLS && !p.has_pred) b = eval_program_n<DEPTH, FP_R, false, true>(p.ps, prog, src, v, ov);
        else b = eval_program_n<DEPTH, FP_R, false, false>(p.ps, prog, src, v, ov);
        if (NULLS && !p.has_pred && p.out_valid[q]) {
#pragma unroll
          for (int r = 0; r < FP_R; r++) {
            const bool inb = (src.valid >> r) & 1u;
            const unsigned vb = __ballot_sync(0xffffffffu, inb && ((ov >> r) & 1u));
            const unsigned ib = __ballot_sync(0xffffffffu, inb);
            if (lane == 0 && ib) {
              p.out_valid[q][src.rows[r] >> 5] = vb;  // the warp's 32 rows are consecutive and 32-aligned
              const unsigned nn = __popc(ib & ~vb);
              if (nn) atomicAdd(&p.null_counts[q], (unsigned long long)nn);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < FP_R; r++) {
          const int j = c * FP_R + r;
          const bool f = (flags >> j) & 1u;
          const unsigned m = __ballot_sync(0xffffffffu, f);
          if (f) {
            const unsigned long long idx = prefix + s_woff[j * FP_WARPS + warp] + __popc(m & lt_mask);
            store_elem(o, odt, (long long)idx, v[r]);
            if constexpr (DEPTH == kCaseDepth)
              if (NULLS && p.out_vbytes[q]) p.out_vbytes[q][idx] = (unsigned char)((ov >> r) & 1u);
            // DivideByZero only counts for rows that survive the filter: ProjectRelation runs on
            // the filtered batch (src/execution/context.rs:140-161).
            if ((b >> r) & 1u) bad = true;
          }
        }
      }
    }
    if (bad) *p.err_flag = 1u;
    __syncthreads();  // s_tile / s_wcount are reused by the next tile
  }
}

// one byte per row -> bits (LSB first), one warp per 32 rows and output word; `zeros` (may be null) gains the number of
// zero bytes: the nulls, when the bytes are validity
__global__ void __launch_bounds__(256) k_pack_bits(const unsigned char* __restrict__ bytes, long long n, unsigned* __restrict__ words,
                                                   unsigned long long* __restrict__ zeros) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long padded = (n + 31) / 32 * 32;
  unsigned z = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < padded; i += stride) {
    const unsigned m = __ballot_sync(0xffffffffu, i < n && bytes[i] != 0);
    const unsigned in = __ballot_sync(0xffffffffu, i < n);
    if ((threadIdx.x & 31) == 0) {
      words[i >> 5] = m;
      z += __popc(in & ~m);
    }
  }
  if (zeros && z) atomicAdd(zeros, (unsigned long long)z);
}
static void pack_bits(dfgpu_ctx* ctx, const unsigned char* bytes, long long n, unsigned* words, unsigned long long* zeros) {
  launch(ctx, "k_pack_bits", k_pack_bits, grid_for(ctx, (n + 31) / 32 * 32, 256, 8), 256, {}, bytes, n, words, zeros);
}
template <int DEPTH, bool NULLS = false>
static void launch_fp(dfgpu_ctx* ctx, const FPParams& p) {
  int per_sm = 0;
  DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_filter_project<DEPTH, NULLS>, FP_THREADS, 0));
  if (per_sm < 1) per_sm = 1;
  static const std::string name = "k_filter_project<" + depth_arg(DEPTH) + (NULLS ? ", true>" : ", false>");
  launch(ctx, name.c_str(), k_filter_project<DEPTH, NULLS>, grid_for(ctx, p.ntiles, 1, per_sm), FP_THREADS, PROFILED, p);
}

void gather_utf8(dfgpu_ctx* ctx, const DevColumn& src, const unsigned long long* d_idx, long long nsel, DevColumn* out);

// A batch of the given column types and no data, for typing programs without a device.  Its ctx is null: it owns
// nothing and its destructor frees nothing.
static dfgpu_batch schema_only(const int32_t* dtypes, int ncols) {
  dfgpu_batch b;
  for (int i = 0; i < ncols; i++) {
    DevColumn c;
    c.dtype = dtypes[i];
    b.cols.push_back(c);
  }
  return b;
}

// nproj == 0: FilterRelation alone emits every input column (filter.rs:55-57).  Points proj / proj_len / nproj at one
// column program per input column, held in `ident`.
struct IdentityProjection {
  std::vector<dfgpu_insn> insn;
  std::vector<const dfgpu_insn*> ptr;
  std::vector<int> len;
};
template <class DtypeOf>
static void project_every_column(int ncols, DtypeOf dtype_of, IdentityProjection& ident, const dfgpu_insn* const*& proj,
                                 const int*& proj_len, int& nproj) {
  if (nproj != 0) return;
  ident.insn.assign(size_t(ncols), dfgpu_insn{});
  for (int i = 0; i < ncols; i++) {
    ident.insn[size_t(i)].op = DFGPU_OP_COL;
    ident.insn[size_t(i)].col = i;
    ident.insn[size_t(i)].dtype = dtype_of(i);
    ident.ptr.push_back(&ident.insn[size_t(i)]);
    ident.len.push_back(1);
  }
  nproj = ncols;
  proj = ident.ptr.data();
  proj_len = ident.len.data();
}

// The WHERE program: program 0 of the set, and Boolean (filter.rs:64-66).
static void add_predicate(ProgramBuilder& pb, const dfgpu_insn* pred, int pred_len) {
  if (pb.out_dtype(pb.add(pred, pred_len, "predicate")) != DFGPU_BOOL)
    fail(DFGPU_ERR_EXECUTION, "Filter expression did not evaluate to boolean");
}

// One output column of dfgpu_filter_project: how it is computed, and what the call allocates and settles for it.
struct OutCol {
  enum Kind {
    VALUE,        // fixed-width value, written by the kernel
    BOOL,         // Boolean: the kernel writes one byte per selected row, packed into bits afterwards
    UTF8_GATHER,  // a Utf8 input column, gathered by the selected row numbers after the kernel (utf8_gather.cu)
    UTF8_VIEW,    // a Utf8 function of one, evaluated over those row numbers (utf8_function.cu)
  } kind = VALUE;
  int slot = -1;  // VALUE / BOOL: the kernel's projection index (its program is slot + has_pred)
  int src = -1;   // UTF8_*: the input column, whose validity the result keeps without a WHERE
  int view = -1;  // UTF8_VIEW: the builder's Utf8 view
  // Under a WHERE the kernel drops the input bitmaps, so only a CASE-made null is a null: the kernel writes such a
  // projection's validity as one byte per selected row (vbytes), packed into the bitmap afterwards.
  bool case_nulls = false;
  bool kernel_validity = false;     // no WHERE, nullable: the kernel writes the bitmap and counts the nulls
  unsigned char* bytes = nullptr;   // BOOL: the kernel's bytes
  unsigned char* vbytes = nullptr;  // case_nulls: the validity bytes
  bool utf8() const { return kind == UTF8_GATHER || kind == UTF8_VIEW; }
};

}  // namespace dfgpu
using namespace dfgpu;

// Host-only type check of one expression program (no ctx, no device): the same ProgramBuilder the
// operators use, over a schema-only stand-in for a batch.
extern "C" int dfgpu_check_program(const int32_t* col_dtypes, int ncols, const dfgpu_insn* prog, int prog_len, int32_t* out_dtype) {
  return guarded([&] {
    if (!col_dtypes || ncols < 0 || !prog || prog_len <= 0 || !out_dtype) fail(DFGPU_ERR_GENERAL, "dfgpu_check_program: null argument");
    const dfgpu_batch schema = schema_only(col_dtypes, ncols);
    ProgramBuilder pb(&schema);
    const int pi = pb.add(prog, prog_len, "expression");
    ProgramSet ps;  // Utf8 predicates are typed, not evaluated
    pb.finish(&ps);  // instruction / column-slot limits
    *out_dtype = pb.out_dtype(pi);
  });
}

extern "C" int dfgpu_filter_project(dfgpu_ctx* ctx, const dfgpu_batch* batch, const dfgpu_insn* pred, int pred_len,
                                    const dfgpu_insn* const* proj, const int* proj_len, int nproj, dfgpu_result** out) {
  return guarded([&] {
    if (!ctx || !batch || !out) fail(DFGPU_ERR_GENERAL, "dfgpu_filter_project: null argument");
    ctx->use();
    ProgramBuilder pb(batch);
    const int has_pred = pred_len > 0 ? 1 : 0;
    if (has_pred) add_predicate(pb, pred, pred_len);
    IdentityProjection ident;
    project_every_column(int(batch->cols.size()), [&](int i) { return batch->cols[size_t(i)].dtype; }, ident, proj, proj_len, nproj);

    // ---- plan: one record per output column ----
    std::vector<OutCol> outs((size_t)nproj);
    int nkern = 0;
    bool any_utf8 = false, any_bool = false, any_case_nulls = false;
    for (int i = 0; i < nproj; i++) {
      OutCol& o = outs[size_t(i)];
      const dfgpu_insn* q = proj[i];
      if (proj_len[i] == 1 && q[0].op == DFGPU_OP_COL && q[0].col >= 0 && size_t(q[0].col) < batch->cols.size() &&
          batch->cols[size_t(q[0].col)].dtype == DFGPU_UTF8) {
        o.kind = OutCol::UTF8_GATHER;
        o.src = q[0].col;
      } else {
        const int pi = pb.add(q, proj_len[i], "projection", &o.view);
        if (o.view >= 0) {
          o.kind = OutCol::UTF8_VIEW;
          o.src = pb.utf8_views()[size_t(o.view)].src;
        } else {
          const int dt = pb.out_dtype(pi);
          if (!is_numeric(dt) && dt != DFGPU_BOOL)
            fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("filter/projection output of type ") + dtype_name(dt) +
                                                " is not supported on the GPU path yet");
          o.kind = dt == DFGPU_BOOL ? OutCol::BOOL : OutCol::VALUE;
          o.slot = nkern++;
          o.case_nulls = has_pred && pb.prog(pi).makes_nulls;
        }
      }
      any_utf8 = any_utf8 || o.utf8();
      any_bool = any_bool || o.kind == OutCol::BOOL;
      any_case_nulls = any_case_nulls || o.case_nulls;
    }
    int rowid_slot = -1;  // the selected row numbers, which the Utf8 outputs are gathered by
    if (any_utf8) {
      pb.add_rowid();
      rowid_slot = nkern++;
    }
    pb.eval_utf8_predicates(ctx);
    // columns referenced anywhere must be null-free and fixed width for now
    FPParams p;
    pb.finish(&p.ps);
    for (int s = 0; s < p.ps.ncols; s++) {
      // Boolean input columns (bit-packed BooleanArray) are read by the direct kernel's interpreter
      if (!is_numeric(p.ps.cols[s].dtype) && p.ps.cols[s].dtype != DFGPU_BOOL)
        fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("expressions over ") + dtype_name(p.ps.cols[s].dtype) + " columns are not supported on the GPU path yet");
    }
    if (p.ps.max_depth > 8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "expression too deep (register stack depth > 8)");
    // without a WHERE over nullable inputs the kernel writes the validity of the nullable projections and counts their nulls
    const bool kernel_nulls = !has_pred && p.ps.has_nulls;
    for (OutCol& o : outs) {
      if (o.slot < 0) continue;
      o.kernel_validity = kernel_nulls && p.ps.nullable[o.slot + has_pred];
      // Boolean projections (comparisons / AND / OR, expression.rs:212-224,236-290) leave the kernel as bytes
      if (o.kind == OutCol::BOOL) p.ps.out_dtype[o.slot + has_pred] = DFGPU_UINT8;
    }

    // ---- allocate and launch ----
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    const long long n = batch->nrows;
    const size_t rows = size_t(n > 0 ? n : 1);
    for (const OutCol& o : outs) {
      DevColumn c;
      c.dtype = o.kind == OutCol::VALUE ? pb.out_dtype(o.slot + has_pred) : o.kind == OutCol::BOOL ? DFGPU_BOOL : DFGPU_UTF8;
      if (o.kind == OutCol::VALUE) c.values_bytes = rows * size_t(dtype_width(c.dtype));
      if (o.kind == OutCol::BOOL) c.values_bytes = size_t((n + 31) / 32) * 4 + 4;  // packed, whole 32-bit words
      if (!o.utf8()) c.values = ctx->alloc(c.values_bytes);
      res->cols.push_back(c);
    }
    if (n == 0) {
      for (size_t i = 0; i < outs.size(); i++) {
        DevColumn& c = res->cols[i];
        if (outs[i].kind == OutCol::BOOL) c.values_bytes = 0;
        if (outs[i].utf8()) {
          c.offsets = (int32_t*)ctx->alloc(4);
          DF_CUDA(cudaMemsetAsync(c.offsets, 0, 4, ctx->stream));
          c.values = ctx->alloc(1);
        }
      }
      DF_CUDA(cudaStreamSynchronize(ctx->stream));  // a result that is not stream-ordered is complete when the call returns
      res->nrows = 0;
      *out = res.release();
      return;
    }
    DevBufs tmp(ctx);  // the kernel's byte outputs, the row numbers and the tile status words
    p.nrows = n;
    p.has_pred = has_pred;
    p.nproj = nkern;
    memset(p.out_valid, 0, sizeof(p.out_valid));
    memset(p.out_vbytes, 0, sizeof(p.out_vbytes));
    static_assert(kMaxProgs <= SCR_FP_NULLS.words, "a null count per program");
    p.null_counts = ctx->d_scratch + SCR_FP_NULLS.at;
    if (kernel_nulls) DF_CUDA(cudaMemsetAsync(p.null_counts, 0, kMaxProgs * 8, ctx->stream));
    for (size_t i = 0; i < outs.size(); i++) {
      OutCol& o = outs[i];
      DevColumn& c = res->cols[i];
      if (o.slot < 0) continue;
      if (o.kind == OutCol::BOOL) o.bytes = tmp.alloc<unsigned char>(rows);
      p.out[o.slot] = o.kind == OutCol::BOOL ? o.bytes : c.values;
      if (o.case_nulls) {
        o.vbytes = tmp.alloc<unsigned char>(rows);
        p.out_vbytes[o.slot] = o.vbytes;
      }
      if (o.kernel_validity) {
        const size_t bitmap_bytes = size_t((n + 31) / 32) * 4;
        c.validity = (uint8_t*)ctx->alloc(bitmap_bytes);
        DF_CUDA(cudaMemsetAsync(c.validity, 0, bitmap_bytes, ctx->stream));
        p.out_valid[o.slot] = (unsigned*)c.validity;
      }
    }
    unsigned long long* row_numbers = nullptr;
    if (rowid_slot >= 0) {
      row_numbers = tmp.alloc(rows * 8);
      p.out[rowid_slot] = row_numbers;
    }
    // tile_status is sized for the smallest tile either kernel uses (1024 rows)
    const size_t max_tiles = size_t((n + 1023) / 1024) + 1;
    // one allocation, one memset: [ticket, pad..] then the tile words.  The row count and the error
    // flag are written by the kernel straight into pinned host memory (zero-copy), so no device-to-host
    // copy follows the kernel.
    unsigned long long* status = tmp.alloc((max_tiles + 8) * 8);
    DF_CUDA(cudaMemsetAsync(status, 0, (max_tiles + 8) * 8, ctx->stream));
    p.tile_status = status + 8;
    p.ticket = (unsigned*)(status + 0);
    // Stream-ordered: when nothing after the kernel needs the row count on the host (no Boolean packing, no Utf8
    // gather, no validity outputs) and no program can raise, the call returns once the kernel is queued.  The kernel
    // writes the count into a word pair the result owns, read when the result is first used (resolve, api.cu).
    const bool stream_ordered = has_pred && !p.ps.has_nulls && !any_utf8 && !any_bool && !has_div(p.ps);
    if (stream_ordered) {
      res->pending = ctx->fp_acquire(res.get());
      p.out_count = ctx->fp_slots[size_t(res->pending)].words;
      p.err_flag = (unsigned*)(p.out_count + 1);
    } else {
      p.out_count = ctx->h_scratch + SCR_FP_ROWS.at;
      p.err_flag = (unsigned*)(ctx->h_scratch + SCR_FP_DIV0.at);
      *p.out_count = 0;
      *p.err_flag = 0;
    }
    p.pred_fast = has_pred ? pb.prog(0).chain : LeafChain{};
    for (int i = 0; i < nkern; i++) p.proj_fast[i] = pb.prog(i + has_pred).leaf;
    const bool fn = has_fn(p.ps);
    if (p.ps.has_nulls) {
      p.ntiles = int((n + FP_TILE - 1) / FP_TILE);
      // the null-aware evaluator lives in the direct kernel only
      if (has_case(p.ps)) launch_fp<kCaseDepth, true>(ctx, p);
      else if (fn) launch_fp<kFnDepth, true>(ctx, p);
      else launch_fp<8, true>(ctx, p);
    } else if (ctx->force_direct_kernel || !launch_fp_tma(ctx, p)) {
      p.ntiles = int((n + FP_TILE - 1) / FP_TILE);
      const int d = p.ps.max_depth;
      if (has_case(p.ps)) launch_fp<kCaseDepth>(ctx, p);
      else if (fn) launch_fp<kFnDepth>(ctx, p);
      else if (d <= 1) launch_fp<1>(ctx, p);
      else if (d <= 2) launch_fp<2>(ctx, p);
      else if (d <= 4) launch_fp<4>(ctx, p);
      else launch_fp<8>(ctx, p);
    }
    if (stream_ordered) {
      DF_CUDA(cudaEventRecord(ctx->fp_slots[size_t(res->pending)].done, ctx->stream));
      if (getenv("DFGPU_TRACE")) fprintf(stderr, "[dfgpu trace] filter_project returns stream-ordered\n");
      *out = res.release();
      return;
    }

    // ---- settle ----
    if (kernel_nulls)
      DF_CUDA(cudaMemcpyAsync(ctx->h_scratch + SCR_FP_NULLS.at, p.null_counts, kMaxProgs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));  // the host reads the row count, the DivideByZero flag and the null counts
    for (size_t i = 0; i < outs.size(); i++)
      if (outs[i].kernel_validity) set_null_count(ctx, res->cols[i], (int64_t)ctx->h_scratch[SCR_FP_NULLS.at + outs[i].slot]);
    if (*p.err_flag != 0) fail(DFGPU_ERR_ARROW, "DivideByZero");
    res->nrows = has_pred ? (int64_t)*p.out_count : n;
    const long long words = (res->nrows + 31) / 32;
    if (any_case_nulls && words > 0) {
      DF_CUDA(cudaMemsetAsync(p.null_counts, 0, kMaxProgs * 8, ctx->stream));
      for (size_t i = 0; i < outs.size(); i++)
        if (outs[i].case_nulls) {
          res->cols[i].validity = (uint8_t*)ctx->alloc(size_t(words) * 4);
          pack_bits(ctx, outs[i].vbytes, res->nrows, (unsigned*)res->cols[i].validity, p.null_counts + outs[i].slot);
        }
      DF_CUDA(cudaMemcpyAsync(ctx->h_scratch + SCR_FP_NULLS.at, p.null_counts, kMaxProgs * 8, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));  // the host reads the packs' null counts
      for (size_t i = 0; i < outs.size(); i++)
        if (outs[i].case_nulls) set_null_count(ctx, res->cols[i], (int64_t)ctx->h_scratch[SCR_FP_NULLS.at + outs[i].slot]);
    }
    for (size_t i = 0; i < outs.size(); i++) {
      const OutCol& o = outs[i];
      DevColumn& c = res->cols[i];
      if (o.kind == OutCol::BOOL) {
        if (words > 0) pack_bits(ctx, o.bytes, res->nrows, (unsigned*)c.values, nullptr);
        c.values_bytes = size_t(res->nrows + 7) / 8;
      } else if (o.kind == OutCol::UTF8_VIEW) {  // without a WHERE every row, in order: no row numbers needed
        pb.eval_utf8_view_rows(ctx, o.view, has_pred ? row_numbers : nullptr, res->nrows, &c);
      } else if (o.kind == OutCol::UTF8_GATHER) {
        gather_utf8(ctx, batch->cols[size_t(o.src)], row_numbers, res->nrows, &c);
      }
      // without a WHERE a Utf8 column passed through keeps its validity (expression.rs:313), and so does a Utf8 function of one
      if (!has_pred && o.utf8() && batch->cols[size_t(o.src)].null_count > 0) {
        const DevColumn& srcc = batch->cols[size_t(o.src)];
        const size_t vb = size_t(n + 7) / 8;
        c.validity = (uint8_t*)ctx->alloc(vb);
        DF_CUDA(cudaMemcpyAsync(c.validity, srcc.validity, vb, cudaMemcpyDeviceToDevice, ctx->stream));
        c.null_count = srcc.null_count;
      }
    }
    // a result that is not stream-ordered is complete when the call returns: wait for the packs, gathers and copies queued
    // after the synchronisation above (its readers may use another stream, and the byte buffers go back to the pool)
    const bool queued_after_sync = any_bool || any_utf8;
    if (queued_after_sync) DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = res.release();
  });
}

// ---------------------------------------------------------------------------------------------
// Host -> host, chunk-pipelined (see include/dfgpu.h).  All H2D copies are queued up front on the
// copy-in stream; chunk c's kernel waits for its copies only; its compacted output is copied back
// on the copy-out stream while chunk c+1 is being filtered and chunk c+2 uploaded.
// ---------------------------------------------------------------------------------------------
extern "C" int dfgpu_filter_project_host(dfgpu_ctx* ctx, const dfgpu_col* cols, int ncols, const dfgpu_insn* pred, int pred_len,
                                         const dfgpu_insn* const* proj, const int* proj_len, int nproj, int64_t chunk_rows,
                                         dfgpu_result** out) {
  return guarded([&] {
    if (!ctx || !out || !cols || ncols < 1) fail(DFGPU_ERR_GENERAL, "dfgpu_filter_project_host: null argument");
    ctx->use();
    const long long n = cols[0].len;
    for (int i = 0; i < ncols; i++) {
      if (cols[i].len != n) fail(DFGPU_ERR_GENERAL, "all columns of a RecordBatch must have the same length");
    }
    IdentityProjection ident;
    project_every_column(ncols, [&](int i) { return cols[i].dtype; }, ident, proj, proj_len, nproj);
    // referenced columns only (the reference uploads nothing, but gathers every column: filter.rs:55-57)
    std::vector<int> remap(size_t(ncols), -1), used;
    auto scan = [&](const dfgpu_insn* p, int len) {
      for (int i = 0; i < len; i++)
        if (p[i].op == DFGPU_OP_COL) {
          if (p[i].col < 0 || p[i].col >= ncols) fail(DFGPU_ERR_INVALID_COLUMN, "column index " + std::to_string(p[i].col) + " out of range");
          if (remap[size_t(p[i].col)] < 0) {
            remap[size_t(p[i].col)] = int(used.size());
            used.push_back(p[i].col);
          }
        }
    };
    if (pred_len > 0) scan(pred, pred_len);
    for (int q = 0; q < nproj; q++) scan(proj[q], proj_len[q]);
    if (used.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "queries that reference no column");
    auto rewrite = [&](const dfgpu_insn* p, int len) {
      std::vector<dfgpu_insn> v(p, p + len);
      for (auto& in : v)
        if (in.op == DFGPU_OP_COL) in.col = remap[size_t(in.col)];
      return v;
    };
    std::vector<dfgpu_insn> pred2 = pred_len > 0 ? rewrite(pred, pred_len) : std::vector<dfgpu_insn>();
    std::vector<std::vector<dfgpu_insn>> proj2;
    std::vector<const dfgpu_insn*> proj2p;
    std::vector<int> proj2l;
    for (int q = 0; q < nproj; q++) {
      proj2.push_back(rewrite(proj[q], proj_len[q]));
    }
    for (auto& v : proj2) {
      proj2p.push_back(v.data());
      proj2l.push_back(int(v.size()));
    }
    // The chunks carry fixed-width values only, and the result columns are pinned host arrays of fixed-width values.
    // Everything else runs the resident operator on the whole batch (same kernels, same results; the result then lives
    // in DEVICE memory: dfgpu_result_on_host says which, dfgpu_result_copy_col works for both).  That is decided here,
    // before anything is uploaded: a referenced input that is not numeric or has a validity bitmap, a projection whose
    // result is not numeric (Boolean), or one with a CASE without ELSE (V_SEL0: the postfix program does not tell a
    // consumed null from a result one) takes the resident operator.
    std::vector<int32_t> used_dtypes;
    bool resident = false;
    for (int c : used) {
      resident = resident || !is_numeric(cols[c].dtype) || cols[c].validity;
      used_dtypes.push_back(cols[c].dtype);
    }
    std::vector<int> out_dtype;
    if (!resident) {  // typed by the front end of every chunk's call, on the same programs
      const dfgpu_batch schema = schema_only(used_dtypes.data(), int(used_dtypes.size()));
      ProgramBuilder pb(&schema);
      if (pred_len > 0) add_predicate(pb, pred2.data(), int(pred2.size()));
      for (int q = 0; q < nproj; q++) {
        const int pi = pb.add(proj2p[size_t(q)], proj2l[size_t(q)], "projection");
        out_dtype.push_back(pb.out_dtype(pi));
        resident = resident || !is_numeric(pb.out_dtype(pi));
        for (const DevInsn& di : pb.prog(pi).code) resident = resident || di.op == V_SEL0;
      }
    }
    if (resident) {
      std::vector<dfgpu_col> sub;
      for (int c : used) sub.push_back(cols[c]);
      dfgpu_batch* b = nullptr;
      int rc = dfgpu_batch_upload(ctx, sub.data(), int(sub.size()), &b);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      struct G { dfgpu_batch* b; ~G() { dfgpu_batch_free(b); } } g{b};
      rc = dfgpu_filter_project(ctx, b, pred2.data(), int(pred2.size()), proj2p.data(), proj2l.data(), nproj, out);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      return;
    }

    // default chunk: big enough that per-chunk launch and copy overheads stay small, small enough that the
    // first upload and the last download, which nothing overlaps, stay short (profiles/e2e_chunks.py sweeps it)
    if (chunk_rows <= 0) chunk_rows = 4ll << 20;
    const long long nchunks = n > 0 ? (n + chunk_rows - 1) / chunk_rows : 1;
    struct Chunk {
      dfgpu_batch batch;
      dfgpu_result* res = nullptr;
      cudaEvent_t ev = nullptr;
    };
    std::vector<std::unique_ptr<Chunk>> chunks;
    struct Cleanup {
      std::vector<std::unique_ptr<Chunk>>* c;
      dfgpu_ctx* ctx;
      ~Cleanup() {
        cudaStreamSynchronize(ctx->stream_in);
        cudaStreamSynchronize(ctx->stream_out);
        for (auto& ch : *c) {
          if (ch->res) delete ch->res;
          if (ch->ev) cudaEventDestroy(ch->ev);
        }
      }
    } cleanup{&chunks, ctx};
    // make the allocations (ordered on ctx->stream) visible to the copy-in stream
    cudaEvent_t ev_alloc;
    DF_CUDA(cudaEventCreateWithFlags(&ev_alloc, cudaEventDisableTiming));
    for (long long c = 0; c < nchunks; c++) {
      auto ch = std::make_unique<Chunk>();
      ch->batch.ctx = ctx;
      const long long r0 = c * (long long)chunk_rows, rows = std::min<long long>((long long)chunk_rows, n - r0);
      ch->batch.nrows = rows > 0 ? rows : 0;
      for (int u : used) {
        DevColumn d;
        d.dtype = cols[u].dtype;
        d.values_bytes = size_t(ch->batch.nrows) * size_t(dtype_width(d.dtype));
        d.values = ctx->alloc(d.values_bytes);
        ch->batch.cols.push_back(d);
      }
      DF_CUDA(cudaEventCreateWithFlags(&ch->ev, cudaEventDisableTiming));
      chunks.push_back(std::move(ch));
    }
    DF_CUDA(cudaEventRecord(ev_alloc, ctx->stream));
    DF_CUDA(cudaStreamWaitEvent(ctx->stream_in, ev_alloc, 0));
    cudaEventDestroy(ev_alloc);
    for (long long c = 0; c < nchunks; c++) {
      Chunk& ch = *chunks[size_t(c)];
      const long long r0 = c * chunk_rows;
      for (size_t k = 0; k < used.size(); k++) {
        const dfgpu_col& hc = cols[used[k]];
        const int w = dtype_width(hc.dtype);
        if (ch.batch.nrows > 0)
          DF_CUDA(cudaMemcpyAsync(ch.batch.cols[k].values, static_cast<const uint8_t*>(hc.values) + size_t(hc.offset + r0) * size_t(w),
                                  size_t(ch.batch.nrows) * size_t(w), cudaMemcpyHostToDevice, ctx->stream_in));
      }
      DF_CUDA(cudaEventRecord(ch.ev, ctx->stream_in));
    }
    // filter chunk by chunk; outputs go back as soon as their size is known
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    res->on_host = true;
    for (int dt : out_dtype) {
      DevColumn hcol;
      hcol.dtype = dt;
      hcol.values_bytes = size_t(n > 0 ? n : 1) * size_t(dtype_width(dt));
      hcol.values = ctx->host_alloc(hcol.values_bytes);
      res->cols.push_back(hcol);
    }
    long long off = 0;
    for (long long c = 0; c < nchunks; c++) {
      Chunk& ch = *chunks[size_t(c)];
      DF_CUDA(cudaStreamWaitEvent(ctx->stream, ch.ev, 0));
      int rc = dfgpu_filter_project(ctx, &ch.batch, pred2.data(), int(pred2.size()), proj2p.data(), proj2l.data(), nproj, &ch.res);
      if (rc != 0) fail(rc, dfgpu_last_error());
      // waits for the kernel of this chunk: its row count sizes the copies, and stream_out reads what it wrote
      resolve(ch.res);
      for (int q = 0; q < nproj; q++) {
        const int w = dtype_width(res->cols[size_t(q)].dtype);
        if (ch.res->nrows > 0)
          DF_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(res->cols[size_t(q)].values) + size_t(off) * size_t(w), ch.res->cols[size_t(q)].values,
                                  size_t(ch.res->nrows) * size_t(w), cudaMemcpyDeviceToHost, ctx->stream_out));
      }
      off += ch.res->nrows;
    }
    DF_CUDA(cudaStreamSynchronize(ctx->stream_out));
    res->nrows = off;
    *out = res.release();
  });
}
