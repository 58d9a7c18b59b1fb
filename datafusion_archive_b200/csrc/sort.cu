// sort.cu — dfgpu_sort: keep the rows where a Boolean program is true, order them stably by a list of key programs and
// gather the first `limit` of them.  The reference plans Sort and Limit (LogicalPlan::Sort / Limit) but leaves both
// unimplemented!() in ExecutionContext::execute (context.rs:113,194); include/dfgpu.h documents the semantics.
//
// The order is a permutation of u32 row ids, built by a stable LSD radix sort with 8-bit digits, one key at a time from
// the last key to the first:
//   k_sort_keep     the keep column's pass bits (value AND validity) as mask words and tile counts (mark_tiles); the
//                   counts are scanned and k_join_select (select_rows, gather.cuh) writes the kept row ids in row order
//   k_sort_iota     without a keep program: the row ids 0..n-1
//   k_sort_encode   per position i, key(perm[i]) as an order-preserving unsigned word of the key's own width (1, 2, 4
//                   or 8 bytes), complemented for DESC, and the OR and AND of all of them: a digit whose bits agree in
//                   both is the same in every row, and its pass is skipped
//   per live digit  k_sort_count (per-tile digit counts in shared memory, stored digit-major), scan_exclusive over the
//                   (digit, tile) counts, and k_sort_scatter: each tile places its (key, row id) pairs at its digit
//                   offsets in tile order, warp by warp and lane by lane, so every pass is stable
// A nullable key takes one more 1-byte pass on its null bit after its value passes (a null's value is encoded as 0, so
// nulls tie with each other).  A Utf8 key is first replaced by a dense u32 rank (utf8_rank), which then sorts as a 4-byte
// key.  Once the permutation is final, gather_column (gather.cuh) copies the first min(limit, kept) rows of every column.
#include <algorithm>
#include <memory>

#include "gather.cuh"
#include "sort.cuh"

namespace dfgpu {

__global__ void __launch_bounds__(SEL_THREADS) k_sort_keep(const unsigned char* __restrict__ vals, const unsigned char* __restrict__ valid, long long n,
                                                          unsigned* __restrict__ mask, unsigned* __restrict__ tile_cnt) {
  mark_tiles(n, mask, tile_cnt, [&](long long r) { return bit_at(vals, (unsigned)r) && (!valid || bit_at(valid, (unsigned)r)); });
}

}  // namespace dfgpu

using namespace dfgpu;

extern "C" int dfgpu_sort(dfgpu_ctx* ctx, const dfgpu_batch* in, const dfgpu_insn* keep, int keep_len, const dfgpu_insn* const* keys, const int* key_len,
                          const int32_t* desc, int nkeys, int64_t limit, dfgpu_result** out) {
  return guarded([&] {
    if (!ctx || !in || !out || keep_len < 0 || nkeys < 0 || (keep_len > 0 && !keep) || (nkeys > 0 && (!keys || !key_len)))
      fail(DFGPU_ERR_GENERAL, "dfgpu_sort: null argument");
    ctx->use();
    const long long n = in->nrows;
    if (n >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "ORDER BY input of 2^32 rows or more");
    std::vector<int32_t> col_dtypes;
    for (const DevColumn& c : in->cols) col_dtypes.push_back(c.dtype);
    // a program's column: a plain column in place, anything else evaluated as a projection
    std::vector<std::unique_ptr<dfgpu_result, int (*)(dfgpu_result*)>> evaluated;
    auto column = [&](const dfgpu_insn* p, int len, int32_t* dt) -> const DevColumn* {
      const int rc = dfgpu_check_program(col_dtypes.empty() ? nullptr : col_dtypes.data(), int(col_dtypes.size()), p, len, dt);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      if (len == 1 && p[0].op == DFGPU_OP_COL) return &in->cols[size_t(p[0].col)];
      dfgpu_result* r = nullptr;
      const int rc2 = dfgpu_filter_project(ctx, in, nullptr, 0, &p, &len, 1, &r);
      if (rc2 != DFGPU_OK) fail(rc2, dfgpu_last_error());
      evaluated.emplace_back(r, dfgpu_result_free);
      resolve(r);
      return &r->cols[0];
    };
    const DevColumn* keep_col = nullptr;
    if (keep_len > 0) {
      int32_t dt = 0;
      keep_col = column(keep, keep_len, &dt);
      if (dt != DFGPU_BOOL) fail(DFGPU_ERR_EXECUTION, std::string("dfgpu_sort: the keep program is ") + dtype_name(dt) + ", not Boolean");
    }
    std::vector<const DevColumn*> key_cols;
    for (int i = 0; i < nkeys; i++) {
      int32_t dt = 0;
      key_cols.push_back(column(keys[i], key_len[i], &dt));
      if (dt == DFGPU_BOOL) fail(DFGPU_ERR_NOT_IMPLEMENTED, "ORDER BY a Boolean key is not supported");
    }
    DevBufs scratch(ctx);
    long long m = n;
    Sorter S = make_sorter(ctx, n, scratch);
    S.cur = 0;
    if (keep_col && n > 0) {
      const long long ntiles = (n + MARK_TILE - 1) / MARK_TILE;
      unsigned* mask = scratch.alloc<unsigned>(size_t(ntiles) * MARK_WORDS * sizeof(unsigned));
      unsigned* tile_cnt = scratch.alloc<unsigned>(size_t(ntiles) * sizeof(unsigned));
      unsigned long long* tile_off = scratch.alloc<unsigned long long>(size_t(ntiles + 1) * sizeof(unsigned long long));
      const int grid = grid_for(ctx, n, MARK_TILE, 8);
      launch(ctx, "k_sort_keep", k_sort_keep, grid, SEL_THREADS, PROFILED, (const unsigned char*)keep_col->values,
             (const unsigned char*)(keep_col->null_count > 0 ? keep_col->validity : nullptr), n, mask, tile_cnt);
      m = (long long)scan_exclusive<unsigned, unsigned long long>(ctx, tile_cnt, tile_off, ntiles, true);
      if (m > 0) select_rows(ctx, grid, mask, ntiles, tile_off, S.perm[0]);
    } else if (n > 0) {
      launch(ctx, "k_sort_iota", k_sort_iota, grid_for(ctx, n, SORT_THREADS, 16), SORT_THREADS, PROFILED, n, S.perm[0]);
    }
    S.m = m;
    S.ntiles = (m + SORT_TILE - 1) / SORT_TILE;
    if (m > 1) {
      for (int i = nkeys - 1; i >= 0; i--) {
        const DevColumn& c = *key_cols[size_t(i)];
        const int d = desc && desc[i] ? 1 : 0;
        const unsigned char* valid = c.null_count > 0 ? c.validity : nullptr;
        if (c.dtype == DFGPU_UTF8) {
          unsigned* rank = scratch.alloc<unsigned>(size_t(n) * 4);
          utf8_rank(S, c, valid, n, scratch, rank);
          S.by<unsigned>(KeySrc{KS_RANK, DFGPU_UINT32, d, 0, rank, valid, nullptr, nullptr});
        } else {
          S.by_width(dtype_width(c.dtype), KeySrc{KS_FIXED, c.dtype, d, 0, c.values, valid, nullptr, nullptr});
        }
        if (valid) S.by<unsigned char>(KeySrc{KS_NULL, 0, d, 0, nullptr, valid, nullptr, nullptr});
      }
    }
    const long long mo = limit < 0 ? m : std::min<long long>(limit, m);
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    res->nrows = mo;
    unsigned long long* d_nulls = scratch.alloc<unsigned long long>(sizeof(unsigned long long));
    unsigned long long* idx64 = nullptr;
    for (const DevColumn& c : in->cols) {
      res->cols.emplace_back();
      gather_column(ctx, c, S.perm[S.cur], mo, scratch, idx64, d_nulls, &res->cols.back());
    }
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = res.release();
  });
}

extern "C" int dfgpu_result_as_batch(const dfgpu_result* r, dfgpu_batch** out) {
  return guarded([&] {
    if (!r || !out) fail(DFGPU_ERR_GENERAL, "dfgpu_result_as_batch: null argument");
    if (r->on_host) fail(DFGPU_ERR_GENERAL, "result lives in host memory: upload it with dfgpu_batch_upload");
    resolve(r);
    auto b = std::make_unique<dfgpu_batch>();
    b->ctx = r->ctx;
    b->nrows = r->nrows;
    b->cols = r->cols;
    b->owns = false;
    *out = b.release();
  });
}
