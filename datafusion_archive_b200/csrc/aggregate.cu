// aggregate.cu — AggregateRelation on the GPU (K4 column reduce, K5 hash-aggregate, K7 table
// compaction, K6 partial-aggregate merge of SURVEY.md §2b).
//
// Reference path replaced: `with_group_by` (src/execution/aggregate.rs:787-952) — per row a
// heap-allocated Vec<GroupByScalar> key, an FNV hash-map lookup, and a boxed ScalarValue folded
// through Rc<RefCell<dyn AggregateFunction>> (aggregate.rs:548-612, 102-283) — and
// `without_group_by` (aggregate.rs:703-785).  Here the map is an open-addressed table in HBM
// (linear probing, 64-bit packed keys claimed with atomicCAS) whose accumulators are updated with
// fire-and-forget L2 reductions: RED.ADD.F64 for f64 SUM, RED.ADD.U64 for COUNT / integer SUM,
// RED.MIN/MAX.U64 on an order-preserving encoding for MIN/MAX (bit-exact for every type).
#include <deque>
#include <memory>

#include "expr_vm.cuh"
#include "hash_table.cuh"

namespace dfgpu {

void utf8_hash(dfgpu_ctx* ctx, const DevColumn& src, long long n, unsigned long long* d_out);
void shift_copy_i32(dfgpu_ctx* ctx, int* dst, const int* src, long long n, int add);
void gather_utf8_multi(dfgpu_ctx* ctx, const Utf8Source* d_srcs, const unsigned long long* d_idx, long long nsel, DevColumn* out);

constexpr int AG_THREADS = 256;
constexpr int AG_R = 2;  // rows per thread per tile: the kernel is bound by scattered L2 reductions, not by loads in flight, so more rows per thread only add registers
constexpr int AG_TILE = AG_THREADS * AG_R;
constexpr int kMaxAggs = 8;
constexpr int kMaxKeys = 4;
constexpr int AG_MAX_PROBE = 1 << 14;
constexpr long long AG_MIN_CAP = 1ll << 22;
constexpr long long AG_SET_MIN_CAP = 1ll << 20;  // COUNT(DISTINCT) pair sets: 16-byte slots
constexpr long long AG_PREFIX_ROWS = 1ll << 20;  // prefix sample that sizes the tables of a first big batch

// Internal function code (not part of the C ABI) of the sum word of an AVG: every AVG(x) is two table words, this one
// and a COUNT of the same argument.  Only the per-row fold sees the argument's type: it widens the value to f64 and
// adds it, and it skips nulls also under GROUP BY.  Everything else -- merges, growth, the exchanges, compaction and
// decoding -- treats the word as an f64 SUM.
constexpr int AGG_AVG_SUM = 16;

struct AggDesc {
  uint8_t func;   // DFGPU_AGG_*
  uint8_t mtype;  // machine type of the argument
  uint8_t dtype;  // Arrow dtype of the argument
  uint8_t out_dtype;
};

// Table addressing.  A slot is a LINE of lw 64-bit words (lw a power of two; word 0 = the packed key) plus
// one word in each of n_add separate arrays.  loc[a] says where accumulator a lives: >= 1 = that word of
// the line, < 0 = additive array ~loc[a].  Three layouts fall out of it:
//   SoA     lw = 1, every accumulator in its own array.  A row's probe and reductions go to different L2
//           slices in parallel; reductions that hit the SAME 32-byte sector as the probe serialise in the
//           slice.
//   hybrid  MIN / MAX accumulators share the line with the key, SUM / COUNT stay in arrays.  The probe is
//           one or two 128-bit loads that also return the current MIN / MAX, and a MIN / MAX reduction is only
//           issued when the row improves on the value just read (monotone accumulators: a stale read can
//           only cause a redundant reduction, never a missed one).  After a group's first few rows almost
//           no row does, so MIN + MAX + SUM costs one load and one reduction per row instead of one load
//           and three reductions.
//   line    every accumulator in the line (lw >= 1 + naggs): one sector per group; wins once the table no
//           longer fits L2 and every touched sector is an HBM transaction.
// cap + 1 slots: slot cap is reserved for the key that equals EMPTY_KEY.  The table without GROUP BY has cap = 0.
struct TableLayout : ProbeRule {
  unsigned long long* base;  // (cap + 1) lines of lw words
  unsigned long long* add;   // n_add arrays of (cap + 1) words
  long long lw, astride;
  signed char loc[kMaxAggs];
  __host__ __device__ __forceinline__ unsigned long long* key(long long slot) const { return base + slot * lw; }
  __host__ __device__ __forceinline__ unsigned long long* val(long long slot, int a) const {
    const int l = loc[a];
    return l >= 0 ? base + slot * lw + l : add + (long long)(~l) * astride + slot;
  }
  // The slot of key k, which is in the table unless the table is inconsistent: cap for EMPTY_KEY when the sentinel slot
  // is in use, -1 when the key is missing.  At most cap probes.
  __device__ __forceinline__ long long find(unsigned long long k, bool sentinel_used) const {
    if (k == EMPTY_KEY) return sentinel_used ? cap : -1;
    unsigned long long h = home(mix64(k));
    for (long long probes = 0; probes < cap; probes++) {
      const unsigned long long cur = __ldcg(key((long long)h));
      if (cur == k) return (long long)h;
      if (cur == EMPTY_KEY) return -1;
      h = next(h);
    }
    return -1;
  }
};

// A COUNT(DISTINCT) pair set: cap slots of two words.
struct SetView : ProbeRule {
  unsigned long long* slots;
};

// plain-column fast path (k_hash_agg_plain): every key and aggregate argument is a plain column of the (at most 4)
// column slots and the WHERE clause, if any, is a chain of column comparisons: no interpreter in the kernel
struct PlainSpec {
  int key_slot[kMaxKeys];
  int arg_slot[kMaxAggs];  // per distinct argument program
  LeafChain pred;          // the WHERE clause (nterms = 0: none)
};

// Slots of the operator's device counters (AggParams::counters, dfgpu_aggstate::d_counters).
constexpr int CTR_GROUPS = 0;    // groups in the table
constexpr int CTR_OVERFLOW = 1;  // rows appended to the overflow list
constexpr int CTR_SENTINEL = 2;  // nonzero: the key that equals EMPTY_KEY holds slot cap
constexpr int CTR_ERROR = 3;     // 1: an expression raised DivideByZero, 2: a merge into the table found no slot
constexpr int CTR_COMPACT = 4;   // entries written by k_compact
constexpr int CTR_DEFERRED = 5;  // wide scan: overflow rows that only met a slot still being published; Utf8 verify: its flag
constexpr int CTR_PASSED = 6;    // reduce with WHERE: rows that passed the predicate
constexpr int CTR_ROWS = 7;      // multi-GPU reduce: rows seen on every rank
constexpr int CTR_NONNULL = 8;   // [8, 8 + kMaxAggs): reduce: non-null inputs per aggregate
constexpr int CTR_SLOTS = CTR_NONNULL + kMaxAggs;

struct AggParams {
  ProgramSet ps;  // programs [0,nkeys) = group keys, then the distinct aggregate-argument programs
  AggDesc aggs[kMaxAggs];
  // aggregates over the same argument expression (MIN(v), MAX(v), SUM(v)) share one evaluation:
  // programs [nkeys, nkeys + nargs) are the DISTINCT argument programs, agg_arg[a] picks one
  int agg_arg[kMaxAggs];
  int nargs;
  unsigned long long key_mask[kMaxKeys];
  int key_shift[kMaxKeys];
  int nkeys, naggs;
  long long nrows;
  long long row_begin;       // process rows [row_begin, row_begin + nrows) of the batch
  const unsigned* row_list;  // non-null: process rows row_list[0..nlist) (overflow replay)
  long long nlist;
  TableLayout t;
  long long max_groups;      // new keys are refused (-> overflow list) beyond this fill
  unsigned long long* counters;  // CTR_SLOTS words, see CTR_*
  unsigned* ovf_rows;
  // front table (FRONT kernels): one table of front_slots per CTA, or — for very few groups — one
  // private table per warp, so that shared-memory atomics only contend inside a warp
  int front_slots;     // power of two
  int front_per_warp;  // 0 / 1
  // fused WHERE (Aggregate{input: Selection}, context.rs:126-139,162-192): program 0 is the predicate and
  // the key / argument programs follow; rows that fail it are skipped before the probe
  int has_pred;
  // wide keys (k_hash_agg_wide): composite keys of more than 64 bits and keys with Utf8 parts.  Line word 0 is a
  // TAG (the 64-bit hash of the key tuple, low bit = ready), words 1..kw the key parts: the 64-bit value of a
  // fixed-width part, or for a Utf8 part a reference (source << 40 | row) to the string of the row that created
  // the group.  Equal tags are confirmed by comparing every part (strings byte by byte), so hash collisions
  // just probe on — the reference's Vec<GroupByScalar> equality (aggregate.rs:65-76, 807-852).
  struct {
    int kw;
    int is_utf8[kMaxKeys];
    const int* off[kMaxKeys];            // this batch's Utf8 key columns
    const unsigned char* bytes[kMaxKeys];
    unsigned long long ref_base[kMaxKeys];  // (source index of this batch's column) << UTF8_SRC_SHIFT
    const Utf8Source* srcs;              // every retained Utf8 key column
  } wide;
  // lean kernel (k_hash_agg_lean): one 8-byte key column, one 8-byte argument column, no predicate
  struct {
    const unsigned long long* key_col;
    const unsigned long long* arg_col;
    unsigned long long* sum_arr;  // additive arrays of SUM / COUNT
    unsigned long long* cnt_arr;
    int min_w, max_w;             // words of MIN / MAX in the line
  } lean;
  PlainSpec plain;
};

// ---- order-preserving encodings so that MIN/MAX are native u64 atomics -----------------------
__device__ __forceinline__ unsigned long long ord_enc(unsigned long long v, int mt) {
  switch (mt) {
    case MT_F64: return (v >> 63) ? ~v : (v ^ 0x8000000000000000ull);
    case MT_F32: { unsigned b = (unsigned)v; return (b >> 31) ? (unsigned long long)(~b) : (unsigned long long)(b ^ 0x80000000u); }
    case MT_I: return v ^ 0x8000000000000000ull;
    default: return v;
  }
}
__host__ __device__ __forceinline__ unsigned long long ord_dec(unsigned long long e, int mt) {
  switch (mt) {
    case MT_F64: return (e >> 63) ? (e ^ 0x8000000000000000ull) : ~e;
    case MT_F32: { unsigned b = (unsigned)e; return (b >> 31) ? (unsigned long long)(b ^ 0x80000000u) : (unsigned long long)(~b); }
    case MT_I: return e ^ 0x8000000000000000ull;
    default: return e;
  }
}
__device__ __forceinline__ bool is_nan_val(unsigned long long v, int mt) {
  if (mt == MT_F64) { double d = u2d(v); return d != d; }
  if (mt == MT_F32) { float f = u2f(v); return f != f; }
  return false;
}
__host__ __device__ __forceinline__ unsigned long long agg_identity(int func) {
  return func == DFGPU_AGG_MIN ? ~0ull : 0ull;
}

// an argument value in the widened 64-bit machine representation, as f64 (AVG): exact for Float32, rounded to nearest
// for integers beyond 2^53
__device__ __forceinline__ double widen_f64(unsigned long long v, int mt) {
  switch (mt) {
    case MT_F64: return u2d(v);
    case MT_F32: return (double)u2f(v);
    case MT_I: return (double)(long long)v;
    default: return (double)v;
  }
}

// fold one value into an accumulator held in a register / shared memory
__device__ __forceinline__ unsigned long long acc_fold(int func, int mt, unsigned long long acc, unsigned long long v) {
  switch (func) {
    case DFGPU_AGG_SUM:
      if (mt == MT_F64) return d2u(u2d(acc) + u2d(v));
      if (mt == MT_F32) return f2u(u2f(acc) + u2f(v));
      return acc + v;
    case AGG_AVG_SUM: return d2u(u2d(acc) + widen_f64(v, mt));
    case DFGPU_AGG_COUNT: return acc + 1ull;
    case DFGPU_AGG_MIN: {
      if (is_nan_val(v, mt)) return acc;  // f64::min ignores NaN (aggregate.rs:139-140)
      unsigned long long e = ord_enc(v, mt);
      return e < acc ? e : acc;
    }
    default: {
      if (is_nan_val(v, mt)) return acc;
      unsigned long long e = ord_enc(v, mt);
      return e > acc ? e : acc;
    }
  }
}
// combine two accumulators
__device__ __forceinline__ unsigned long long acc_merge(int func, int mt, unsigned long long a, unsigned long long b) {
  switch (func) {
    case DFGPU_AGG_SUM:
      if (mt == MT_F64) return d2u(u2d(a) + u2d(b));
      if (mt == MT_F32) return f2u(u2f(a) + u2f(b));
      return a + b;
    case AGG_AVG_SUM: return d2u(u2d(a) + u2d(b));
    case DFGPU_AGG_COUNT: return a + b;
    case DFGPU_AGG_MIN: return a < b ? a : b;
    default: return a > b ? a : b;
  }
}
// combine an accumulator into global memory (fire-and-forget reductions)
__device__ __forceinline__ void acc_merge_global(int func, int mt, unsigned long long* p, unsigned long long b) {
  switch (func) {
    case DFGPU_AGG_SUM:
      if (mt == MT_F64) atomicAdd((double*)p, u2d(b));
      else if (mt == MT_F32) atomicAdd((float*)p, u2f(b));
      else atomicAdd(p, b);
      break;
    case AGG_AVG_SUM: atomicAdd((double*)p, u2d(b)); break;
    case DFGPU_AGG_COUNT: atomicAdd(p, b); break;
    case DFGPU_AGG_MIN: atomicMin(p, b); break;
    default: atomicMax(p, b); break;
  }
}
// fold one raw value into global or shared memory
__device__ __forceinline__ void acc_fold_global(int func, int mt, unsigned long long* p, unsigned long long v) {
  switch (func) {
    case DFGPU_AGG_SUM:
      if (mt == MT_F64) atomicAdd((double*)p, u2d(v));
      else if (mt == MT_F32) atomicAdd((float*)p, u2f(v));
      else atomicAdd(p, v);
      break;
    case DFGPU_AGG_COUNT: atomicAdd(p, 1ull); break;
    case DFGPU_AGG_MIN:
      if (!is_nan_val(v, mt)) atomicMin(p, ord_enc(v, mt));
      break;
    default:
      if (!is_nan_val(v, mt)) atomicMax(p, ord_enc(v, mt));
      break;
  }
}

// One table line as read by a probe: word 0 = key, words 1..3 = the accumulators that share the line.
struct Line {
  unsigned long long w[4];
};
// A 4-word line as two 128-bit loads (sm_90 has no 256-bit global load); both land in the same 32-byte
// sector.  The halves are not read atomically together, which the protocol tolerates: a key seen in word 0
// is final, and the accumulators are monotone, so an older or newer word 1..3 can only cause a redundant
// MIN / MAX reduction, never a missed one.
__device__ __forceinline__ void load_line4(const unsigned long long* q, Line& ln) {
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(ln.w[0]), "=l"(ln.w[1]) : "l"(q) : "memory");
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(ln.w[2]), "=l"(ln.w[3]) : "l"(q + 2) : "memory");
}
// What a probe loads at a slot: LW > 0 = the first words of lines LW words apart, LW known at compile time (the lean
// scan, whose words past the line are never read); LINE_RT = up to 4 words of the table's lw-word lines (the generic
// scan: the probe also returns the in-line MIN / MAX); LINE_KEY = the key word alone (merges).
constexpr int LINE_RT = 0, LINE_KEY = -1;
template <int LW>
__device__ __forceinline__ unsigned long long* line_at(const TableLayout& t, unsigned long long slot) {
  return LW > 0 ? t.base + slot * LW : t.key((long long)slot);
}
template <int LW>
__device__ __forceinline__ void load_line(const TableLayout& t, unsigned long long slot, Line& ln) {
  const unsigned long long* q = line_at<LW>(t, slot);
  const long long w = LW > 0 ? LW : (LW == LINE_RT ? t.lw : 1);
  if (w >= 4) {  // lines are 32-byte aligned
    load_line4(q, ln);
  } else if (w == 2) {
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(ln.w[0]), "=l"(ln.w[1]) : "l"(q) : "memory");
    if (LW <= 0) ln.w[2] = ln.w[3] = 0ull;
  } else {
    asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(ln.w[0]) : "l"(q) : "memory");
    if (LW <= 0) ln.w[1] = ln.w[2] = ln.w[3] = 0ull;
  }
}
__device__ __forceinline__ unsigned long long line_word(const Line& ln, int l) {
  return l == 1 ? ln.w[1] : (l == 2 ? ln.w[2] : ln.w[3]);
}

// Find the slot of `key`, claiming an empty one when the key is new.  `h` is the home slot on entry and the key's slot
// on exit; `ln` is the line read at h on entry and the line of the key's slot on exit (as it was when this thread read
// it: a slot claimed meanwhile still shows its initial accumulator identities, which is what the conditional
// MIN / MAX update needs).  Returns false when the key is new and the table refuses new keys (fill limit /
// probe limit): the row goes to the overflow list.
template <int LW>
__device__ __forceinline__ bool probe_insert(const TableLayout& t, unsigned long long key, Line& ln, unsigned long long& h, bool full,
                                             unsigned& new_groups) {
  for (int probes = 0; probes < AG_MAX_PROBE; ++probes) {
    if (ln.w[0] == key) return true;
    if (ln.w[0] == EMPTY_KEY) {
      if (full) return false;
      const unsigned long long old = atomicCAS(line_at<LW>(t, h), EMPTY_KEY, key);
      if (old == EMPTY_KEY) { new_groups++; return true; }
      if (old == key) return true;
    }
    h = t.next(h);
    load_line<LW>(t, h, ln);
  }
  return false;
}

// fold one raw value into global memory; `cur` = the accumulator as read with the probe (have_cur): a
// MIN / MAX that the row does not improve needs no reduction (the stored value only moves towards it)
__device__ __forceinline__ void acc_fold_global_cond(int func, int mt, unsigned long long* p, unsigned long long v, bool have_cur,
                                                     unsigned long long cur) {
  if (func == DFGPU_AGG_MIN) {
    if (is_nan_val(v, mt)) return;
    const unsigned long long e = ord_enc(v, mt);
    if (!have_cur || e < cur) atomicMin(p, e);
  } else if (func == DFGPU_AGG_MAX) {
    if (is_nan_val(v, mt)) return;
    const unsigned long long e = ord_enc(v, mt);
    if (!have_cur || e > cur) atomicMax(p, e);
  } else {
    acc_fold_global(func, mt, p, v);
  }
}

constexpr int AG_FRONT_SLOTS = 2048;   // per-CTA shared-memory front table (low-cardinality GROUP BY)
constexpr int AG_FRONT_PROBES = 8;
constexpr int AG_FRONT_MAX_GROUPS = 1024;

// ---- row sources of the scan kernel -----------------------------------------------------------------
// InterpSrc: keys, arguments and the WHERE predicate are expression programs run by the interpreter of
// expr_vm.cuh, AG_R rows per thread.
// NULLS: like the reference, keys and MIN/MAX/SUM arguments are read ignoring the validity bitmap
// (`array.value(row)`, aggregate.rs:561-601, 807-852; a null produced by arithmetic reads as the
// builder's default 0); only COUNT and AVG (extensions, §DESIGN) honour nulls.  A predicate that evaluates to
// null reads as its value false (filter.rs:86 `filter.value(i)`).  Under a WHERE the reference aggregates
// FilterRelation's output, whose arrays carry no bitmap (filter.rs:83-91): keys and arguments are then
// evaluated as over null-free arrays (the rule of filter_project.cu), so every surviving row counts.
template <int DEPTH, int R, bool NULLS, class Rows>
__device__ __forceinline__ unsigned eval_after_where(const AggParams& p, int prog, const Rows& g,
                                                     unsigned long long (&v)[R], unsigned& valid) {
  if (NULLS && !p.has_pred) return eval_program_n<DEPTH, R, false, true>(p.ps, prog, g, v, valid);
  return eval_program_n<DEPTH, R, false, false>(p.ps, prog, g, v, valid);
}

template <int DEPTH, bool NULLS>
struct InterpSrc {
  static constexpr int R = AG_R;
  GlobalRows<R> g;
  unsigned mask;  // rows to aggregate: in range and passing the predicate
  unsigned bad = 0;
  __device__ __forceinline__ void load(const AggParams& p, long long tb, long long n, int tid, unsigned long long policy) {
    g.valid = 0;
    g.l2_policy = policy;
#pragma unroll
    for (int r = 0; r < R; r++) {
      const long long i = tb + (long long)r * AG_THREADS + tid;
      g.rows[r] = i < n ? (p.row_list ? (long long)p.row_list[i] : p.row_begin + i) : -1;
      if (i < n) g.valid |= 1u << r;
    }
    mask = g.valid;
    bad = 0;
  }
  __device__ __forceinline__ void prepare(const AggParams& p) {
    if (p.has_pred) {
      unsigned long long v[R];
      unsigned pv;
      bad |= eval_program_n<DEPTH, R, false, NULLS>(p.ps, 0, g, v, pv);  // FilterRelation evaluates the predicate on every row
      unsigned keep = 0;
#pragma unroll
      for (int r = 0; r < R; r++) keep |= (unsigned)(v[r] & 1ull) << r;
      mask &= keep;
    }
  }
  __device__ __forceinline__ void key(const AggParams& p, int k, unsigned long long (&v)[R]) {
    unsigned kv;
    bad |= eval_after_where<DEPTH, R, NULLS>(p, p.has_pred + k, g, v, kv) & mask;
  }
  // returns the DivideByZero bits of the rows; av = validity bits of the argument values
  __device__ __forceinline__ unsigned arg(const AggParams& p, int gi, unsigned long long (&v)[R], unsigned& av) {
    return eval_after_where<DEPTH, R, NULLS>(p, p.has_pred + p.nkeys + gi, g, v, av);
  }
  __device__ __forceinline__ unsigned rowid(int r) const { return (unsigned)g.rows[r]; }
};

// PlainSrc: every key / argument is a plain 4- or 8-byte column and the predicate a chain of column
// comparisons.  A thread owns two CONSECUTIVE rows, so an 8-byte column is one 128-bit load per thread
// (coalesced 512 bytes per warp instruction) and a 4-byte column one 64-bit load; values are kept in the
// widened 64-bit machine representation of the interpreter, so everything downstream is shared.
__device__ __forceinline__ void ld_pair64(const void* base, long long row, bool both, unsigned long long policy, unsigned long long (&out)[2]) {
  const unsigned long long* q = (const unsigned long long*)base + row;
  if (both) {
    if (policy)
      asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(out[0]), "=l"(out[1]) : "l"(q), "l"(policy));
    else
      asm volatile("ld.global.nc.L1::no_allocate.v2.b64 {%0, %1}, [%2];" : "=l"(out[0]), "=l"(out[1]) : "l"(q));
  } else {
    out[0] = __ldg(q);
    out[1] = 0ull;
  }
}
__device__ __forceinline__ void ld_pair32(const void* base, long long row, bool both, bool sign, unsigned long long (&out)[2]) {
  const unsigned* q = (const unsigned*)base + row;
  unsigned lo, hi = 0;
  if (both) {
    const uint2 t = __ldg((const uint2*)q);
    lo = t.x;
    hi = t.y;
  } else {
    lo = __ldg(q);
  }
  out[0] = sign ? (unsigned long long)(long long)(int)lo : (unsigned long long)lo;
  out[1] = sign ? (unsigned long long)(long long)(int)hi : (unsigned long long)hi;
}
__device__ __forceinline__ unsigned cmp_bits2(int op, int mt, const unsigned long long (&a)[2], const unsigned long long (&b)[2]) {
  unsigned f = 0;
#define DF_C2(EXPR) _Pragma("unroll") for (int r = 0; r < 2; r++) { const unsigned long long x = a[r], y = b[r]; f |= (unsigned)(EXPR) << r; }
#define DF_C2_OPS(CAST)                           \
  switch (op) {                                   \
    case V_EQ: DF_C2(CAST(x) == CAST(y)) break;   \
    case V_NE: DF_C2(CAST(x) != CAST(y)) break;   \
    case V_LT: DF_C2(CAST(x) < CAST(y)) break;    \
    case V_LE: DF_C2(CAST(x) <= CAST(y)) break;   \
    case V_GT: DF_C2(CAST(x) > CAST(y)) break;    \
    default: DF_C2(CAST(x) >= CAST(y)) break;     \
  }
  switch (mt) {
    case MT_F64: DF_C2_OPS(u2d) break;
    case MT_F32: DF_C2_OPS(u2f) break;
    case MT_I: DF_C2_OPS((long long)) break;
    default: DF_C2_OPS((unsigned long long)) break;
  }
#undef DF_C2_OPS
#undef DF_C2
  return f;
}
// NC: column slots the instantiation holds (2 = the common key + value shape: fewer registers, more CTAs
// per SM).
template <int NC>
struct PlainSrc {
  static constexpr int R = 2;
  unsigned long long cv[NC][2];
  long long row0;
  unsigned mask;
  unsigned bad = 0;
  // value selects instead of indexed access: the column values stay in registers
  __device__ __forceinline__ void col(int s, unsigned long long (&v)[2]) const {
    if (NC == 2) {
      v[0] = s == 0 ? cv[0][0] : cv[1][0];
      v[1] = s == 0 ? cv[0][1] : cv[1][1];
    } else {
      v[0] = s == 0 ? cv[0][0] : (s == 1 ? cv[1][0] : (s == 2 ? cv[2 % NC][0] : cv[3 % NC][0]));
      v[1] = s == 0 ? cv[0][1] : (s == 1 ? cv[1][1] : (s == 2 ? cv[2 % NC][1] : cv[3 % NC][1]));
    }
  }
  __device__ __forceinline__ void load(const AggParams& p, long long tb, long long n, int tid, unsigned long long policy) {
    const long long i = tb + 2ll * tid;
    row0 = p.row_begin + i;  // even: tb and row_begin are even (host-checked)
    mask = (i < n ? 1u : 0u) | (i + 1 < n ? 2u : 0u);
    bad = 0;
    const bool both = mask == 3u;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      cv[c][0] = cv[c][1] = 0ull;
      if (c < p.ps.ncols && mask) {
        const int dt = p.ps.cols[c].dtype;  // warp-uniform
        if (dt == DFGPU_FLOAT64 || dt == DFGPU_INT64 || dt == DFGPU_UINT64) ld_pair64(p.ps.cols[c].ptr, row0, both, policy, cv[c]);
        else ld_pair32(p.ps.cols[c].ptr, row0, both, dt == DFGPU_INT32, cv[c]);
      }
    }
  }
  __device__ __forceinline__ void prepare(const AggParams& p) {
    if (p.plain.pred.nterms > 0) {
      unsigned keep = 0;
      for (int t = 0; t < p.plain.pred.nterms; t++) {
        const Leaf& pt = p.plain.pred.term[t];
        unsigned long long x[2], y[2];
        col(pt.a, x);
        if (pt.kind == 2) col(pt.b, y);
        else y[0] = y[1] = pt.imm;
        const unsigned f = cmp_bits2(pt.op, pt.mtype, x, y);
        keep = t == 0 ? f : (pt.conn ? (keep | f) : (keep & f));
      }
      mask &= keep;
    }
  }
  __device__ __forceinline__ void key(const AggParams& p, int k, unsigned long long (&v)[2]) { col(p.plain.key_slot[k], v); }
  __device__ __forceinline__ unsigned arg(const AggParams& p, int gi, unsigned long long (&v)[2], unsigned& av) {
    col(p.plain.arg_slot[gi], v);
    av = 3u;
    return 0u;
  }
  __device__ __forceinline__ unsigned rowid(int r) const { return (unsigned)(row0 + r); }
};

// K5 scan.  Per row: key -> mix64 -> linear probing over table lines (ld.global.cg, 64/128 bits or 2 x 128: the
// probe also brings the in-line MIN / MAX accumulators) -> atomicCAS to claim an empty slot -> one
// fire-and-forget L2 reduction per additive accumulator and per MIN / MAX that the row improves.
// FRONT: a per-CTA open-addressed table in shared memory absorbs the updates (shared-memory atomics),
// and is merged into the global table once, when the CTA is done.  Used when the sampled prefix shows
// few groups: with a handful of hot keys every global reduction would serialise on the same L2 sector.
template <class Src, bool FRONT, bool NULLS>
__device__ __forceinline__ void hash_agg_body(const AggParams& p, unsigned long long* s_front) {
  constexpr int R = Src::R;
  const int FS = p.front_slots;                                            // slots per front table
  const int ftables = p.front_per_warp ? AG_THREADS / 32 : 1;              // tables per CTA
  unsigned long long* ftab = s_front + (p.front_per_warp ? (size_t)(threadIdx.x >> 5) * FS * (1 + p.naggs) : 0);
  if (FRONT) {
    for (int i = threadIdx.x; i < FS * ftables; i += AG_THREADS) {
      unsigned long long* tb = s_front + (size_t)(i / FS) * FS * (1 + p.naggs);
      tb[i % FS] = EMPTY_KEY;
      for (int a = 0; a < p.naggs; a++) tb[(1 + a) * FS + (i % FS)] = agg_identity(p.aggs[a].func);
    }
    __syncthreads();
  }
  const int tid = threadIdx.x, lane = tid & 31;
  const long long n = p.row_list ? p.nlist : p.nrows;
  // the input is read exactly once: mark its lines evict-first so that they do not displace the table
  const unsigned long long stream_policy = l2_evict_first_policy();
  bool bad = false;
  constexpr int TILE = AG_THREADS * R;
  const long long tstep = (long long)gridDim.x * TILE;
  Src src;
  for (long long tb = (long long)blockIdx.x * TILE; tb < n; tb += tstep) {
    // fill limit, once per warp per tile (no CTA-wide barrier in the steady state)
    unsigned long long filled = 0;
    if (lane == 0) filled = __ldcg(&p.counters[CTR_GROUPS]);
    filled = __shfl_sync(0xffffffffu, filled, 0);
    const bool full = (long long)filled >= p.max_groups;
    src.load(p, tb, n, tid, stream_policy);
    src.prepare(p);
    // group key: one packed 64-bit word (GroupByScalar vector of aggregate.rs:807-852)
    unsigned long long key[R];
#pragma unroll
    for (int r = 0; r < R; r++) key[r] = 0;
    for (int k = 0; k < p.nkeys; k++) {
      unsigned long long v[R];
      src.key(p, k, v);
#pragma unroll
      for (int r = 0; r < R; r++) key[r] |= (v[r] & p.key_mask[k]) << p.key_shift[k];
    }
    // front table (shared memory): claim / find the key there first
    int fslot[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
      fslot[r] = -1;
      if (FRONT && ((src.mask >> r) & 1u) && key[r] != EMPTY_KEY) {
        unsigned fh = (unsigned)(mix64(key[r]) >> 40) & (unsigned)(FS - 1);
        for (int pr = 0; pr < AG_FRONT_PROBES; pr++) {
          unsigned long long c = ftab[fh];
          if (c == EMPTY_KEY) c = atomicCAS(&ftab[fh], EMPTY_KEY, key[r]);
          if (c == key[r] || c == EMPTY_KEY) { fslot[r] = (int)fh; break; }
          fh = (fh + 1) & (unsigned)(FS - 1);
        }
      }
    }
    // first probe of all R rows issued back to back (R independent L2 requests in flight)
    unsigned long long h[R];
    Line ln[R];
    bool probing[R];
#pragma unroll
    for (int r = 0; r < R; r++) {
      const unsigned long long hs = mix64(key[r]);
      h[r] = p.t.home(hs);
      probing[r] = ((src.mask >> r) & 1u) && key[r] != EMPTY_KEY && fslot[r] < 0;
      ln[r].w[0] = ln[r].w[1] = ln[r].w[2] = ln[r].w[3] = 0ull;
      if (probing[r]) load_line<LINE_RT>(p.t, h[r], ln[r]);
    }
    long long slot[R];
    unsigned new_groups = 0;
#pragma unroll
    for (int r = 0; r < R; r++) {
      slot[r] = -1;
      if (!((src.mask >> r) & 1u) || fslot[r] >= 0) continue;
      if (key[r] == EMPTY_KEY) {  // the one key value that collides with the empty marker
        if (__ldcg(&p.counters[CTR_SENTINEL]) == 0ull) p.counters[CTR_SENTINEL] = 1ull;
        slot[r] = p.t.cap;
        continue;
      }
      slot[r] = probe_insert<LINE_RT>(p.t, key[r], ln[r], h[r], full, new_groups) ? (long long)h[r] : -1;
      if (slot[r] < 0) {
        const unsigned long long at = atomicAdd(&p.counters[CTR_OVERFLOW], 1ull);
        p.ovf_rows[at] = src.rowid(r);
      }
    }
    // accumulators (update_accumulators, aggregate.rs:548-612): argument evaluated once per row
    for (int g = 0; g < p.nargs; g++) {
      unsigned long long v[R];
      unsigned av;
      const unsigned b = src.arg(p, g, v, av);
      for (int a = 0; a < p.naggs; a++) {
        if (p.agg_arg[a] != g) continue;
        // AVG's sum word: the value is widened to f64 here and folded as an f64 SUM
        const bool avg = p.aggs[a].func == AGG_AVG_SUM;
        const int func = avg ? int(DFGPU_AGG_SUM) : p.aggs[a].func, mt = avg ? int(MT_F64) : p.aggs[a].mtype, l = p.t.loc[a];
        const bool cond = l >= 1 && l <= 3 && (func == DFGPU_AGG_MIN || func == DFGPU_AGG_MAX);
#pragma unroll
        for (int r = 0; r < R; r++) {
          if (NULLS && (func == DFGPU_AGG_COUNT || avg) && !((av >> r) & 1u)) continue;  // COUNT and AVG skip nulls
          const unsigned long long x = avg ? d2u(widen_f64(v[r], p.aggs[a].mtype)) : v[r];
          if (FRONT && fslot[r] >= 0 && ((src.mask >> r) & 1u)) {
            acc_fold_global(func, mt, &ftab[(1 + a) * FS + fslot[r]], x);
            if ((b >> r) & 1u) bad = true;
          } else if (slot[r] >= 0) {
            acc_fold_global_cond(func, mt, p.t.val(slot[r], a), x, cond && probing[r], cond ? line_word(ln[r], l) : 0ull);
            if ((b >> r) & 1u) bad = true;
          }
        }
      }
    }
    bad = bad || src.bad != 0;
    // one counter update per warp
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
    if (lane == 0 && new_groups) atomicAdd(&p.counters[CTR_GROUPS], (unsigned long long)new_groups);
  }
  if (FRONT) {
    // merge this CTA's front table into the global table.  New keys are always admitted here; the host
    // lowers max_groups of a FRONT launch by grid x front slots, so the table stays at most half full.
    __syncthreads();
    unsigned new_groups = 0;
    for (int i = threadIdx.x; i < FS * ftables; i += AG_THREADS) {
      const unsigned long long* tb = s_front + (size_t)(i / FS) * FS * (1 + p.naggs);
      const int j = i % FS;
      const unsigned long long key = tb[j];
      if (key == EMPTY_KEY) continue;
      unsigned long long h = p.t.home(mix64(key));
      Line ln;
      load_line<LINE_KEY>(p.t, h, ln);
      if (!probe_insert<LINE_KEY>(p.t, key, ln, h, false, new_groups)) { p.counters[CTR_ERROR] = 2ull; continue; }
      for (int a = 0; a < p.naggs; a++)
        acc_merge_global(p.aggs[a].func, p.aggs[a].mtype, p.t.val((long long)h, a), tb[(1 + a) * FS + j]);
    }
    if (new_groups) atomicAdd(&p.counters[CTR_GROUPS], (unsigned long long)new_groups);
  }
  if (bad) p.counters[CTR_ERROR] = 1ull;
}

// Occupancy target (H100): the global-table scan wants its interpreter stack in registers more than a fourth
// CTA per SM (3: up to 80 registers, no spills), the front-table scan wants the fourth CTA (4: 64 registers).
template <int DEPTH, bool FRONT, bool NULLS>
__global__ void __launch_bounds__(AG_THREADS, FRONT ? 4 : 3) k_hash_agg(const __grid_constant__ AggParams p) {
  extern __shared__ unsigned long long s_front[];  // FRONT: keys[AG_FRONT_SLOTS] then vals[naggs][AG_FRONT_SLOTS]
  hash_agg_body<InterpSrc<DEPTH, NULLS>, FRONT, NULLS>(p, s_front);
}
template <int NC, bool FRONT>
__global__ void __launch_bounds__(AG_THREADS, 4) k_hash_agg_plain(const __grid_constant__ AggParams p) {
  extern __shared__ unsigned long long s_front[];
  hash_agg_body<PlainSrc<NC>, FRONT, false>(p, s_front);
}

// K5, lean form: the canonical GROUP BY shape — one 8-byte integer key column, one 8-byte argument column, any
// subset M of {MIN = 1, MAX = 2, SUM = 4, COUNT = 8} over it, no WHERE — with everything that is dynamic in the
// generic body (loops over keys / arguments / aggregates, dtype and function switches, layout arithmetic)
// resolved at compile time: ~60 instructions per row instead of ~300 (ncu: the generic kernels are issue-bound
// well before the LSU / L2 ceiling of their scattered operations).  Same table, same protocol.
template <int M, int MT>
__global__ void __launch_bounds__(AG_THREADS, 5) k_hash_agg_lean(const __grid_constant__ AggParams p) {
  constexpr bool HAS_MIN = (M & 1) != 0, HAS_MAX = (M & 2) != 0, HAS_SUM = (M & 4) != 0, HAS_CNT = (M & 8) != 0;
  constexpr int LW = (HAS_MIN && HAS_MAX) ? 4 : ((HAS_MIN || HAS_MAX) ? 2 : 1);  // the hybrid layout's line for this M (host-checked)
  const int tid = threadIdx.x, lane = tid & 31;
  const long long n = p.nrows;
  const unsigned long long* __restrict__ kc = p.lean.key_col + p.row_begin;
  const unsigned long long* __restrict__ vc = p.lean.arg_col + p.row_begin;
  unsigned long long* const base = p.t.base;
  const unsigned long long policy = l2_evict_first_policy();
  constexpr int TILE = AG_THREADS * 2;
  const long long tstep = (long long)gridDim.x * TILE;
  // software pipeline: the two 128-bit loads of the NEXT tile are in flight while this tile's probes and
  // reductions are issued (HBM latency of the stream and L2 latency of the probe chain overlap per thread)
  // (only for the 1-word line of SUM / COUNT shapes: the 4-word line of MIN / MAX needs the registers)
  constexpr bool PF = LW == 1;
  unsigned long long nk[2] = {0ull, 0ull}, nv[2] = {0ull, 0ull};
  if (PF) {
    const long long i0 = (long long)blockIdx.x * TILE + 2ll * tid;
    if (i0 < n) {
      ld_pair64(kc, i0, i0 + 1 < n, policy, nk);
      ld_pair64(vc, i0, i0 + 1 < n, policy, nv);
    }
  }
  for (long long tb = (long long)blockIdx.x * TILE; tb < n; tb += tstep) {
    unsigned long long filled = 0;
    if (lane == 0) filled = __ldcg(&p.counters[CTR_GROUPS]);
    filled = __shfl_sync(0xffffffffu, filled, 0);
    const bool full = (long long)filled >= p.max_groups;
    const long long i = tb + 2ll * tid;
    const bool any = i < n, both = i + 1 < n;
    if (!PF && any) {
      ld_pair64(kc, i, both, policy, nk);
      ld_pair64(vc, i, both, policy, nv);
    }
    unsigned long long k[2] = {nk[0], nk[1]}, v[2] = {nv[0], nv[1]};
    if (PF) {
      const long long j = i + tstep;
      if (j < n) {
        ld_pair64(kc, j, j + 1 < n, policy, nk);
        ld_pair64(vc, j, j + 1 < n, policy, nv);
      }
    }
    unsigned long long slot[2];
    Line ln[2];
    bool act[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
      slot[r] = p.t.home(mix64(k[r]));
      act[r] = r == 0 ? any : both;
      if (act[r] && k[r] != EMPTY_KEY) load_line<LW>(p.t, slot[r], ln[r]);
    }
    unsigned new_groups = 0;
#pragma unroll
    for (int r = 0; r < 2; r++) {
      if (!act[r]) continue;
      bool have_line = true;
      if (k[r] == EMPTY_KEY) {  // the one key value that collides with the empty marker
        if (__ldcg(&p.counters[CTR_SENTINEL]) == 0ull) p.counters[CTR_SENTINEL] = 1ull;
        slot[r] = (unsigned long long)p.t.cap;
        have_line = false;
      } else {
        if (!probe_insert<LW>(p.t, k[r], ln[r], slot[r], full, new_groups)) {  // table refuses new keys: the row is replayed after the table has grown
          const unsigned long long at = atomicAdd(&p.counters[CTR_OVERFLOW], 1ull);
          p.ovf_rows[at] = (unsigned)(p.row_begin + i + r);
          continue;
        }
      }
      unsigned long long* const line = base + slot[r] * LW;
      if (HAS_MIN || HAS_MAX) {
        if (!is_nan_val(v[r], MT)) {  // f64::min / f64::max ignore NaN (aggregate.rs:139-140, 208-209)
          const unsigned long long e = ord_enc(v[r], MT);
          if (HAS_MIN && (!have_line || e < line_word(ln[r], p.lean.min_w))) atomicMin(line + p.lean.min_w, e);
          if (HAS_MAX && (!have_line || e > line_word(ln[r], p.lean.max_w))) atomicMax(line + p.lean.max_w, e);
        }
      }
      if (HAS_SUM) {
        if (MT == MT_F64) atomicAdd((double*)(p.lean.sum_arr + slot[r]), u2d(v[r]));
        else atomicAdd(p.lean.sum_arr + slot[r], v[r]);
      }
      if (HAS_CNT) atomicAdd(p.lean.cnt_arr + slot[r], 1ull);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
    if (lane == 0 && new_groups) atomicAdd(&p.counters[CTR_GROUPS], (unsigned long long)new_groups);
  }
}

// ---- wide / mixed keys ------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long wide_tag(unsigned long long h) {  // ready form: low bit set, never EMPTY_KEY
  unsigned long long t = h | 1ull;
  if (t == EMPTY_KEY) t ^= 2ull;
  return t;
}
__device__ __forceinline__ bool utf8_equal(const int* off_a, const unsigned char* bytes_a, long long ra, const Utf8Source& sb, long long rb) {
  const int sa = off_a[ra], la = off_a[ra + 1] - sa, s2 = sb.off[rb], lb = sb.off[rb + 1] - s2;
  if (la != lb) return false;
  for (int i = 0; i < la; i++)
    if (bytes_a[sa + i] != sb.bytes[s2 + i]) return false;
  return true;
}
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* q) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(q) : "memory");
  return v;
}

// K5 for wide keys.  Claim protocol of a slot: CAS the tag word EMPTY -> tag & ~1 (busy), store the key parts,
// fence, store tag | 1 (ready).  A row that meets a busy slot with its own tag polls briefly and otherwise
// defers itself to the replay list (counter CTR_DEFERRED counts those: they need no table growth, the slot is
// ready by the time the replay runs), so no thread ever waits on another one indefinitely.
template <int DEPTH, bool NULLS>
__global__ void __launch_bounds__(AG_THREADS) k_hash_agg_wide(const __grid_constant__ AggParams p) {
  typedef InterpSrc<DEPTH, NULLS> Src;
  constexpr int R = Src::R;
  const int tid = threadIdx.x, lane = tid & 31;
  const long long n = p.row_list ? p.nlist : p.nrows;
  const int KW = p.wide.kw;
  bool bad = false;
  constexpr int TILE = AG_THREADS * R;
  for (long long tb = (long long)blockIdx.x * TILE; tb < n; tb += (long long)gridDim.x * TILE) {
    unsigned long long filled = 0;
    if (lane == 0) filled = __ldcg(&p.counters[CTR_GROUPS]);
    filled = __shfl_sync(0xffffffffu, filled, 0);
    const bool full = (long long)filled >= p.max_groups;
    Src src;
    src.load(p, tb, n, tid, 0ull);
    src.prepare(p);
    // key parts: value of a fixed-width part; for a Utf8 part the program reads the string's 64-bit hash
    unsigned long long part[kMaxKeys][R];
    unsigned long long hsh[R];
#pragma unroll
    for (int r = 0; r < R; r++) hsh[r] = 0x9e3779b97f4a7c15ull;
    for (int k = 0; k < kMaxKeys; k++) {
      if (k >= KW) break;
      unsigned long long v[R];
      src.key(p, k, v);
#pragma unroll
      for (int r = 0; r < R; r++) {
        part[k][r] = v[r];
        hsh[r] = mix64(hsh[r] ^ (v[r] + 0x9e3779b97f4a7c15ull * (unsigned long long)(k + 1)));
      }
    }
    long long slot[R];
    unsigned new_groups = 0;
#pragma unroll
    for (int r = 0; r < R; r++) {
      slot[r] = -1;
      if (!((src.mask >> r) & 1u)) continue;
      const long long row = src.g.rows[r];
      const unsigned long long ready = wide_tag(hsh[r]), busy = ready & ~1ull;
      unsigned long long h = p.t.home(hsh[r]);
      bool deferred = false;
      for (int probes = 0; probes < AG_MAX_PROBE; ++probes) {
        unsigned long long* line = p.t.key((long long)h);
        unsigned long long t = ld_volatile_u64(line);
        if (t == EMPTY_KEY) {
          if (full) break;
          t = atomicCAS(line, EMPTY_KEY, busy);
          if (t == EMPTY_KEY) {  // claimed: publish the key parts, then the ready tag
            for (int k = 0; k < KW; k++) line[1 + k] = p.wide.is_utf8[k] ? (p.wide.ref_base[k] | (unsigned long long)row) : part[k][r];
            __threadfence();
            atomicExch(line, ready);
            new_groups++;
            slot[r] = (long long)h;
            break;
          }
        }
        if ((t | 1ull) == ready) {
          for (int spin = 0; t == busy && spin < 64; spin++) { __nanosleep(64); t = ld_volatile_u64(line); }
          if (t == busy) { deferred = true; break; }
          __threadfence();
          bool same = true;
          for (int k = 0; same && k < KW; k++) {
            const unsigned long long w = __ldcg(line + 1 + k);
            if (p.wide.is_utf8[k]) {
              const Utf8Source& sc = p.wide.srcs[w >> UTF8_SRC_SHIFT];
              same = utf8_equal(p.wide.off[k], p.wide.bytes[k], row, sc, (long long)(w & ((1ull << UTF8_SRC_SHIFT) - 1ull)));
            } else {
              same = w == part[k][r];
            }
          }
          if (same) { slot[r] = (long long)h; break; }
        }
        h = p.t.next(h);
      }
      if (slot[r] < 0) {
        const unsigned long long at = atomicAdd(&p.counters[CTR_OVERFLOW], 1ull);
        p.ovf_rows[at] = (unsigned)row;
        if (deferred) atomicAdd(&p.counters[CTR_DEFERRED], 1ull);
      }
    }
    for (int g = 0; g < p.nargs; g++) {
      unsigned long long v[R];
      unsigned av;
      const unsigned b = src.arg(p, g, v, av);
      for (int a = 0; a < p.naggs; a++) {
        if (p.agg_arg[a] != g) continue;
        const bool avg = p.aggs[a].func == AGG_AVG_SUM;  // widened here, folded as an f64 SUM
        const int func = avg ? int(DFGPU_AGG_SUM) : p.aggs[a].func, mt = avg ? int(MT_F64) : p.aggs[a].mtype;
#pragma unroll
        for (int r = 0; r < R; r++) {
          if (NULLS && (func == DFGPU_AGG_COUNT || avg) && !((av >> r) & 1u)) continue;
          if (slot[r] >= 0) {
            acc_fold_global(func, mt, p.t.val(slot[r], a), avg ? d2u(widen_f64(v[r], p.aggs[a].mtype)) : v[r]);
            if ((b >> r) & 1u) bad = true;
          }
        }
      }
    }
    bad = bad || src.bad != 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
    if (lane == 0 && new_groups) atomicAdd(&p.counters[CTR_GROUPS], (unsigned long long)new_groups);
  }
  if (bad) p.counters[CTR_ERROR] = 1ull;
}

// Re-insertion of the (distinct) groups of a wide-key table into a bigger one: every entry goes to the first
// empty slot after its home; no key comparison is needed because the source table holds each key once.  An entry that
// finds no empty slot in cap probes sets *error to 2.
struct WideMoveParams {
  TableLayout from, to;
  int kw, naggs;
  unsigned long long* error;
};
__global__ void __launch_bounds__(256) k_wide_move(const __grid_constant__ WideMoveParams p) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < p.from.cap; s += (long long)gridDim.x * blockDim.x) {
    const unsigned long long* src = p.from.key(s);
    const unsigned long long tag = src[0];
    if (tag == EMPTY_KEY) continue;
    unsigned long long h = p.to.home(tag & ~1ull);  // the tag IS the hash (but for its low bit): same home rule as the scan
    long long probes = 0;
    for (; probes < p.to.cap; probes++) {
      unsigned long long* dst = p.to.key((long long)h);
      if (atomicCAS(dst, EMPTY_KEY, tag) == EMPTY_KEY) {
        for (int k = 0; k < p.kw; k++) dst[1 + k] = src[1 + k];
        for (int a = 0; a < p.naggs; a++) *p.to.val((long long)h, a) = *p.from.val(s, a);
        break;
      }
      h = p.to.next(h);
    }
    if (probes == p.to.cap) *p.error = 2ull;
  }
}

// K4: no GROUP BY.  Per-thread accumulators live in shared memory (one 8-byte cell per thread per
// aggregate, conflict-free), block-reduced at the end, one global reduction per CTA per aggregate.
constexpr int RD_R = 8;  // rows per thread per tile in the column reduce (more bytes in flight per SM)
constexpr int RD_TILE = AG_THREADS * RD_R;

// NULLS: array_ops::{min,max,sum} skip nulls and report None when nothing was non-null
// (restated from arrow 0.12; call sites aggregate.rs:347-541): the number of non-null inputs per
// aggregate is accumulated in counter CTR_NONNULL + a so finish can emit a null.  Under a WHERE the
// arguments are read as over FilterRelation's bitmap-free output (eval_after_where): only a CASE-made null
// (extended interpreter) is skipped, and without one an aggregate is null only when no row passed.
template <int DEPTH, bool NULLS>
__global__ void __launch_bounds__(AG_THREADS) k_reduce(const __grid_constant__ AggParams p) {
  __shared__ unsigned long long s_acc[kMaxAggs][AG_THREADS];
  __shared__ unsigned long long s_red[AG_THREADS / 32];
  unsigned nn[kMaxAggs];
#pragma unroll
  for (int a = 0; a < kMaxAggs; a++) nn[a] = 0;
  unsigned passed = 0;  // rows that passed the fused predicate (counter CTR_PASSED: an aggregate over zero rows is null)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int a = 0; a < p.naggs; a++) s_acc[a][tid] = agg_identity(p.aggs[a].func);
  bool bad = false;
  for (long long tb = (long long)blockIdx.x * RD_TILE; tb < p.nrows; tb += (long long)gridDim.x * RD_TILE) {
    GlobalRows<RD_R> src;
    src.valid = 0;
    long long (&rows)[RD_R] = src.rows;
#pragma unroll
    for (int r = 0; r < RD_R; r++) {
      const long long i = tb + (long long)r * AG_THREADS + tid;
      rows[r] = i < p.nrows ? i : -1;
      if (i < p.nrows) src.valid |= 1u << r;
    }
    unsigned rmask = src.valid;  // rows that pass the fused WHERE predicate (program 0)
    if (p.has_pred) {
      unsigned long long v[RD_R];
      unsigned pv;
      const unsigned b = eval_program_n<DEPTH, RD_R, false, NULLS>(p.ps, 0, src, v, pv);
      bad = bad || (b != 0);
      unsigned keep = 0;
#pragma unroll
      for (int r = 0; r < RD_R; r++) keep |= (unsigned)(v[r] & 1ull) << r;
      rmask &= keep;
    }
    if (p.has_pred) passed += __popc(rmask);
    for (int g = 0; g < p.nargs; g++) {
      unsigned long long v[RD_R];
      unsigned av;
      const unsigned b = eval_after_where<DEPTH, RD_R, NULLS>(p, p.has_pred + g, src, v, av);
      bad = bad || ((b & rmask) != 0);
#pragma unroll
      for (int a = 0; a < kMaxAggs; a++) {
        if (a >= p.naggs || p.agg_arg[a] != g) continue;
        const int func = p.aggs[a].func, mt = p.aggs[a].mtype;
        unsigned long long acc = s_acc[a][tid];
#pragma unroll
        for (int r = 0; r < RD_R; r++)
          if (((rmask >> r) & 1u) && (!NULLS || ((av >> r) & 1u))) acc = acc_fold(func, mt, acc, v[r]);
        s_acc[a][tid] = acc;
        // under a WHERE the host counts CTR_PASSED instead, unless a CASE can make nulls (extended interpreter)
        if (NULLS && (!p.has_pred || DEPTH == kCaseDepth)) nn[a] += __popc(av & rmask);
      }
    }
  }
  for (int a = 0; a < p.naggs; a++) {
    const int func = p.aggs[a].func, mt = p.aggs[a].mtype;
    unsigned long long acc = s_acc[a][tid];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = acc_merge(func, mt, acc, __shfl_xor_sync(0xffffffffu, acc, o));
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      acc = lane < AG_THREADS / 32 ? s_red[lane] : agg_identity(func);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc = acc_merge(func, mt, acc, __shfl_xor_sync(0xffffffffu, acc, o));
      if (lane == 0) acc_merge_global(func, mt, p.t.val(0, a), acc);  // cap == 0: slot 0
    }
    __syncthreads();
  }
  if (NULLS) {
#pragma unroll
    for (int a = 0; a < kMaxAggs; a++) {
      unsigned c = nn[a];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0 && c && a < p.naggs) atomicAdd(&p.counters[CTR_NONNULL + a], (unsigned long long)c);
    }
  }
  if (p.has_pred) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) passed += __shfl_xor_sync(0xffffffffu, passed, o);
    if (lane == 0 && passed) atomicAdd(&p.counters[CTR_PASSED], (unsigned long long)passed);
  }
  if (bad) p.counters[CTR_ERROR] = 1ull;
}

// K4 fast path: every aggregate argument is a plain, null-free Float64 column.  One pass per distinct
// column with 128-bit loads; SUM / MIN / MAX / COUNT of the column are all cheap enough to be computed
// together and the requested ones are merged into the accumulators.
struct ReduceF64Params {
  const double* col[kMaxAggs];  // distinct argument columns
  int ncols;
  long long nrows;
  int naggs;
  AggDesc aggs[kMaxAggs];
  int agg_arg[kMaxAggs];
  TableLayout t;
};
__global__ void __launch_bounds__(256) k_reduce_f64(const __grid_constant__ ReduceF64Params p) {
  __shared__ unsigned long long s_red[3][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long npairs = p.nrows >> 1;
  for (int g = 0; g < p.ncols; g++) {
    const double2* __restrict__ c2 = reinterpret_cast<const double2*>(p.col[g]);
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    unsigned long long mn = ~0ull, mx = 0ull;
    auto fold = [&](double v, double& s) {
      s += v;
      if (v == v) {  // MIN / MAX skip NaN (f64::min / f64::max, aggregate.rs:139-140,208-209)
        const unsigned long long e = ord_enc(d2u(v), MT_F64);
        mn = e < mn ? e : mn;
        mx = e > mx ? e : mx;
      }
    };
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + tid;
    for (; i + stride < npairs; i += 2 * stride) {  // two independent 128-bit loads in flight
      const double2 a = __ldg(&c2[i]), b = __ldg(&c2[i + stride]);
      fold(a.x, s0); fold(a.y, s1); fold(b.x, s2); fold(b.y, s3);
    }
    if (i < npairs) { const double2 a = __ldg(&c2[i]); fold(a.x, s0); fold(a.y, s1); }
    if ((p.nrows & 1) && blockIdx.x == 0 && tid == 0) fold(p.col[g][p.nrows - 1], s2);
    unsigned long long sum = d2u((s0 + s1) + (s2 + s3));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum = d2u(u2d(sum) + u2d(__shfl_xor_sync(0xffffffffu, sum, o)));
      const unsigned long long a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
      mn = a < mn ? a : mn;
      mx = b > mx ? b : mx;
    }
    if (lane == 0) { s_red[0][warp] = sum; s_red[1][warp] = mn; s_red[2][warp] = mx; }
    __syncthreads();
    if (warp == 0) {
      sum = lane < 8 ? s_red[0][lane] : 0ull;
      mn = lane < 8 ? s_red[1][lane] : ~0ull;
      mx = lane < 8 ? s_red[2][lane] : 0ull;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) {
        sum = d2u(u2d(sum) + u2d(__shfl_xor_sync(0xffffffffu, sum, o)));
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, mn, o), b = __shfl_xor_sync(0xffffffffu, mx, o);
        mn = a < mn ? a : mn;
        mx = b > mx ? b : mx;
      }
      if (lane == 0) {
        for (int a = 0; a < p.naggs; a++) {
          if (p.agg_arg[a] != g) continue;
          const int f = p.aggs[a].func;
          if (f == DFGPU_AGG_SUM || f == AGG_AVG_SUM) atomicAdd((double*)p.t.val(0, a), u2d(sum));
          else if (f == DFGPU_AGG_MIN) atomicMin(p.t.val(0, a), mn);
          else if (f == DFGPU_AGG_MAX) atomicMax(p.t.val(0, a), mx);
          else if (blockIdx.x == 0) atomicAdd(p.t.val(0, a), (unsigned long long)p.nrows);  // COUNT of a null-free column
        }
      }
    }
    __syncthreads();
  }
}

// K7: scan the table, emit occupied slots densely.  raw != 0 keeps packed keys / undecoded
// accumulators (the exchange format of the multi-GPU merge).
struct CompactParams {
  TableLayout t;
  int sentinel_used;
  int nkeys, naggs, raw;
  long long raw_stride;  // raw output: element idx of every raw array lives at idx * raw_stride (0 = 1: dense arrays)
  const unsigned long long* sentinel_flag;  // non-null: device flag that says whether the sentinel slot (slot cap) is in use
  int wide_kw;           // wide keys: line words 1..wide_kw are the key parts (a Utf8 part = a string reference)
  int key_is_utf8[kMaxKeys];
  AggDesc aggs[kMaxAggs];
  // aggregates over the same argument expression (MIN(v), MAX(v), SUM(v)) share one evaluation:
  // programs [nkeys, nkeys + nargs) are the DISTINCT argument programs, agg_arg[a] picks one
  int agg_arg[kMaxAggs];
  int nargs;
  unsigned long long key_mask[kMaxKeys];
  int key_shift[kMaxKeys];
  int key_dtype[kMaxKeys];
  void* out_keys[kMaxKeys];
  void* out_vals[kMaxAggs];
  unsigned long long* counter;
};

__global__ void __launch_bounds__(256) k_compact(const __grid_constant__ CompactParams p) {
  const int lane = threadIdx.x & 31;
  const long long total = p.t.cap + 1;
  const long long step = (long long)gridDim.x * blockDim.x;
  // round the loop bound up to a warp multiple so ballots stay converged
  for (long long s0 = (long long)blockIdx.x * blockDim.x; s0 < total; s0 += step) {
    const long long s = s0 + threadIdx.x;
    bool occ = false;
    unsigned long long key = 0;
    if (s < p.t.cap) { key = *p.t.key(s); occ = key != EMPTY_KEY; }
    else if (s == p.t.cap) { key = EMPTY_KEY; occ = p.sentinel_used != 0 || (p.sentinel_flag && *p.sentinel_flag != 0ull); }
    const unsigned m = __ballot_sync(0xffffffffu, occ);
    if (!m) continue;
    unsigned long long basei = 0;
    if (lane == 0) basei = atomicAdd(p.counter, (unsigned long long)__popc(m));
    basei = __shfl_sync(0xffffffffu, basei, 0);
    if (!occ) continue;
    const long long idx = (long long)(basei + __popc(m & ((1u << lane) - 1u)));
    if (p.raw) {
      const long long at = p.raw_stride ? idx * p.raw_stride : idx;
      ((unsigned long long*)p.out_keys[0])[at] = key;
      for (int a = 0; a < p.naggs; a++) ((unsigned long long*)p.out_vals[a])[at] = *p.t.val(s, a);
    } else {
      for (int k = 0; k < p.nkeys; k++) {
        if (p.wide_kw) {
          const unsigned long long w = p.t.key(s)[1 + k];
          if (p.key_is_utf8[k]) ((unsigned long long*)p.out_keys[k])[idx] = w;  // string reference, gathered by the host
          else store_elem(p.out_keys[k], p.key_dtype[k], idx, w);
          continue;
        }
        unsigned long long v = (key >> p.key_shift[k]) & p.key_mask[k];
        store_elem(p.out_keys[k], p.key_dtype[k], idx, v);
      }
      for (int a = 0; a < p.naggs; a++) {
        unsigned long long v = *p.t.val(s, a);
        const int f = p.aggs[a].func;
        if (f == DFGPU_AGG_MIN || f == DFGPU_AGG_MAX) v = ord_dec(v, p.aggs[a].mtype);
        store_elem(p.out_vals[a], p.aggs[a].out_dtype, idx, v);
      }
    }
  }
}

// Re-insert (raw key, raw accumulators) entries into a table: used to grow the table and to merge
// the partial aggregates of other GPUs (K6).
struct MergeParams {
  const unsigned long long* in_keys;
  const unsigned long long* in_vals[kMaxAggs];
  long long in_stride;  // entry i of every input array lives at i * in_stride (0 = 1: dense arrays)
  long long n;
  TableLayout t;
  int naggs;
  AggDesc aggs[kMaxAggs];
  unsigned long long* counters;
};

__global__ void __launch_bounds__(256) k_merge(const __grid_constant__ MergeParams p) {
  unsigned new_groups = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    const long long at = p.in_stride ? i * p.in_stride : i;
    const unsigned long long key = p.in_keys[at];
    long long slot;
    if (key == EMPTY_KEY) {
      p.counters[CTR_SENTINEL] = 1ull;
      slot = p.t.cap;
    } else {
      unsigned long long h = p.t.home(mix64(key));
      Line ln;
      load_line<LINE_KEY>(p.t, h, ln);
      if (!probe_insert<LINE_KEY>(p.t, key, ln, h, false, new_groups)) { p.counters[CTR_ERROR] = 2ull; continue; }  // cannot happen: caller sizes the table
      slot = (long long)h;
    }
    for (int a = 0; a < p.naggs; a++)
      acc_merge_global(p.aggs[a].func, p.aggs[a].mtype, p.t.val(slot, a), p.in_vals[a][at]);
  }
  if (new_groups) atomicAdd(&p.counters[CTR_GROUPS], (unsigned long long)new_groups);
}

// ---- owner-partitioned exchange of partial aggregates (multi-GPU merge, SURVEY.md §8e) -----------------
// Every group key has one OWNER rank, a function of the key alone, so that each rank merges only 1/W of the
// keys: owner = bits of mix64(key) that the table slot does not use.
constexpr int AG_MAX_WORLD = 64;
__device__ __forceinline__ int owner_of(unsigned long long key, int world) {
  return key == EMPTY_KEY ? 0 : (int)((mix64(key) & 0xffffffffull) % (unsigned long long)world);
}
struct OwnerParams {
  const unsigned long long* keys;              // raw (packed) keys of the local groups
  const unsigned long long* vals[kMaxAggs];    // raw accumulators, dense arrays
  long long n;
  int world, naggs;
  unsigned long long* counts;                  // [world] entries per owner
  unsigned long long seg_off[AG_MAX_WORLD];    // scatter: first entry of owner o's segment in `rows`
  unsigned long long* cursor;                  // [world], zeroed
  unsigned long long* rows;                    // scatter output: entries of (1 + naggs) words, grouped by owner
};
__global__ void __launch_bounds__(256) k_owner_count(const __grid_constant__ OwnerParams p) {
  __shared__ unsigned s_cnt[AG_MAX_WORLD];
  if (threadIdx.x < AG_MAX_WORLD) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&s_cnt[owner_of(p.keys[i], p.world)], 1u);
  __syncthreads();
  if (threadIdx.x < p.world && s_cnt[threadIdx.x]) atomicAdd(&p.counts[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
}
__global__ void __launch_bounds__(256) k_owner_scatter(const __grid_constant__ OwnerParams p) {
  const long long E = 1 + p.naggs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = p.keys[i];
    const int o = owner_of(key, p.world);
    const unsigned long long j = p.seg_off[o] + atomicAdd(&p.cursor[o], 1ull);
    unsigned long long* row = p.rows + j * E;
    row[0] = key;
    for (int a = 0; a < p.naggs; a++) row[1 + a] = p.vals[a][i];
  }
}

// raw rows (key, accumulators...) -> typed result columns: group columns first, then aggregates
// (aggregate.rs:890-949); the decode half of k_compact for rows that arrive from the exchange
struct DecodeParams {
  const unsigned long long* rows;
  long long n;
  // rows arrive as `nseg` segments of seg_stride entries each, of which the first seg_n[r] are real (the padded
  // all-gather of the owned groups); nseg == 0: one dense list
  int nseg;
  long long seg_stride;
  long long seg_n[AG_MAX_WORLD];
  int nkeys, naggs;
  AggDesc aggs[kMaxAggs];
  unsigned long long key_mask[kMaxKeys];
  int key_shift[kMaxKeys];
  int key_dtype[kMaxKeys];
  void* out_keys[kMaxKeys];
  void* out_vals[kMaxAggs];
};
__global__ void __launch_bounds__(256) k_decode_rows(const __grid_constant__ DecodeParams p) {
  const long long E = 1 + p.naggs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    long long at = i;
    if (p.nseg) {  // dense output index -> (segment, entry)
      long long j = i;
      int r = 0;
      while (r < p.nseg - 1 && j >= p.seg_n[r]) j -= p.seg_n[r++];
      at = (long long)r * p.seg_stride + j;
    }
    const unsigned long long* row = p.rows + at * E;
    const unsigned long long key = row[0];
    for (int k = 0; k < p.nkeys; k++) store_elem(p.out_keys[k], p.key_dtype[k], i, (key >> p.key_shift[k]) & p.key_mask[k]);
    for (int a = 0; a < p.naggs; a++) {
      unsigned long long v = row[1 + a];
      const int f = p.aggs[a].func;
      if (f == DFGPU_AGG_MIN || f == DFGPU_AGG_MAX) v = ord_dec(v, p.aggs[a].mtype);
      store_elem(p.out_vals[a], p.aggs[a].out_dtype, i, v);
    }
  }
}

// AVG output: from the sum and count columns of an AVG's two words (compacted or decoded), the Float64 means, a
// bit-packed validity bitmap (a group, or the scalar row, with no non-null value is null) and the number of nulls.
struct AvgFinishParams {
  const double* sum;
  const unsigned long long* cnt;
  long long n;
  double* out;
  unsigned* validity;  // (n + 31) / 32 words: bit j of word w is row 32 w + j (arrow's LSB-first bytes)
  unsigned long long* nulls;
};
__global__ void __launch_bounds__(256) k_avg_finish(const __grid_constant__ AvgFinishParams p) {
  const int lane = threadIdx.x & 31;
  unsigned nulls = 0;
  // the loop bound is a multiple of the block for every thread, so ballots stay converged
  for (long long i0 = (long long)blockIdx.x * blockDim.x; i0 < p.n; i0 += (long long)gridDim.x * blockDim.x) {
    const long long i = i0 + threadIdx.x;
    const bool in = i < p.n;
    const unsigned long long c = in ? p.cnt[i] : 0ull;
    if (in) p.out[i] = c ? p.sum[i] / (double)c : 0.0;
    const unsigned valid = __ballot_sync(0xffffffffu, c != 0ull), rows = __ballot_sync(0xffffffffu, in);
    if (lane == 0 && rows) {
      p.validity[i >> 5] = valid;
      nulls += (unsigned)__popc(rows & ~valid);
    }
  }
  if (lane == 0 && nulls) atomicAdd(p.nulls, (unsigned long long)nulls);
}

// Utf8 GROUP BY keys are grouped by a 64-bit hash of the string; accumulator `rep_agg` holds the
// earliest (source << 40 | row) of each group.  Every row's string must equal its group's
// representative string, otherwise two different strings collided on the hash.
struct VerifyParams {
  const unsigned long long* hashes;
  long long n;
  TableLayout t;
  int rep_agg;
  const int* off;
  const unsigned char* bytes;
  const Utf8Source* srcs;
  unsigned long long* flag;
  int has_pred;  // a fused WHERE ran: a row it dropped may have no group
};
__global__ void __launch_bounds__(256) k_utf8_group_verify(const __grid_constant__ VerifyParams p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    const long long slot = p.t.find(p.hashes[i], true);
    if (slot < 0) {
      if (!p.has_pred) *p.flag = 2ull;
      continue;
    }
    const unsigned long long rep = *p.t.val(slot, p.rep_agg);
    const Utf8Source& sc = p.srcs[rep >> UTF8_SRC_SHIFT];
    const long long r = (long long)(rep & ((1ull << UTF8_SRC_SHIFT) - 1ull));
    const int s = p.off[i], len = p.off[i + 1] - s, s2 = sc.off[r], len2 = sc.off[r + 1] - s2;
    bool same = len == len2;
    for (int b = 0; same && b < len; b++) same = p.bytes[s + b] == sc.bytes[s2 + b];
    if (!same) *p.flag = 1ull;
  }
}

// fill the table with empty keys and accumulator identities
struct InitParams {
  TableLayout t;
  long long nslots;
  int naggs;
  unsigned long long ident[kMaxAggs];
};
__global__ void __launch_bounds__(256) k_table_init(const __grid_constant__ InitParams p) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < p.nslots; s += (long long)gridDim.x * blockDim.x) {
    *p.t.key(s) = EMPTY_KEY;
    for (int a = 0; a < p.naggs; a++) *p.t.val(s, a) = p.ident[a];
  }
}

// ---- COUNT(DISTINCT x): pair sets ----------------------------------------------------------------------------
// One open-addressed set per distinct argument program.  A slot is 16 bytes, (packed group key, normalised value),
// both words EMPTY_KEY when empty.  A slot is only ever written by the 128-bit CAS that claims it, so it changes
// once, from empty to its pair.  The one pair equal to the empty marker is kept in a flag counter instead.
constexpr int DCTR_OVERFLOW = 0;  // rows appended to the overflow list
constexpr int DCTR_ERROR = 1;     // 1: an expression raised DivideByZero, 2: a pair found no slot, or no group
constexpr int DCTR_SET = 2;       // [DCTR_SET + 2s]: pairs in set s, [DCTR_SET + 2s + 1]: nonzero when set s holds the empty-marker pair
constexpr int DCTR_SLOTS = DCTR_SET + 2 * kMaxAggs;

struct SetParams {
  SetView set[kMaxAggs];
  long long max_fill[kMaxAggs];         // new pairs are refused (-> overflow list) beyond this fill
  int mt[kMaxAggs];                     // machine type of the argument
};

// 128-bit atomicCAS (ATOMG.E.CAS.128 on sm_90); returns the slot as it was, read atomically
__device__ __forceinline__ void cas128(unsigned long long* q, unsigned long long cmp_lo, unsigned long long cmp_hi, unsigned long long new_lo,
                                       unsigned long long new_hi, unsigned long long& old_lo, unsigned long long& old_hi) {
  asm volatile(
      "{\n\t.reg .b128 d, c, s;\n\t"
      "mov.b128 c, {%2, %3};\n\t"
      "mov.b128 s, {%4, %5};\n\t"
      "atom.global.cas.b128 d, [%6], c, s;\n\t"
      "mov.b128 {%0, %1}, d;\n\t}"
      : "=l"(old_lo), "=l"(old_hi)
      : "l"(cmp_lo), "l"(cmp_hi), "l"(new_lo), "l"(new_hi), "l"(q)
      : "memory");
}

// The word distinctness is decided on: SQL `=` for floats (+0.0 equals -0.0), except that every NaN is one value.
__device__ __forceinline__ unsigned long long distinct_norm(unsigned long long v, int mt) {
  if (mt == MT_F64) {
    const double d = u2d(v);
    return d != d ? 0x7ff8000000000000ull : (d == 0.0 ? 0ull : v);
  }
  if (mt == MT_F32) {
    const float f = u2f(v);
    return f != f ? 0x7fc00000ull : (f == 0.0f ? 0ull : (v & 0xffffffffull));
  }
  return v;
}

// Insert (key, val): 1 = inserted, 0 = already there, -1 = not inserted (full: the set refuses new pairs; or probe limit).
__device__ __forceinline__ int set_insert(const SetView& set, unsigned long long key, unsigned long long val, bool full) {
  unsigned long long h = set.home(mix64(val ^ mix64(key)));
  for (int probes = 0; probes < AG_MAX_PROBE; ++probes) {
    unsigned long long* q = set.slots + 2 * h;
    unsigned long long a, b;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(q) : "memory");
    // the halves of a plain load may straddle a claim: only a view without an EMPTY_KEY half is certainly a
    // published pair; otherwise the CAS (a no-op when full) reads the slot atomically, claiming it when empty
    if (a == EMPTY_KEY || b == EMPTY_KEY) {
      cas128(q, EMPTY_KEY, EMPTY_KEY, full ? EMPTY_KEY : key, full ? EMPTY_KEY : val, a, b);
      if (a == EMPTY_KEY && b == EMPTY_KEY) return full ? -1 : 1;
    }
    if (a == key && b == val) return 0;
    h = set.next(h);
  }
  return -1;
}

// Insert the (group key, argument) pairs of a batch into the sets, one set per argument program p.ps[has_pred +
// nkeys + s].  Runs after the group scan over the same rows: every key it packs (exactly as the scan packs it) is
// already in the group table.  Rows that fail the WHERE clause are skipped, and so are null arguments when there is
// no WHERE (under one, InterpSrc reads the arguments as over null-free arrays).  A row that some set
// refused goes to the overflow list and is replayed into every set after growth (inserting a pair twice is harmless).
template <class Src, bool NULLS>
__device__ __forceinline__ void distinct_insert_body(const AggParams& p, const SetParams& sp) {
  constexpr int R = Src::R;
  constexpr int TILE = AG_THREADS * R;
  const int tid = threadIdx.x, lane = tid & 31;
  const long long n = p.row_list ? p.nlist : p.nrows;
  const unsigned long long stream_policy = l2_evict_first_policy();
  bool bad = false;
  Src src;
  for (long long tb = (long long)blockIdx.x * TILE; tb < n; tb += (long long)gridDim.x * TILE) {
    unsigned full = 0;  // bit s: set s refuses new pairs (fill limit, once per warp per tile)
    if (lane == 0)
      for (int s = 0; s < p.nargs; s++)
        if ((long long)__ldcg(&p.counters[DCTR_SET + 2 * s]) >= sp.max_fill[s]) full |= 1u << s;
    full = __shfl_sync(0xffffffffu, full, 0);
    src.load(p, tb, n, tid, stream_policy);
    src.prepare(p);
    unsigned long long key[R];
#pragma unroll
    for (int r = 0; r < R; r++) key[r] = 0;
    for (int k = 0; k < p.nkeys; k++) {
      unsigned long long v[R];
      src.key(p, k, v);
#pragma unroll
      for (int r = 0; r < R; r++) key[r] |= (v[r] & p.key_mask[k]) << p.key_shift[k];
    }
    unsigned refused = 0;
    for (int s = 0; s < p.nargs; s++) {
      unsigned long long v[R];
      unsigned av;
      const unsigned b = src.arg(p, s, v, av);
      unsigned added = 0;
#pragma unroll
      for (int r = 0; r < R; r++) {
        if (!((src.mask >> r) & 1u) || (NULLS && !((av >> r) & 1u))) continue;
        if ((b >> r) & 1u) bad = true;
        const unsigned long long val = distinct_norm(v[r], sp.mt[s]);
        if (key[r] == EMPTY_KEY && val == EMPTY_KEY) {
          if (__ldcg(&p.counters[DCTR_SET + 2 * s + 1]) == 0ull) p.counters[DCTR_SET + 2 * s + 1] = 1ull;
          continue;
        }
        const int rc = set_insert(sp.set[s], key[r], val, ((full >> s) & 1u) != 0);
        if (rc > 0) added++;
        else if (rc < 0) refused |= 1u << r;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) added += __shfl_xor_sync(0xffffffffu, added, o);
      if (lane == 0 && added) atomicAdd(&p.counters[DCTR_SET + 2 * s], (unsigned long long)added);
    }
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (!((refused >> r) & 1u)) continue;
      const unsigned long long at = atomicAdd(&p.counters[DCTR_OVERFLOW], 1ull);
      p.ovf_rows[at] = src.rowid(r);
    }
    bad = bad || src.bad != 0;
  }
  if (bad) p.counters[DCTR_ERROR] = 1ull;
}
template <int DEPTH, bool NULLS>
__global__ void __launch_bounds__(AG_THREADS, 3) k_distinct_insert(const __grid_constant__ AggParams p, const __grid_constant__ SetParams sp) {
  distinct_insert_body<InterpSrc<DEPTH, NULLS>, NULLS>(p, sp);
}
template <int NC>
__global__ void __launch_bounds__(AG_THREADS) k_distinct_insert_plain(const __grid_constant__ AggParams p, const __grid_constant__ SetParams sp) {
  distinct_insert_body<PlainSrc<NC>, false>(p, sp);
}

// Re-insertion of a set's pairs into a bigger set (growth).
struct SetMoveParams {
  SetView from, to;
  unsigned long long* error;
};
__global__ void __launch_bounds__(256) k_set_move(const __grid_constant__ SetMoveParams p) {
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < p.from.cap; s += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = p.from.slots[2 * s], val = p.from.slots[2 * s + 1];
    if (key == EMPTY_KEY && val == EMPTY_KEY) continue;
    if (set_insert(p.to, key, val, false) < 0) *p.error = 2ull;
  }
}

// Count a set's pairs into the group table: +1 on the accumulator words `words` of the pair's group.  Index `set.cap` is
// the empty-marker pair (flag `marker`), whose group is the sentinel slot.  A pair whose group is missing sets `error`.
struct DistinctCountParams {
  SetView set;
  const unsigned long long* marker;
  TableLayout t;
  int sentinel_used;
  int nwords;
  int words[kMaxAggs];
  unsigned long long* error;
};
__global__ void __launch_bounds__(256) k_distinct_count(const __grid_constant__ DistinctCountParams p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= p.set.cap; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long key = EMPTY_KEY;
    if (i < p.set.cap) {
      key = p.set.slots[2 * i];
      if (key == EMPTY_KEY && p.set.slots[2 * i + 1] == EMPTY_KEY) continue;
    } else if (*p.marker == 0ull) {
      continue;
    }
    const long long slot = p.t.find(key, p.sentinel_used != 0);
    if (slot < 0) { *p.error = 2ull; continue; }
    for (int w = 0; w < p.nwords; w++) atomicAdd(p.t.val(slot, p.words[w]), 1ull);
  }
}

}  // namespace dfgpu

using namespace dfgpu;

// ---------------------------------------------------------------------------------------------
// host state of one AggregateRelation
// ---------------------------------------------------------------------------------------------
struct dfgpu_aggstate {
  dfgpu_ctx* ctx = nullptr;
  std::vector<std::vector<dfgpu_insn>> key_progs;
  std::vector<std::vector<dfgpu_insn>> arg_progs;
  std::vector<int> funcs, out_dtypes;
  int nkeys = 0, naggs = 0;
  // resolved at the first update
  bool typed = false;
  std::vector<int> key_dtypes;
  std::vector<int> key_shift;
  std::vector<unsigned long long> key_mask;
  std::vector<AggDesc> descs;
  // table
  long long expected = 0;
  TableLayout t{};
  bool aos = false;        // "line" layout: every accumulator shares the line with the key (tables beyond L2)
  std::vector<dfgpu_insn> pred_prog;  // fused WHERE predicate (dfgpu_aggregate_set_predicate); empty = none
  // the bytes of the DFGPU_OP_LIT_UTF8 literals of the kept programs: the caller's are borrowed for the call only
  std::deque<std::string> utf8_lits;
  void own_literals(std::vector<dfgpu_insn>& prog) {
    for (dfgpu_insn& in : prog)
      if (in.op == DFGPU_OP_LIT_UTF8 && in.col > 0 && in.lit.str) {  // malformed ones are refused when compiled
        utf8_lits.emplace_back(in.lit.str, size_t(in.col));
        in.lit.str = utf8_lits.back().data();
      }
  }
  bool use_front = false;  // route rows through the per-CTA shared-memory front table
  // wide keys: composite keys of more than 64 bits or with Utf8 parts (k_hash_agg_wide)
  bool wide = false;
  std::vector<int> key_is_utf8;
  // Utf8 GROUP BY key (aggregate.rs:842-847): grouped by a 64-bit string hash; the last accumulator is a
  // hidden MIN(source << 40 | row) = representative row of the group; the key columns of all batches are
  // retained so the representatives' strings can be gathered at finish
  bool utf8_key = false;
  std::vector<void*> utf8_owned;         // retained offsets / bytes buffers (device)
  std::vector<Utf8Source> utf8_srcs;     // host copy of the source table
  Utf8Source* d_utf8_srcs = nullptr;
  bool saw_nulls = false;  // some batch went through the null-aware reduce: per-aggregate non-null counts are on the device
  std::vector<long long> nonnull_host = std::vector<long long>(8, 0);
  unsigned long long* d_counters = nullptr;  // CTR_SLOTS words, see CTR_*
  long long ngroups = 0;
  bool sentinel_used = false;
  long long rows_seen = 0;
  bool finished = false;
  // COUNT(DISTINCT): key_progs / arg_progs / funcs / out_dtypes above describe the accumulators the scan kernels
  // update, table words [0, nscan).  Word nscan + j belongs to the j-th COUNT(DISTINCT), which counts the pairs of set
  // dist_set[j]; set s holds the (packed key, value) pairs of argument program dist_progs[s].
  int nscan = 0;
  std::vector<std::vector<dfgpu_insn>> dist_progs;
  std::vector<int> dist_set;
  // AVG: each one is two scan words, an AGG_AVG_SUM word and the COUNT word right after it; out_word points at the sum
  // word and out_is_avg says that the output is computed from the pair (k_avg_finish)
  std::vector<int> out_word;        // user aggregate -> table word
  std::vector<char> out_is_avg;
  bool emit_words = false;          // finish returns one column per table word (the regroup merge across ranks)
  std::vector<int> dist_dtypes;     // argument dtype per set, typed at the first batch
  std::vector<SetView> sets;
  unsigned long long* d_dctr = nullptr;  // DCTR_SLOTS words, see DCTR_*

  ~dfgpu_aggstate() {
    if (ctx) {
      ctx->free(t.base);
      ctx->free(d_counters);
      for (void* p : utf8_owned) ctx->free(p);
      ctx->free(d_utf8_srcs);
      for (const SetView& s : sets) ctx->free(s.slots);
      ctx->free(d_dctr);
    }
  }
};

namespace {

// Growth policy of the group table and the pair sets (sized by table_cap, hash_table.cuh): a table takes new entries up
// to half full and grows x4.
long long fill_limit(long long cap) { return cap / 2; }
long long grown_cap(long long cap) { return cap * 4; }

// The operator's launches: AG_THREADS threads per CTA, one CTA per `per_block` work items, at most `per_sm` CTAs per SM (0: as
// many as the occupancy calculator fits with opts.smem bytes of dynamic shared memory).  bind(grid) runs first and sets
// what depends on the grid in the caller's objects that `args` refer to.  Profiled launches are the scans, reduces and
// COUNT(DISTINCT) inserts.
template <class... P, class Bind>
void launch_ag(dfgpu_ctx* ctx, void (*kern)(P...), const char* name, long long work_items, int per_block, int per_sm, const LaunchOpts& opts,
               Bind&& bind, const P&... args) {
  if (per_sm == 0) {
    DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, AG_THREADS, opts.smem));
    per_sm = std::max(per_sm, 1);
  }
  const int grid = grid_for(ctx, work_items, per_block, per_sm);
  bind(grid);
  launch(ctx, name, kern, grid, AG_THREADS, opts, args...);
}
// A launch whose arguments do not depend on the grid.
template <class P>
void launch_kernel(dfgpu_ctx* ctx, void (*kern)(P), const char* name, const P& p, long long work_items, int per_block, int per_sm,
                   const LaunchOpts& opts = {}) {
  launch_ag(ctx, kern, name, work_items, per_block, per_sm, opts, [](int) {}, p);
}

// A kernel instantiation and its trace name.  FRONT scan kernels route rows through the shared-memory front table.
template <class... P>
struct Kernel {
  void (*fn)(P...);
  const char* name;
  bool front = false;
};
using ScanKernel = Kernel<AggParams>;

template <int DEPTH>
ScanKernel hash_agg_kernel(bool front) {
  static const std::string with_front = "k_hash_agg<" + depth_arg(DEPTH) + ", true, false>";
  static const std::string without = "k_hash_agg<" + depth_arg(DEPTH) + ", false, false>";
  if (front) return {k_hash_agg<DEPTH, true, false>, with_front.c_str(), true};
  return {k_hash_agg<DEPTH, false, false>, without.c_str(), false};
}
template <int M>
ScanKernel lean_kernel_m(int mt) {
  static const std::string name[3] = {"k_hash_agg_lean<" + std::to_string(M) + ", " + std::to_string(int(MT_F64)) + ">",
                                      "k_hash_agg_lean<" + std::to_string(M) + ", " + std::to_string(int(MT_I)) + ">",
                                      "k_hash_agg_lean<" + std::to_string(M) + ", " + std::to_string(int(MT_U)) + ">"};
  if (mt == MT_F64) return {k_hash_agg_lean<M, MT_F64>, name[0].c_str(), false};
  if (mt == MT_I) return {k_hash_agg_lean<M, MT_I>, name[1].c_str(), false};
  return {k_hash_agg_lean<M, MT_U>, name[2].c_str(), false};
}
ScanKernel lean_kernel(int mask, int mt) {
  switch (mask) {
#define DF_LEAN(M) case M: return lean_kernel_m<M>(mt);
    DF_LEAN(1) DF_LEAN(2) DF_LEAN(3) DF_LEAN(4) DF_LEAN(5) DF_LEAN(6) DF_LEAN(7) DF_LEAN(8)
    DF_LEAN(9) DF_LEAN(10) DF_LEAN(11) DF_LEAN(12) DF_LEAN(13) DF_LEAN(14) DF_LEAN(15)
#undef DF_LEAN
    default: fail(DFGPU_ERR_INTERNAL, "lean kernel: bad aggregate mask");
  }
}
template <int DEPTH, bool NULLS = false>
Kernel<AggParams> reduce_kernel() {
  static const std::string name = "k_reduce<" + depth_arg(DEPTH) + (NULLS ? ", true>" : ", false>");
  return {k_reduce<DEPTH, NULLS>, name.c_str()};
}

// groups x (1 + naggs) sectors is what the SoA layout keeps hot in L2; beyond this many bytes the
// table is built AoS (one sector per group).  H100 L2 = 50 MB, shared with the streaming input.
constexpr long long AG_SOA_L2_BUDGET = 24ll << 20;

// Cardinality estimate from a prefix sample: `d` distinct keys among the first `s` rows.  Under a
// uniform model E[d] = G (1 - exp(-s / G)); solved for G by bisection and capped by the rows of the
// batch.  Skewed keys make this an under-estimate, which the growth path absorbs.
long long estimate_groups(long long d, long long s, long long total_rows) {
  if (d <= 0) return 0;
  if (double(d) >= 0.995 * double(s)) return total_rows;  // (almost) every sampled row was a new group
  double lo = double(d), hi = 1e13;
  for (int it = 0; it < 80; it++) {
    const double g = 0.5 * (lo + hi);
    const double e = g * -expm1(-double(s) / g);
    if (e < double(d)) lo = g; else hi = g;
  }
  const double g = 0.5 * (lo + hi);
  return g > double(total_rows) ? total_rows : (long long)g;
}

// Capacity for a table that holds `seen` distinct entries after the first `prefix_rows` rows of a batch of `batch_rows`:
// sized for the estimated total (*est), but halved while it exceeds what 1/8 of device memory holds at `slot_bytes` per
// slot; never below the current capacity `cur_cap`.
long long prefix_cap(const dfgpu_ctx* ctx, long long seen, long long prefix_rows, long long batch_rows, long long slot_bytes,
                     long long cur_cap, long long min_cap, long long* est = nullptr) {
  const long long e = std::max(estimate_groups(seen, prefix_rows, batch_rows), seen);
  if (est) *est = e;
  const long long afford = (long long)(ctx->device_mem_bytes / 8) / slot_bytes;
  long long want = table_cap(e, min_cap);
  while (want > cur_cap && want > afford) want >>= 1;
  return std::max(want, cur_cap);
}

void layout_shape(const std::vector<AggDesc>& descs, int naggs, int nkeys, bool line_mode, long long* lw, int* n_add, signed char* loc, int kw = 0) {
  *lw = 1;
  *n_add = 0;
  if (nkeys > 0 && (line_mode || kw > 0)) {  // wide keys: tag, kw key parts, then every accumulator, all in the line
    while (*lw < 1 + kw + naggs) *lw <<= 1;
    for (int a = 0; a < naggs; a++) loc[a] = (signed char)(1 + kw + a);
    return;
  }
  int nmm = 0;
  for (int a = 0; a < naggs; a++) {
    const bool mm = descs[size_t(a)].func == DFGPU_AGG_MIN || descs[size_t(a)].func == DFGPU_AGG_MAX;
    if (nkeys > 0 && mm) loc[a] = (signed char)(1 + nmm++);
    else loc[a] = (signed char)~((*n_add)++);
  }
  while (*lw < 1 + nmm) *lw <<= 1;
}
// Bytes the scan keeps hot in L2 with the hybrid layout: one sector (or lw/4) per group for the line, and
// every sector of each additive array once a quarter of its slots is in use.  Beyond the budget the table
// is built in "line" form (one sector per group, whatever the number of aggregates).
bool want_aos(long long groups, const std::vector<AggDesc>& descs, int naggs) {
  static const char* force = getenv("DFGPU_AGG_LAYOUT");  // A/B switch: "line" | "hybrid"
  if (force && std::string(force) == "line") return true;
  if (force && std::string(force) == "hybrid") return false;
  long long lw;
  int n_add;
  signed char loc[kMaxAggs];
  layout_shape(descs, naggs, 1, false, &lw, &n_add, loc);
  const long long cap = table_cap(groups, AG_MIN_CAP);
  const long long line_hot = std::min(cap * 8 * lw, groups * std::max<long long>(32, 8 * lw));
  const long long arr_hot = std::min(cap * 8, groups * 32);
  return line_hot + n_add * arr_hot > AG_SOA_L2_BUDGET;
}

TableLayout table_alloc(dfgpu_ctx* ctx, int naggs, int nkeys, const std::vector<AggDesc>& descs, long long cap, bool aos, int kw = 0) {
  InitParams ip;
  memset(&ip, 0, sizeof(ip));
  int n_add = 0;
  ip.t.set_cap(cap);
  layout_shape(descs, naggs, nkeys, aos, &ip.t.lw, &n_add, ip.t.loc, kw);
  const size_t line_words = size_t(cap + 1) * size_t(ip.t.lw);
  const size_t words = line_words + size_t(n_add) * size_t(cap + 1);
  ip.t.base = (unsigned long long*)ctx->alloc(words * 8);  // >= 256-byte aligned: lines of up to 32 bytes never straddle a sector
  ip.t.add = ip.t.base + line_words;
  ip.t.astride = cap + 1;
  ip.nslots = cap + 1;
  ip.naggs = naggs;
  for (int a = 0; a < naggs; a++) ip.ident[a] = agg_identity(descs[size_t(a)].func);
  launch_kernel(ctx, k_table_init, "k_table_init", ip, ip.nslots, 256 * 4, 16);
  return ip.t;
}

// counter slots [0, CTR_NONNULL) -> host8 (synchronises the stream)
void read_counters(dfgpu_aggstate* st, unsigned long long* host8) { read_words(st->ctx, st->d_counters, CTR_NONNULL * 8, host8); }
// one counter slot (synchronises the stream)
unsigned long long read_counter(dfgpu_aggstate* st, int slot) { return read_word(st->ctx, st->d_counters + slot); }

// Raw compaction (k_compact, raw = 1) of table t: the occupied slots as (packed key, accumulators) entries.  Entry i's
// key goes to keys[i * stride] and accumulator a to vals[a * val_step + i * stride] (stride 0 = 1); the number of
// entries to counter CTR_COMPACT.
void compact_raw(dfgpu_aggstate* st, const TableLayout& t, int sentinel_used, const unsigned long long* sentinel_flag, unsigned long long* keys,
                 unsigned long long* vals, size_t val_step, long long stride) {
  dfgpu_ctx* ctx = st->ctx;
  CompactParams cp;
  memset(&cp, 0, sizeof(cp));
  cp.t = t;
  cp.sentinel_used = sentinel_used;
  cp.sentinel_flag = sentinel_flag;
  cp.nkeys = st->nkeys;
  cp.naggs = st->naggs;
  cp.raw = 1;
  cp.raw_stride = stride;
  cp.out_keys[0] = keys;
  for (int a = 0; a < st->naggs; a++) {
    cp.aggs[a] = st->descs[size_t(a)];
    cp.out_vals[a] = vals + size_t(a) * val_step;
  }
  DF_CUDA(cudaMemsetAsync(st->d_counters + CTR_COMPACT, 0, 8, ctx->stream));
  cp.counter = st->d_counters + CTR_COMPACT;
  launch_kernel(ctx, k_compact, "k_compact", cp, t.cap + 1, 256, 8);
}

// Grow the table to new_cap.  Wide tables move their slots (k_wide_move: every entry is distinct); the others are
// raw-compacted and merged into the new table (k_merge), which may also change their layout.
void table_grow(dfgpu_aggstate* st, long long new_cap) {
  dfgpu_ctx* ctx = st->ctx;
  const bool aos = st->aos || want_aos(std::max(st->ngroups, new_cap / 8), st->descs, st->naggs);
  TableLayout nt = table_alloc(ctx, st->naggs, st->nkeys, st->descs, new_cap, aos, st->wide ? st->nkeys : 0);
  DevBufs tmp(ctx);
  if (st->wide) {
    WideMoveParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.from = st->t;
    mp.to = nt;
    mp.kw = st->nkeys;
    mp.naggs = st->naggs;
    mp.error = st->d_counters + CTR_ERROR;
    launch_kernel(ctx, k_wide_move, "k_wide_move", mp, st->t.cap, 256, 8);
  } else {
    const size_t cnt = size_t(st->ngroups + 1);
    unsigned long long* ck = tmp.alloc(cnt * 8);
    unsigned long long* cv = tmp.alloc(cnt * 8 * size_t(st->naggs > 0 ? st->naggs : 1));
    compact_raw(st, st->t, st->sentinel_used, nullptr, ck, cv, cnt, 0);
    MergeParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.in_keys = ck;
    for (int a = 0; a < st->naggs; a++) {
      mp.in_vals[a] = cv + size_t(a) * cnt;
      mp.aggs[a] = st->descs[size_t(a)];
    }
    mp.n = st->ngroups + (st->sentinel_used ? 1 : 0);
    mp.t = nt;
    mp.naggs = st->naggs;
    DF_CUDA(cudaMemsetAsync(st->d_counters + CTR_GROUPS, 0, 8, ctx->stream));  // ngroups is recounted by the merge
    mp.counters = st->d_counters;
    if (mp.n > 0) launch_kernel(ctx, k_merge, "k_merge", mp, mp.n, 256, 8);
  }
  if (read_counter(st, CTR_ERROR) == 2) {
    ctx->free(nt.base);
    fail(DFGPU_ERR_INTERNAL, "table growth could not place a group");
  }
  ctx->free(st->t.base);
  st->t = nt;
  st->aos = aos;
}

}  // namespace

extern "C" int dfgpu_aggregate_create(dfgpu_ctx* ctx, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                                      const dfgpu_agg* aggs, int naggs, int64_t expected_groups, dfgpu_aggstate** out) {
  return guarded([&] {
    if (!ctx || !out) fail(DFGPU_ERR_GENERAL, "dfgpu_aggregate_create: null argument");
    if (nkeys < 0 || nkeys > kMaxKeys) fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than " + std::to_string(kMaxKeys) + " GROUP BY expressions");
    if (naggs < 1) fail(DFGPU_ERR_GENERAL, "aggregate needs at least one aggregate expression");
    if (naggs > kMaxAggs) fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than " + std::to_string(kMaxAggs) + " aggregate expressions");
    ctx->use();
    auto st = std::make_unique<dfgpu_aggstate>();
    st->ctx = ctx;
    st->nkeys = nkeys;
    st->naggs = naggs;
    st->expected = expected_groups;
    for (int k = 0; k < nkeys; k++) {
      st->key_progs.emplace_back(keys[k], keys[k] + key_len[k]);
      st->own_literals(st->key_progs.back());
    }
    std::vector<int> dist_user;  // user aggregates that are COUNT(DISTINCT)
    for (int a = 0; a < naggs; a++) {
      // compile_expr accepts min/max/count/sum (expression.rs:98-107), this engine also COUNT(DISTINCT) and AVG;
      // anything else is General("Unsupported aggregate function ...")
      if (aggs[a].func < DFGPU_AGG_MIN || aggs[a].func > DFGPU_AGG_AVG)
        fail(DFGPU_ERR_GENERAL, "Unsupported aggregate function '" + std::to_string(aggs[a].func) + "'");
      std::vector<dfgpu_insn> prog(aggs[a].arg, aggs[a].arg + aggs[a].arg_len);
      st->own_literals(prog);
      st->out_is_avg.push_back(aggs[a].func == DFGPU_AGG_AVG ? 1 : 0);
      if (aggs[a].func == DFGPU_AGG_AVG) {
        if (aggs[a].out_dtype != 0 && aggs[a].out_dtype != DFGPU_FLOAT64)
          fail(DFGPU_ERR_EXECUTION, "unexpected type when creating array from aggregate map");
        // two scan words of its own, never shared with a SUM(x) / COUNT(x) of the query: under GROUP BY those read
        // null rows, AVG skips them
        st->out_word.push_back(int(st->funcs.size()));
        for (int f : {AGG_AVG_SUM, int(DFGPU_AGG_COUNT)}) {
          st->arg_progs.push_back(prog);
          st->funcs.push_back(f);
          st->out_dtypes.push_back(f == AGG_AVG_SUM ? DFGPU_FLOAT64 : DFGPU_UINT64);
        }
        continue;
      }
      if (aggs[a].func == DFGPU_AGG_COUNT_DISTINCT) {
        if (aggs[a].out_dtype != 0 && aggs[a].out_dtype != DFGPU_UINT64)
          fail(DFGPU_ERR_EXECUTION, "unexpected type when creating array from aggregate map");
        // COUNT(DISTINCT) over the same argument program share one set
        int s = 0;
        while (s < int(st->dist_progs.size()) && !(st->dist_progs[size_t(s)].size() == prog.size() &&
                                                   memcmp(st->dist_progs[size_t(s)].data(), prog.data(), prog.size() * sizeof(dfgpu_insn)) == 0))
          s++;
        if (s == int(st->dist_progs.size())) st->dist_progs.push_back(prog);
        st->dist_set.push_back(s);
        dist_user.push_back(a);
        st->out_word.push_back(-1);
        continue;
      }
      st->out_word.push_back(int(st->funcs.size()));
      st->arg_progs.push_back(prog);
      st->funcs.push_back(aggs[a].func);
      st->out_dtypes.push_back(aggs[a].out_dtype);
    }
    // the pair exchange across ranks is not built: refuse where the communicator is known (and again at finish, for
    // one attached after create)
    if (!dist_user.empty() && ctx->world > 1) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) with a communicator attached");
    st->nscan = int(st->funcs.size());
    st->naggs = st->nscan + int(dist_user.size());  // table words
    if (st->naggs > kMaxAggs)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "aggregates that need more than " + std::to_string(kMaxAggs) + " accumulator words (each AVG takes two)");
    for (size_t j = 0; j < dist_user.size(); j++) st->out_word[size_t(dist_user[j])] = st->nscan + int(j);
    st->d_counters = (unsigned long long*)ctx->alloc(CTR_SLOTS * 8);
    DF_CUDA(cudaMemsetAsync(st->d_counters, 0, CTR_SLOTS * 8, ctx->stream));
    if (!dist_user.empty()) {
      st->d_dctr = (unsigned long long*)ctx->alloc(DCTR_SLOTS * 8);
      DF_CUDA(cudaMemsetAsync(st->d_dctr, 0, DCTR_SLOTS * 8, ctx->stream));
    }
    *out = st.release();
  });
}

extern "C" int dfgpu_aggregate_set_predicate(dfgpu_aggstate* st, const dfgpu_insn* pred, int pred_len) {
  return guarded([&] {
    if (!st || (pred_len > 0 && !pred)) fail(DFGPU_ERR_GENERAL, "dfgpu_aggregate_set_predicate: null argument");
    if (st->rows_seen > 0 || st->typed) fail(DFGPU_ERR_GENERAL, "the predicate must be set before the first batch");
    st->pred_prog.assign(pred, pred + (pred_len > 0 ? pred_len : 0));
    st->own_literals(st->pred_prog);  // replayed on every update
  });
}

namespace {
void agg_update(dfgpu_aggstate* st, const dfgpu_batch* batch);
}

extern "C" int dfgpu_aggregate_update(dfgpu_aggstate* st, const dfgpu_batch* batch) {
  return guarded([&] {
    if (!st || !batch) fail(DFGPU_ERR_GENERAL, "dfgpu_aggregate_update: null argument");
    agg_update(st, batch);
  });
}

// One big host RecordBatch: row-range chunks, every H2D copy queued up front on the copy-in stream, the
// scan of chunk c waits only for chunk c's copies — PCIe and the scan kernel overlap, and the table is
// the only state carried from chunk to chunk (update_accumulators is per row: aggregate.rs:548-612).
extern "C" int dfgpu_aggregate_update_host(dfgpu_aggstate* st, const dfgpu_col* cols, int ncols, int64_t chunk_rows) {
  return guarded([&] {
    if (!st || (ncols > 0 && !cols)) fail(DFGPU_ERR_GENERAL, "dfgpu_aggregate_update_host: null argument");
    dfgpu_ctx* ctx = st->ctx;
    ctx->use();
    const int64_t n = ncols > 0 ? cols[0].len : 0;
    bool streamable = n > 0;
    for (int i = 0; i < ncols; i++) {
      if (cols[i].len != n) fail(DFGPU_ERR_GENERAL, "all columns of a RecordBatch must have the same length");
      streamable = streamable && dtype_width(cols[i].dtype) > 0 && !cols[i].validity && cols[i].values;
    }
    if (chunk_rows <= 0) chunk_rows = 8ll << 20;
    chunk_rows = (chunk_rows + 1023) / 1024 * 1024;  // chunks start on even, 16-byte aligned rows of every column
    if (!streamable || n <= chunk_rows) {
      // small, nullable or variable-width batches: plain upload (Utf8 / validity handling lives there)
      dfgpu_batch* b = nullptr;
      int rc = dfgpu_batch_upload(ctx, cols, ncols, &b);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      struct G { dfgpu_batch* b; ~G() { dfgpu_batch_free(b); } } g{b};
      agg_update(st, b);
      return;
    }
    const int nchunks = int((n + chunk_rows - 1) / chunk_rows);
    DevBufs dev(ctx);  // freed after the Cleanup below has drained both streams
    std::vector<cudaEvent_t> evs(size_t(nchunks), nullptr);
    struct Cleanup {
      dfgpu_ctx* c; std::vector<cudaEvent_t>* e;
      ~Cleanup() {
        cudaStreamSynchronize(c->stream_in);
        cudaStreamSynchronize(c->stream);
        for (cudaEvent_t x : *e) if (x) cudaEventDestroy(x);
      }
    } cleanup{ctx, &evs};
    for (int i = 0; i < ncols; i++) dev.alloc<void>(size_t(n) * size_t(dtype_width(cols[i].dtype)));
    // the device buffers may have been used on ctx->stream before (cached blocks): order the copies after it
    cudaEvent_t ready;
    DF_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    DF_CUDA(cudaEventRecord(ready, ctx->stream));
    DF_CUDA(cudaStreamWaitEvent(ctx->stream_in, ready, 0));
    DF_CUDA(cudaEventDestroy(ready));
    for (int c = 0; c < nchunks; c++) {
      const int64_t lo = int64_t(c) * chunk_rows, cnt = std::min<int64_t>(chunk_rows, n - lo);
      for (int i = 0; i < ncols; i++) {
        const size_t w = size_t(dtype_width(cols[i].dtype));
        DF_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(dev.blocks[size_t(i)]) + size_t(lo) * w,
                                static_cast<const uint8_t*>(cols[i].values) + size_t(cols[i].offset + lo) * w, size_t(cnt) * w,
                                cudaMemcpyHostToDevice, ctx->stream_in));
      }
      DF_CUDA(cudaEventCreateWithFlags(&evs[size_t(c)], cudaEventDisableTiming));
      DF_CUDA(cudaEventRecord(evs[size_t(c)], ctx->stream_in));
    }
    for (int c = 0; c < nchunks; c++) {
      const int64_t lo = int64_t(c) * chunk_rows, cnt = std::min<int64_t>(chunk_rows, n - lo);
      DF_CUDA(cudaStreamWaitEvent(ctx->stream, evs[size_t(c)], 0));
      dfgpu_batch view;  // borrows the chunk's slices of the device buffers
      view.ctx = ctx;
      view.owns = false;
      view.nrows = cnt;
      for (int i = 0; i < ncols; i++) {
        DevColumn d;
        d.dtype = cols[i].dtype;
        const size_t w = size_t(dtype_width(cols[i].dtype));
        d.values = static_cast<uint8_t*>(dev.blocks[size_t(i)]) + size_t(lo) * w;
        d.values_bytes = size_t(cnt) * w;
        view.cols.push_back(d);
      }
      agg_update(st, &view);
    }
  });
}

namespace {

// The batch's column that a key program reads when the program is one plain Utf8 column, else null.
const DevColumn* plain_utf8_col(const std::vector<dfgpu_insn>& kp, const dfgpu_batch* batch) {
  if (kp.size() != 1 || kp[0].op != DFGPU_OP_COL || kp[0].col < 0 || size_t(kp[0].col) >= batch->cols.size()) return nullptr;
  const DevColumn& c = batch->cols[size_t(kp[0].col)];
  return c.dtype == DFGPU_UTF8 ? &c : nullptr;
}

// Keep a copy of a batch's Utf8 key column: a group refers to its string as (source << UTF8_SRC_SHIFT | row), and the
// strings are gathered at finish.  Returns the column's source index; upload_utf8_srcs makes it visible to kernels.
unsigned long long retain_utf8(dfgpu_aggstate* st, const DevColumn& c, long long nrows) {
  dfgpu_ctx* ctx = st->ctx;
  const size_t ob = size_t(nrows + 1) * 4, vb = c.values_bytes ? c.values_bytes : 1;
  int* off = (int*)ctx->alloc(ob);
  unsigned char* bytes = (unsigned char*)ctx->alloc(vb);
  DF_CUDA(cudaMemcpyAsync(off, c.offsets, ob, cudaMemcpyDeviceToDevice, ctx->stream));
  if (c.values_bytes) DF_CUDA(cudaMemcpyAsync(bytes, c.values, c.values_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  st->utf8_owned.push_back(off);
  st->utf8_owned.push_back(bytes);
  st->utf8_srcs.push_back(Utf8Source{off, bytes});
  return st->utf8_srcs.size() - 1;
}
void upload_utf8_srcs(dfgpu_aggstate* st) {
  dfgpu_ctx* ctx = st->ctx;
  ctx->free(st->d_utf8_srcs);
  st->d_utf8_srcs = (Utf8Source*)ctx->alloc(st->utf8_srcs.size() * sizeof(Utf8Source));
  DF_CUDA(cudaMemcpyAsync(st->d_utf8_srcs, st->utf8_srcs.data(), st->utf8_srcs.size() * sizeof(Utf8Source), cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));  // utf8_srcs may reallocate on the next batch
}

// Pack the key parts into one 64-bit word, the last key in the low bits; a Utf8 part (wide keys) takes a whole word.
// Returns whether the keys need the wide table: more than 64 key bits, or a Utf8 part next to other parts.
bool pack_keys(dfgpu_aggstate* st) {
  const size_t nk = size_t(st->nkeys);
  st->key_shift.assign(nk, 0);
  st->key_mask.assign(nk, 0);
  st->key_is_utf8.assign(nk, 0);
  int bits = 0;
  bool any_utf8 = false;
  for (int k = st->nkeys - 1; k >= 0; k--) {
    const bool u = st->key_dtypes[size_t(k)] == DFGPU_UTF8;
    const int w = u ? 64 : dtype_width(st->key_dtypes[size_t(k)]) * 8;
    st->key_shift[size_t(k)] = bits > 63 ? 0 : bits;
    st->key_mask[size_t(k)] = w == 64 ? ~0ull : ((1ull << w) - 1ull);
    st->key_is_utf8[size_t(k)] = u ? 1 : 0;
    any_utf8 = any_utf8 || u;
    bits += w;
  }
  if (st->nkeys == 1) st->key_mask[0] = ~0ull;  // single key: keep the sign-extended 64-bit value
  return bits > 64 || any_utf8;
}

// The programs of one batch: the fused WHERE (program 0, FilterRelation under the aggregate, context.rs:126-139), the
// GROUP BY keys, the distinct aggregate arguments and, for a single Utf8 key, the hidden representative.  A Utf8 key
// column is read as a column of its 64-bit string hashes.
struct BatchPrograms {
  ProgramBuilder pb;
  DevBufs hashes;  // the string hashes of the Utf8 key columns
  int has_pred = 0;
  std::vector<int> key_dtypes;  // a Utf8 part of a wide key is Utf8, the single Utf8 key UInt64 (its hash)
  std::vector<AggDesc> descs;
  std::vector<int> agg_arg;
  int nargs = 0;
  const DevColumn* ukey = nullptr;  // the single Utf8 key column (grouped by hash, then verified)
  const unsigned long long* ukey_hash = nullptr;
  std::vector<const DevColumn*> key_utf8;  // per key part (not the single Utf8 key): its Utf8 column, or null
  // COUNT(DISTINCT): the WHERE clause, the keys and the argument of each set, for k_distinct_insert
  ProgramBuilder dpb;
  std::vector<int> dist_dtypes;
  BatchPrograms(const dfgpu_batch* batch, dfgpu_ctx* ctx) : pb(batch), hashes(ctx), dpb(batch) {}
};

// Compile a batch's programs and type its aggregates.  The single Utf8 key column is retained here, because the
// representative program refers to the source index it is retained under.
void compile_batch(dfgpu_aggstate* st, const dfgpu_batch* batch, BatchPrograms& bp) {
  dfgpu_ctx* ctx = st->ctx;
  ProgramBuilder& pb = bp.pb;
  bp.has_pred = st->pred_prog.empty() ? 0 : 1;
  if (bp.has_pred) {
    const int pi = pb.add(st->pred_prog.data(), int(st->pred_prog.size()), "filter expression");
    if (pb.out_dtype(pi) != DFGPU_BOOL) fail(DFGPU_ERR_EXECUTION, "Filter expression did not evaluate to boolean");  // filter.rs:62-67
  }
  auto hash_key = [&](const DevColumn& c) {
    unsigned long long* h = bp.hashes.alloc(size_t(batch->nrows > 0 ? batch->nrows : 1) * 8);
    utf8_hash(ctx, c, batch->nrows, h);
    pb.add_synthetic_column(h, DFGPU_UINT64);
    return h;
  };
  const bool distinct = !st->dist_progs.empty();
  bp.ukey = st->nkeys == 1 ? plain_utf8_col(st->key_progs[0], batch) : nullptr;
  if (bp.ukey && distinct) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) with a Utf8 GROUP BY key");
  if (bp.ukey) {
    if (st->typed && !st->utf8_key) fail(DFGPU_ERR_GENERAL, "GROUP BY key types changed between batches");
    if (!st->typed && st->naggs >= kMaxAggs) fail(DFGPU_ERR_NOT_IMPLEMENTED, "Utf8 GROUP BY key with " + std::to_string(kMaxAggs) + " aggregates");
    if (st->utf8_srcs.size() >= (1u << 20)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than 2^20 batches with a Utf8 GROUP BY key");
    bp.ukey_hash = hash_key(*bp.ukey);
    bp.key_dtypes.push_back(DFGPU_UINT64);
  } else {
    for (int k = 0; k < st->nkeys; k++) {  // key parts: integer expressions and plain Utf8 columns
      const auto& kp = st->key_progs[size_t(k)];
      const DevColumn* uc = plain_utf8_col(kp, batch);
      bp.key_utf8.push_back(uc);
      if (uc && distinct) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) with a Utf8 GROUP BY key part");
      if (uc) {
        hash_key(*uc);
        bp.key_dtypes.push_back(DFGPU_UTF8);
        continue;
      }
      const int dt = pb.out_dtype(pb.add(kp.data(), int(kp.size()), "GROUP BY expression"));
      if (dt == DFGPU_UTF8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "Utf8 GROUP BY keys must be plain columns");
      if (!is_int(dt)) fail(DFGPU_ERR_EXECUTION, "Unsupported GROUP BY data type");  // aggregate.rs:848-850
      bp.key_dtypes.push_back(dt);
    }
  }
  const int user_aggs = int(st->funcs.size());  // the hidden representative is appended below
  bp.agg_arg.assign(size_t(user_aggs), 0);
  for (int a = 0; a < user_aggs; a++) {
    // identical argument expressions are compiled (and evaluated) once
    int same = -1;
    for (int b = 0; b < a && same < 0; b++) {
      const auto &x = st->arg_progs[size_t(a)], &y = st->arg_progs[size_t(b)];
      if (x.size() == y.size() && memcmp(x.data(), y.data(), x.size() * sizeof(dfgpu_insn)) == 0) same = b;
    }
    int pi;
    if (same >= 0) {
      bp.agg_arg[size_t(a)] = bp.agg_arg[size_t(same)];
      pi = bp.has_pred + st->nkeys + bp.agg_arg[size_t(a)];
    } else {
      pi = pb.add(st->arg_progs[size_t(a)].data(), int(st->arg_progs[size_t(a)].size()), "aggregate argument");
      bp.agg_arg[size_t(a)] = bp.nargs++;
    }
    int dt = pb.out_dtype(pi);
    if (!is_numeric(dt)) fail(DFGPU_ERR_EXECUTION, std::string("Unsupported data type for aggregate: ") + dtype_name(dt));
    AggDesc d;
    d.func = uint8_t(st->funcs[size_t(a)]);
    d.mtype = mtype_of(dt);
    d.dtype = uint8_t(dt);
    int want = d.func == DFGPU_AGG_COUNT ? DFGPU_UINT64 : (d.func == AGG_AVG_SUM ? DFGPU_FLOAT64 : dt);
    int odt = st->out_dtypes[size_t(a)];
    if (odt == 0) odt = want;
    if (odt != want)  // the reference would hit "unexpected type when creating array from aggregate map" (aggregate.rs:683-695)
      fail(DFGPU_ERR_EXECUTION, "unexpected type when creating array from aggregate map");
    d.out_dtype = uint8_t(odt);
    bp.descs.push_back(d);
  }
  if (distinct) {
    // the words COUNT(DISTINCT) counts into at finish: a COUNT for growth, exchange and compaction
    for (size_t j = 0; j < st->dist_set.size(); j++) bp.descs.push_back(AggDesc{DFGPU_AGG_COUNT, MT_U, DFGPU_UINT64, DFGPU_UINT64});
    if (bp.has_pred) bp.dpb.add(st->pred_prog.data(), int(st->pred_prog.size()), "filter expression");
    for (int k = 0; k < st->nkeys; k++) bp.dpb.add(st->key_progs[size_t(k)].data(), int(st->key_progs[size_t(k)].size()), "GROUP BY expression");
    for (const auto& prog : st->dist_progs) {
      const int dt = bp.dpb.out_dtype(bp.dpb.add(prog.data(), int(prog.size()), "aggregate argument"));
      if (dt == DFGPU_UTF8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) of a Utf8 argument");
      if (!is_numeric(dt)) fail(DFGPU_ERR_EXECUTION, std::string("Unsupported data type for aggregate: ") + dtype_name(dt));
      bp.dist_dtypes.push_back(dt);
    }
  }
  if (bp.ukey) {
    // hidden accumulator: MIN(source << 40 | row)
    pb.add_rowid_plus((unsigned long long)st->utf8_srcs.size() << UTF8_SRC_SHIFT);
    bp.agg_arg.push_back(bp.nargs++);
    bp.descs.push_back(AggDesc{DFGPU_AGG_MIN, MT_U, DFGPU_UINT64, DFGPU_UINT64});
    if (!st->typed) {
      st->utf8_key = true;
      st->naggs += 1;
    }
    retain_utf8(st, *bp.ukey, batch->nrows);
    upload_utf8_srcs(st);
  }
  pb.eval_utf8_predicates(ctx);
  bp.dpb.eval_utf8_predicates(ctx);
}

// Whether programs [has_pred] + nkeys keys + nargs arguments of `pb` fit the interpreter-free PlainSrc: at most 4 column
// slots, all 4/8-byte, null-free and 16-byte aligned, every key and argument a plain column and the WHERE clause, if
// any, a comparison chain.  If so, *out describes them.
bool plain_spec(const ProgramBuilder& pb, const ProgramSet& ps, int has_pred, int nkeys, int nargs, PlainSpec* out) {
  PlainSpec sp;
  memset(&sp, 0, sizeof(sp));
  bool ok = !ps.has_nulls && ps.ncols <= 4;
  for (int c = 0; ok && c < ps.ncols; c++)
    ok = is_numeric4or8(ps.cols[c].dtype) && (reinterpret_cast<uintptr_t>(ps.cols[c].ptr) & 15) == 0;
  for (int k = 0; ok && k < nkeys; k++) {
    ok = pb.prog(has_pred + k).leaf.kind == 1;
    sp.key_slot[k] = pb.prog(has_pred + k).leaf.a;
  }
  for (int g = 0; ok && g < nargs; g++) {
    ok = pb.prog(has_pred + nkeys + g).leaf.kind == 1;
    sp.arg_slot[g] = pb.prog(has_pred + nkeys + g).leaf.a;
  }
  if (ok && has_pred) {
    sp.pred = pb.prog(0).chain;
    ok = sp.pred.nterms > 0;
  }
  if (ok) *out = sp;
  return ok;
}

SetView set_alloc(dfgpu_ctx* ctx, long long cap);

// The first batch types the operator: key packing, table form and capacity.  Later batches must bring the same types.
void type_batch(dfgpu_aggstate* st, const BatchPrograms& bp) {
  if (st->typed) {
    if (bp.key_dtypes != st->key_dtypes) fail(DFGPU_ERR_GENERAL, "GROUP BY key types changed between batches");
    for (int a = 0; a < st->naggs; a++)
      if (bp.descs[size_t(a)].dtype != st->descs[size_t(a)].dtype) fail(DFGPU_ERR_GENERAL, "aggregate argument types changed between batches");
    if (bp.dist_dtypes != st->dist_dtypes) fail(DFGPU_ERR_GENERAL, "aggregate argument types changed between batches");
    return;
  }
  st->key_dtypes = bp.key_dtypes;
  st->descs = bp.descs;
  st->wide = pack_keys(st);
  if (st->wide && !st->dist_progs.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) with GROUP BY keys wider than 64 bits");
  st->dist_dtypes = bp.dist_dtypes;
  st->typed = true;
  const long long cap = st->nkeys == 0 ? 0 : table_cap(st->expected, AG_MIN_CAP);
  st->aos = st->wide || (st->nkeys > 0 && want_aos(st->expected, st->descs, st->naggs));
  st->t = table_alloc(st->ctx, st->naggs, st->nkeys, st->descs, cap, st->aos, st->wide ? st->nkeys : 0);
  for (size_t s = 0; s < st->dist_progs.size(); s++) st->sets.push_back(set_alloc(st->ctx, table_cap(st->expected, AG_SET_MIN_CAP)));
}

// ---- COUNT(DISTINCT) ----------------------------------------------------------------------------------------
SetView set_alloc(dfgpu_ctx* ctx, long long cap) {
  SetView set;
  set.set_cap(cap);
  set.slots = (unsigned long long*)ctx->alloc(size_t(cap) * 16);
  DF_CUDA(cudaMemsetAsync(set.slots, 0xff, size_t(cap) * 16, ctx->stream));  // every word EMPTY_KEY
  return set;
}

// DCTR_* slots -> host (synchronises the stream)
void read_dctr(dfgpu_aggstate* st, unsigned long long* host) { read_words(st->ctx, st->d_dctr, DCTR_SLOTS * 8, host); }

// Grow set s to new_cap by re-inserting its pairs (their number does not change).
void set_grow(dfgpu_aggstate* st, int s, long long new_cap) {
  dfgpu_ctx* ctx = st->ctx;
  SetMoveParams mp;
  mp.from = st->sets[size_t(s)];
  mp.to = set_alloc(ctx, new_cap);
  mp.error = st->d_dctr + DCTR_ERROR;
  launch_kernel(ctx, k_set_move, "k_set_move", mp, mp.from.cap, 256 * 4, 8);
  unsigned long long c[DCTR_SLOTS];
  read_dctr(st, c);
  if (c[DCTR_ERROR] == 2) fail(DFGPU_ERR_INTERNAL, "COUNT(DISTINCT) set growth could not place a pair");
  ctx->free(mp.from.slots);
  st->sets[size_t(s)] = mp.to;
}

// The parameters of a batch's COUNT(DISTINCT) insert, which puts the (group key, argument) pairs of the batch's rows into
// every set after the group scan of the same rows: its own program set (WHERE, keys, set arguments), the keys packed
// exactly as the scan packs them.  *plain: p.plain describes the programs for k_distinct_insert_plain.
AggParams plan_insert(const dfgpu_aggstate* st, const BatchPrograms& bp, bool* plain) {
  AggParams p;
  memset(&p, 0, sizeof(p));
  bp.dpb.finish(&p.ps);
  if (p.ps.max_depth > 8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "expression too deep (register stack depth > 8)");
  p.has_pred = bp.has_pred;
  p.nkeys = st->nkeys;
  p.nargs = int(st->dist_progs.size());
  for (int k = 0; k < st->nkeys; k++) {
    p.key_mask[k] = st->key_mask[size_t(k)];
    p.key_shift[k] = st->key_shift[size_t(k)];
  }
  p.counters = st->d_dctr;
  *plain = plain_spec(bp.dpb, p.ps, bp.has_pred, st->nkeys, p.nargs, &p.plain);
  return p;
}

// The insert kernel of one round.  Replays read a row list and the plain kernels start on an even row, so both take the
// interpreter.
Kernel<AggParams, SetParams> choose_insert(const AggParams& p, bool plain_ok) {
  const bool fn = has_fn(p.ps), plain = plain_ok && !p.row_list && (p.row_begin & 1) == 0;
  if (has_case(p.ps) && p.ps.has_nulls) return {k_distinct_insert<kCaseDepth, true>, "k_distinct_insert<kCaseDepth, true>"};
  if (has_case(p.ps)) return {k_distinct_insert<kCaseDepth, false>, "k_distinct_insert<kCaseDepth, false>"};
  if (fn && p.ps.has_nulls) return {k_distinct_insert<kFnDepth, true>, "k_distinct_insert<kFnDepth, true>"};
  if (fn) return {k_distinct_insert<kFnDepth, false>, "k_distinct_insert<kFnDepth, false>"};
  if (p.ps.has_nulls) return {k_distinct_insert<8, true>, "k_distinct_insert<8, true>"};
  if (plain && p.ps.ncols <= 2) return {k_distinct_insert_plain<2>, "k_distinct_insert_plain<2>"};
  if (plain) return {k_distinct_insert_plain<4>, "k_distinct_insert_plain<4>"};
  if (p.ps.max_depth <= 2) return {k_distinct_insert<2, false>, "k_distinct_insert<2, false>"};
  return {k_distinct_insert<8, false>, "k_distinct_insert<8, false>"};
}

// One round of the insert over the rows p describes, then the growth rule of the sets: each set that refused pairs at
// its fill limit, or went past it, grows x4; when rows were refused and no set grew, the probe limit refused them below
// the fill limit, and every set grows.  As for the group table (scan_round), that happens at most once per batch
// (*probe_grown): pairs whose hashes share their top bits share a home at every capacity.  Returns the number of rows
// refused.
long long insert_round(dfgpu_aggstate* st, AggParams& p, bool plain, bool* probe_grown) {
  const int nsets = int(st->dist_progs.size());
  const Kernel<AggParams, SetParams> k = choose_insert(p, plain);
  SetParams sp;
  memset(&sp, 0, sizeof(sp));
  for (int s = 0; s < nsets; s++) {
    sp.set[s] = st->sets[size_t(s)];
    sp.mt[s] = mtype_of(st->dist_dtypes[size_t(s)]);
  }
  // A warp reads the fill once per tile and adds its tile's pairs after it, so up to one tile per warp of the grid
  // (grid x AG_TILE pairs per set) is inserted past what the others read: the fill limit is lowered by that much,
  // which keeps every set at most half full.
  launch_ag(st->ctx, k.fn, k.name, p.row_list ? p.nlist : p.nrows, AG_TILE, 0, PROFILED, [&](int grid) {
    for (int s = 0; s < nsets; s++) sp.max_fill[s] = std::max<long long>(0, fill_limit(sp.set[s].cap) - (long long)grid * AG_TILE);
  }, p, sp);
  unsigned long long c[DCTR_SLOTS];
  read_dctr(st, c);
  if (c[DCTR_ERROR]) fail(DFGPU_ERR_ARROW, "DivideByZero");
  const long long novf = (long long)c[DCTR_OVERFLOW];
  bool grow[kMaxAggs], any = false;
  for (int s = 0; s < nsets; s++) {
    const long long n = (long long)c[DCTR_SET + 2 * s];
    grow[s] = (novf > 0 && n >= sp.max_fill[s]) || n > fill_limit(sp.set[s].cap);  // refused pairs at its fill limit, or past it
    any = any || grow[s];
  }
  if (novf > 0 && !any) {
    if (*probe_grown)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) pairs whose hashes share one home slot: more than the probe limit of " +
                                          std::to_string(AG_MAX_PROBE) + " pairs on one probe chain");
    *probe_grown = true;
  }
  for (int s = 0; s < nsets; s++)
    if (grow[s] || (novf > 0 && !any)) set_grow(st, s, grown_cap(sp.set[s].cap));
  return novf;
}

// GROUP BY at finish: add each set's pairs to the COUNT(DISTINCT) words of their groups.
void distinct_count(dfgpu_aggstate* st, const TableLayout& t, int sentinel_used) {
  dfgpu_ctx* ctx = st->ctx;
  DF_CUDA(cudaMemsetAsync(st->d_dctr + DCTR_ERROR, 0, 8, ctx->stream));
  for (size_t s = 0; s < st->dist_progs.size(); s++) {
    DistinctCountParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.set = st->sets[s];
    cp.marker = st->d_dctr + DCTR_SET + 2 * s + 1;
    cp.t = t;
    cp.sentinel_used = sentinel_used;
    for (size_t j = 0; j < st->dist_set.size(); j++)
      if (st->dist_set[j] == int(s)) cp.words[cp.nwords++] = st->nscan + int(j);
    cp.error = st->d_dctr + DCTR_ERROR;
    launch_kernel(ctx, k_distinct_count, "k_distinct_count", cp, cp.set.cap + 1, 256 * 4, 8);
  }
  unsigned long long c[DCTR_SLOTS];
  read_dctr(st, c);
  if (c[DCTR_ERROR]) fail(DFGPU_ERR_INTERNAL, "COUNT(DISTINCT) found a pair whose group is not in the table");
}

// No GROUP BY at finish: each COUNT(DISTINCT) is the number of pairs in its set.
void distinct_count_scalar(dfgpu_aggstate* st) {
  dfgpu_ctx* ctx = st->ctx;
  unsigned long long c[DCTR_SLOTS], n[kMaxAggs];
  read_dctr(st, c);
  for (size_t j = 0; j < st->dist_set.size(); j++) {
    const int s = st->dist_set[j];
    n[j] = c[DCTR_SET + 2 * s] + (c[DCTR_SET + 2 * s + 1] ? 1ull : 0ull);
    DF_CUDA(cudaMemcpyAsync(st->t.val(0, st->nscan + int(j)), &n[j], 8, cudaMemcpyHostToDevice, ctx->stream));
  }
  DF_CUDA(cudaStreamSynchronize(ctx->stream));  // `n` is a stack array
}

// No GROUP BY: one reduce over the batch.
void reduce_update(dfgpu_aggstate* st, const BatchPrograms& bp, AggParams& p) {
  dfgpu_ctx* ctx = st->ctx;
  p.t = st->t;
  if (p.naggs == 0) return;  // COUNT(DISTINCT) alone: nothing for the reduce kernels to do
  if (bp.has_pred) DF_CUDA(cudaMemsetAsync(st->d_counters + CTR_PASSED, 0, 8, ctx->stream));
  const int d = p.ps.max_depth;
  const bool fn = has_fn(p.ps);
  Kernel<AggParams> k{};
  if (p.ps.has_nulls) {
    st->saw_nulls = true;
    k = has_case(p.ps) ? reduce_kernel<kCaseDepth, true>() : fn ? reduce_kernel<kFnDepth, true>() : reduce_kernel<8, true>();
  } else {
    if (!bp.has_pred)
      for (int a = 0; a < st->naggs; a++) st->nonnull_host[size_t(a)] += p.nrows;
    // fast path: every distinct argument is a plain Float64 column
    bool plain = !bp.has_pred;
    ReduceF64Params rp;
    memset(&rp, 0, sizeof(rp));
    for (int g = 0; g < bp.nargs && plain; g++) {
      const Leaf& f = bp.pb.prog(g).leaf;
      plain = f.kind == 1 && f.dtype == DFGPU_FLOAT64 && (reinterpret_cast<uintptr_t>(p.ps.cols[f.a].ptr) & 15) == 0;
      if (plain) rp.col[g] = (const double*)p.ps.cols[f.a].ptr;
    }
    if (plain) {
      rp.ncols = bp.nargs;
      rp.nrows = p.nrows;
      rp.naggs = p.naggs;
      for (int a = 0; a < p.naggs; a++) { rp.aggs[a] = p.aggs[a]; rp.agg_arg[a] = p.agg_arg[a]; }
      rp.t = st->t;
      launch_kernel(ctx, k_reduce_f64, "k_reduce_f64", rp, p.nrows, 256 * 8, 8, PROFILED);
    } else if (has_case(p.ps)) k = reduce_kernel<kCaseDepth>();
    else if (fn) k = reduce_kernel<kFnDepth>();
    else if (d <= 1) k = reduce_kernel<1>();
    else if (d <= 2) k = reduce_kernel<2>();
    else if (d <= 4) k = reduce_kernel<4>();
    else k = reduce_kernel<8>();
  }
  if (k.fn) launch_kernel(ctx, k.fn, k.name, p, p.nrows, RD_TILE, 0, PROFILED);
  unsigned long long c[CTR_NONNULL];
  read_counters(st, c);
  if (c[CTR_ERROR]) fail(DFGPU_ERR_ARROW, "DivideByZero");
  // the arguments are read as over FilterRelation's null-free output: every row that passed is an input, unless a CASE
  // made a null (the kernel then counted the non-null inputs itself)
  if (bp.has_pred && !(p.ps.has_nulls && has_case(p.ps)))
    for (int a = 0; a < st->naggs; a++) st->nonnull_host[size_t(a)] += (long long)c[CTR_PASSED];
}

// What the interpreter-free scan kernels can do with a batch (once per batch; narrow keys only).
struct ScanPlan {
  bool plain = false;  // keys and arguments are plain 4/8-byte columns and the WHERE clause, if any, a chain of column
                       // comparisons: p.plain describes them for k_hash_agg_plain
  int lean_mask = 0;   // nonzero: k_hash_agg_lean applies, with this aggregate set (MIN 1, MAX 2, SUM 4, COUNT 8)
  int lean_mt = 0;     // and this machine type of the argument
};
ScanPlan plan_scan(const dfgpu_aggstate* st, const BatchPrograms& bp, AggParams& p) {
  ScanPlan plan;
  static const bool plain_off = getenv("DFGPU_AGG_PLAIN") && atoi(getenv("DFGPU_AGG_PLAIN")) == 0;  // A/B switch
  plan.plain = !plain_off && plain_spec(bp.pb, p.ps, bp.has_pred, st->nkeys, bp.nargs, &p.plain);
  // lean kernel: one 8-byte integer key column, one 8-byte argument column, distinct MIN/MAX/SUM/COUNT, no WHERE
  static const bool lean_off = getenv("DFGPU_AGG_LEAN") && atoi(getenv("DFGPU_AGG_LEAN")) == 0;  // A/B switch
  bool ok = !lean_off && plan.plain && !bp.has_pred && st->nkeys == 1 && bp.nargs == 1 && is_numeric8(p.ps.cols[p.plain.key_slot[0]].dtype) &&
       is_numeric8(p.ps.cols[p.plain.arg_slot[0]].dtype);
  int mask = 0;
  for (int a = 0; ok && a < p.naggs; a++) {
    int f = st->descs[size_t(a)].func;
    if (f == AGG_AVG_SUM) {  // the lean SUM adds the argument as it is: that is AVG's f64 sum for a Float64 argument only
      ok = st->descs[size_t(a)].mtype == MT_F64;
      f = DFGPU_AGG_SUM;
    }
    const int bit = 1 << (f - 1);  // MIN 1, MAX 2, SUM 4, COUNT 8
    ok = ok && !(mask & bit);
    mask |= bit;
  }
  if (ok) {
    plan.lean_mask = mask;
    plan.lean_mt = mtype_of(p.ps.cols[p.plain.arg_slot[0]].dtype);
  }
  return plan;
}

// The scan kernel of one round.  Replays read a row list and the plain and lean kernels start on an even row, so both
// take the interpreter; FRONT routes rows through the shared-memory front table.  A lean launch gets its table
// addresses in p.lean.
ScanKernel choose_scan(const dfgpu_aggstate* st, AggParams& p, const ScanPlan& plan, bool replay, bool front) {
  const bool fn = has_fn(p.ps), cs = has_case(p.ps);
  if (st->wide) {
    if (cs && p.ps.has_nulls) return {k_hash_agg_wide<kCaseDepth, true>, "k_hash_agg_wide<kCaseDepth, true>", false};
    if (cs) return {k_hash_agg_wide<kCaseDepth, false>, "k_hash_agg_wide<kCaseDepth, false>", false};
    if (fn && p.ps.has_nulls) return {k_hash_agg_wide<kFnDepth, true>, "k_hash_agg_wide<kFnDepth, true>", false};
    if (fn) return {k_hash_agg_wide<kFnDepth, false>, "k_hash_agg_wide<kFnDepth, false>", false};
    if (p.ps.has_nulls) return {k_hash_agg_wide<8, true>, "k_hash_agg_wide<8, true>", false};
    return {k_hash_agg_wide<8, false>, "k_hash_agg_wide<8, false>", false};
  }
  if (cs && p.ps.has_nulls) return {k_hash_agg<kCaseDepth, false, true>, "k_hash_agg<kCaseDepth, false, true>", false};
  if (fn && p.ps.has_nulls) return {k_hash_agg<kFnDepth, false, true>, "k_hash_agg<kFnDepth, false, true>", false};
  if (p.ps.has_nulls) return {k_hash_agg<8, false, true>, "k_hash_agg<8, false, true>", false};
  const bool even = (p.row_begin & 1) == 0;
  if (plan.lean_mask && !replay && !front && !st->aos && even) {
    // the lean kernel addresses the hybrid layout directly
    p.lean.key_col = (const unsigned long long*)p.ps.cols[p.plain.key_slot[0]].ptr;
    p.lean.arg_col = (const unsigned long long*)p.ps.cols[p.plain.arg_slot[0]].ptr;
    p.lean.min_w = p.lean.max_w = 0;
    p.lean.sum_arr = p.lean.cnt_arr = nullptr;
    for (int a = 0; a < p.naggs; a++) {
      const int f = st->descs[size_t(a)].func, l = st->t.loc[a];
      if (f == DFGPU_AGG_MIN) p.lean.min_w = l;
      else if (f == DFGPU_AGG_MAX) p.lean.max_w = l;
      else if (f == DFGPU_AGG_SUM || f == AGG_AVG_SUM) p.lean.sum_arr = st->t.add + (long long)(~l) * st->t.astride;
      else p.lean.cnt_arr = st->t.add + (long long)(~l) * st->t.astride;
    }
    bool layout_ok = st->t.lw == (((plan.lean_mask & 3) == 3) ? 4 : ((plan.lean_mask & 3) ? 2 : 1));
    for (int a = 0; a < p.naggs; a++) {
      const int f = st->descs[size_t(a)].func;
      layout_ok = layout_ok && ((f == DFGPU_AGG_MIN || f == DFGPU_AGG_MAX) ? st->t.loc[a] >= 1 : st->t.loc[a] < 0);
    }
    if (layout_ok) return lean_kernel(plan.lean_mask, plan.lean_mt);
    return {k_hash_agg_plain<2, false>, "k_hash_agg_plain<2, false>", false};
  }
  if (plan.plain && !replay && even) {
    const bool two = p.ps.ncols <= 2;
    if (front) {
      if (two) return {k_hash_agg_plain<2, true>, "k_hash_agg_plain<2, true>", true};
      return {k_hash_agg_plain<4, true>, "k_hash_agg_plain<4, true>", true};
    }
    if (two) return {k_hash_agg_plain<2, false>, "k_hash_agg_plain<2, false>", false};
    return {k_hash_agg_plain<4, false>, "k_hash_agg_plain<4, false>", false};
  }
  const int d = p.ps.max_depth;
  if (cs) return hash_agg_kernel<kCaseDepth>(front);
  if (fn) return hash_agg_kernel<kFnDepth>(front);
  if (d <= 1) return hash_agg_kernel<1>(front);
  if (d <= 2) return hash_agg_kernel<2>(front);
  if (d <= 4) return hash_agg_kernel<4>(front);
  return hash_agg_kernel<8>(front);
}

// Single Utf8 key: every row's string must equal its group's representative string, or two strings share a hash.
void verify_utf8_groups(dfgpu_aggstate* st, const BatchPrograms& bp, long long nrows) {
  dfgpu_ctx* ctx = st->ctx;
  VerifyParams vp;
  memset(&vp, 0, sizeof(vp));
  vp.hashes = bp.ukey_hash;
  vp.n = nrows;
  vp.t = st->t;
  vp.rep_agg = st->naggs - 1;
  vp.off = bp.ukey->offsets;
  vp.bytes = (const unsigned char*)bp.ukey->values;
  vp.srcs = st->d_utf8_srcs;
  vp.flag = st->d_counters + CTR_DEFERRED;
  vp.has_pred = bp.has_pred;
  DF_CUDA(cudaMemsetAsync(vp.flag, 0, 8, ctx->stream));
  launch_kernel(ctx, k_utf8_group_verify, "k_utf8_group_verify", vp, nrows, 256, 8);
  const unsigned long long flag = read_counter(st, CTR_DEFERRED);
  if (flag == 1ull) fail(DFGPU_ERR_INTERNAL, "two different Utf8 GROUP BY keys share a 64-bit hash (p < 1e-7 per 1e6 distinct keys)");
  if (flag) fail(DFGPU_ERR_INTERNAL, "Utf8 GROUP BY verification could not find a group");
}

// The grow-and-replay loop of the group table and of the COUNT(DISTINCT) sets.  run() passes rows [begin, begin + count)
// of the batch through round(), then the rows it refused through it again, until a round refuses none.  round() launches
// one kernel over the rows p describes, the range or the last round's overflow list, applies the growth rule of its
// table or sets and returns the number of rows it appended to p.ovf_rows (counted in `overflow`).  The batch's two
// overflow lists alternate; the second is allocated when a round first needs it.
struct GrowAndReplay {
  DevBufs bufs;
  size_t bytes;
  unsigned* list[2];
  GrowAndReplay(dfgpu_ctx* ctx, long long nrows) : bufs(ctx), bytes(size_t(nrows) * 4), list{bufs.alloc<unsigned>(bytes), nullptr} {}
  template <class Round>
  void run(AggParams& p, unsigned long long* overflow, long long begin, long long count, const char* no_convergence, Round&& round) {
    p.row_begin = begin;
    p.nrows = count;
    p.row_list = nullptr;
    p.nlist = 0;
    for (int i = 0, cur = 0;; i++, cur ^= 1) {
      if (i > 60) fail(DFGPU_ERR_INTERNAL, no_convergence);
      if (!list[cur]) list[cur] = bufs.alloc<unsigned>(bytes);
      p.ovf_rows = list[cur];
      DF_CUDA(cudaMemsetAsync(overflow, 0, 8, bufs.ctx->stream));
      const long long novf = round();
      if (novf == 0) return;
      p.row_list = list[cur];
      p.nlist = novf;
    }
  }
};

// One round of the group scan over the rows p describes, then the growth rule of the table: x4 when it went past its
// fill limit, or when it refused rows -- except when each of them only met a slot that was still being published
// (counter CTR_DEFERRED, which only wide scans set): those are replayed as they are.  Returns the number of rows refused.
//
// Rows refused while the table is below the round's own fill limit met the probe limit: AG_MAX_PROBE occupied slots
// after their home.  Growth spreads a cluster of ordinary keys, but keys whose hashes share their top bits share a
// home at every capacity, and growing again would only multiply the table until allocation fails.  So a batch grows
// at most once for that reason (*probe_grown); the next such round fails.
long long scan_round(dfgpu_aggstate* st, AggParams& p, const ScanPlan& plan, Trace& tr, bool prefix, bool* probe_grown) {
  dfgpu_ctx* ctx = st->ctx;
  const bool replay = p.row_list != nullptr;
  p.t = st->t;
  p.max_groups = fill_limit(st->t.cap);
  // <= 64 groups: one private 256-slot table per warp (same shared-memory footprint as the
  // CTA-wide 2048-slot table); otherwise one table per CTA
  p.front_per_warp = st->ngroups <= 64 ? 1 : 0;
  p.front_slots = p.front_per_warp ? AG_FRONT_SLOTS / (AG_THREADS / 32) : AG_FRONT_SLOTS;
  // (A persisting-L2 access-policy window over the table was tried and removed: it slowed the scan
  // several-fold at 1e5 and 1e6 groups.)
  const ScanKernel k = choose_scan(st, p, plan, replay, st->use_front && !replay);
  const size_t smem = k.front ? size_t(AG_FRONT_SLOTS) * 8 * size_t(1 + p.naggs) : 0;
  if (k.front && ctx->first_use((const void*)k.fn))
    DF_CUDA(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, AG_FRONT_SLOTS * 8 * (1 + kMaxAggs)));
  // FRONT launches admit the keys of every CTA's front table unconditionally when the CTA retires, so the fill limit of
  // the global path is lowered by what they can add (grid x front slots): the table stays at most half full and the
  // front merge always finds a slot.
  launch_ag(ctx, k.fn, k.name, replay ? p.nlist : p.nrows, AG_TILE, 0, LaunchOpts{smem, true}, [&](int grid) {
    if (k.front) p.max_groups = std::max<long long>(0, p.max_groups - (long long)grid * AG_FRONT_SLOTS);
  }, p);
  unsigned long long c[CTR_NONNULL];
  read_counters(st, c);
  if (c[CTR_ERROR] == 2) fail(DFGPU_ERR_INTERNAL, "front-table merge could not find a slot");
  if (c[CTR_ERROR]) fail(DFGPU_ERR_ARROW, "DivideByZero");
  st->ngroups = (long long)c[CTR_GROUPS];
  st->sentinel_used = c[CTR_SENTINEL] != 0;
  const long long novf = (long long)c[CTR_OVERFLOW], deferred = (long long)c[CTR_DEFERRED];
  if (deferred) DF_CUDA(cudaMemsetAsync(st->d_counters + CTR_DEFERRED, 0, 8, ctx->stream));
  tr.mark(prefix ? "scan kernel (prefix)" : "scan kernel");
  // a row refused for the fill limit read a group count >= max_groups, which only grows: below it, no row was
  if (novf > deferred && st->ngroups < p.max_groups) {
    if (*probe_grown)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "GROUP BY keys whose hashes share one home slot: more than the probe limit of " +
                                          std::to_string(AG_MAX_PROBE) + " keys on one probe chain");
    *probe_grown = true;
  }
  if (st->ngroups > fill_limit(st->t.cap) || (novf > 0 && novf != deferred)) {
    table_grow(st, grown_cap(st->t.cap));
    if (novf == 0) tr.mark("table_grow (load factor)");
  }
  return novf;
}

// The row ranges, (begin, count), that a batch goes through the table and the sets in.  A first big batch with no
// cardinality hint is cut after a 1 Mi-row prefix: what the prefix produces sizes the sets and decides the table's
// capacity and layout (hybrid while the hot sectors fit L2, line beyond) before the rest of the batch is touched.  Wide
// tables are line-laid-out from the start.
std::vector<std::pair<long long, long long>> batch_ranges(const dfgpu_aggstate* st, long long nrows) {
  if (st->rows_seen == nrows && st->expected == 0 && !st->aos && nrows >= 4 * AG_PREFIX_ROWS)
    return {{0, AG_PREFIX_ROWS}, {AG_PREFIX_ROWS, nrows - AG_PREFIX_ROWS}};
  return {{0, nrows}};
}

// After the prefix of a first batch of `batch_rows` rows: size each set, then the table, for the number of entries
// estimated from the prefix -- one rebuild of a ~1 Mi-entry table or set instead of repeated x4 growth and replays.
void size_from_prefix(dfgpu_aggstate* st, long long batch_rows, Trace& tr) {
  if (!st->dist_progs.empty()) {
    unsigned long long c[DCTR_SLOTS];
    read_dctr(st, c);
    for (size_t s = 0; s < st->dist_progs.size(); s++) {
      const long long cur_cap = st->sets[s].cap;
      const long long want = prefix_cap(st->ctx, (long long)c[DCTR_SET + 2 * s], AG_PREFIX_ROWS, batch_rows, 16, cur_cap, AG_SET_MIN_CAP);
      if (want > cur_cap) set_grow(st, int(s), want);
    }
  }
  if (st->nkeys == 0) return;
  long long est = 0;
  const long long want_cap = prefix_cap(st->ctx, st->ngroups, AG_PREFIX_ROWS, batch_rows, 32 * (1 + st->naggs), st->t.cap, AG_MIN_CAP, &est);
  const bool to_aos = !st->aos && want_aos(est, st->descs, st->naggs);
  if (to_aos || want_cap > st->t.cap) {
    st->aos = st->aos || to_aos;
    table_grow(st, want_cap);
    tr.mark("table_grow (prefix estimate)");
  }
}

void agg_update(dfgpu_aggstate* st, const dfgpu_batch* batch) {
  if (st->finished) fail(DFGPU_ERR_GENERAL, "aggregate already finished");
  dfgpu_ctx* ctx = st->ctx;
  ctx->use();
  if (batch->nrows >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "batches of 2^32 rows or more");
  Trace tr(ctx);
  BatchPrograms bp(batch, ctx);
  compile_batch(st, batch, bp);
  type_batch(st, bp);
  tr.mark("programs + table alloc");
  AggParams p;
  memset(&p, 0, sizeof(p));
  bp.pb.finish(&p.ps);
  for (int s = 0; s < p.ps.ncols; s++)
    if (!is_numeric(p.ps.cols[s].dtype) && p.ps.cols[s].dtype != DFGPU_BOOL)  // Boolean columns: WHERE operands (boolean_ops!)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("expressions over ") + dtype_name(p.ps.cols[s].dtype) + " columns are not supported on the GPU path yet");
  if (p.ps.max_depth > 8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "expression too deep (register stack depth > 8)");
  st->rows_seen += batch->nrows;
  if (batch->nrows == 0) return;

  p.nkeys = st->nkeys;
  p.naggs = st->naggs - int(st->dist_set.size());  // the scan kernels never see the COUNT(DISTINCT) words
  for (int a = 0; a < p.naggs; a++) {
    p.aggs[a] = st->descs[size_t(a)];
    p.agg_arg[a] = bp.agg_arg[size_t(a)];
  }
  p.nargs = bp.nargs;
  for (int k = 0; k < st->nkeys; k++) {
    p.key_mask[k] = st->key_mask[size_t(k)];
    p.key_shift[k] = st->key_shift[size_t(k)];
  }
  p.nrows = batch->nrows;
  p.counters = st->d_counters;
  p.has_pred = bp.has_pred;
  const bool group_by = st->nkeys > 0, distinct = !st->dist_progs.empty();
  if (!group_by) {
    reduce_update(st, bp, p);  // one launch over the whole batch
    if (!distinct) return;
  } else if (st->wide) {
    // retain this batch's Utf8 key columns: a group's string lives in the batch whose row created it
    p.wide.kw = st->nkeys;
    bool new_src = false;
    for (int k = 0; k < st->nkeys; k++) {
      p.wide.is_utf8[k] = st->key_is_utf8[size_t(k)];
      const DevColumn* uc = bp.key_utf8[size_t(k)];
      if (!uc) continue;
      if (st->utf8_srcs.size() >= (1u << 20)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than 2^20 retained Utf8 GROUP BY key columns");
      p.wide.ref_base[k] = retain_utf8(st, *uc, batch->nrows) << UTF8_SRC_SHIFT;
      p.wide.off[k] = st->utf8_srcs.back().off;
      p.wide.bytes[k] = st->utf8_srcs.back().bytes;
      new_src = true;
    }
    if (new_src) upload_utf8_srcs(st);
    p.wide.srcs = st->d_utf8_srcs;
  }
  const ScanPlan plan = group_by && !st->wide ? plan_scan(st, bp, p) : ScanPlan{};
  bool ins_plain = false;
  AggParams ins = distinct ? plan_insert(st, bp, &ins_plain) : AggParams{};
  GrowAndReplay loop(ctx, batch->nrows);
  tr.mark("overflow list alloc");
  const auto ranges = batch_ranges(st, batch->nrows);
  bool table_probe_grown = false, set_probe_grown = false;  // growth for the probe limit, once per batch
  for (size_t ri = 0; ri < ranges.size(); ri++) {
    const long long begin = ranges[ri].first, count = ranges[ri].second;
    const bool prefix = ranges.size() > 1 && ri == 0;
    if (group_by)
      loop.run(p, st->d_counters + CTR_OVERFLOW, begin, count, "hash table growth did not converge",
               [&] { return scan_round(st, p, plan, tr, prefix, &table_probe_grown); });
    // after the group scan of the same rows: every key the insert packs is in the table
    if (distinct)
      loop.run(ins, st->d_dctr + DCTR_OVERFLOW, begin, count, "COUNT(DISTINCT) set growth did not converge",
               [&] { return insert_round(st, ins, ins_plain, &set_probe_grown); });
    // few groups so far: later rows of this stream go through the shared-memory front table
    if (group_by) st->use_front = st->ngroups <= AG_FRONT_MAX_GROUPS && st->rows_seen >= (1ll << 20);
    if (prefix) size_from_prefix(st, batch->nrows, tr);
  }
  if (bp.ukey) verify_utf8_groups(st, bp, batch->nrows);
}
}  // namespace

// ---------------------------------------------------------------------------------------------
// multi-GPU merge of partial aggregates (SURVEY.md §8e).  Every rank ends with the global result.
//   no GROUP BY : one ncclAllReduce per accumulator (api.cu comm_allreduce_aggs)
//   GROUP BY    : open-addressed slots are not canonical across ranks, so the all-reduce is sparse and
//                 owner-partitioned:  raw-compact the local table -> count entries per owner rank ->
//                 all-gather a (header, counts) record -> scatter the entries into per-owner segments ->
//                 ONE grouped ncclSend/ncclRecv all-to-all -> each rank merges only the keys it owns into a
//                 fresh table (k_merge) -> compacts them -> all ranks gather the owned segments
//                 (grouped ncclBroadcast) and decode the same rows in the same order, so results are
//                 bit-identical on every rank.  Work per rank is O(G_local + G/W + G), not O(W x G).
// A rank that never saw a batch takes part with zero entries and adopts the key / argument types of a rank
// that did (they travel in the header).
// ---------------------------------------------------------------------------------------------
namespace {

void agg_export_raw(dfgpu_aggstate* st, DevBufs& bufs, unsigned long long** keys, unsigned long long** vals, long long* n) {
  const long long cnt = st->nkeys == 0 ? 1 : st->ngroups + (st->sentinel_used ? 1 : 0);
  const size_t alloc_n = size_t(cnt > 0 ? cnt : 1);
  *keys = bufs.alloc(alloc_n * 8);
  *vals = bufs.alloc(alloc_n * 8 * size_t(st->naggs));
  compact_raw(st, st->t, st->nkeys == 0 ? 1 : (st->sentinel_used ? 1 : 0), nullptr, *keys, *vals, alloc_n, 0);
  *n = cnt;
}

// no GROUP BY
void agg_exchange_scalars(dfgpu_ctx* ctx, dfgpu_aggstate* st) {
  int funcs[kMaxAggs], mtypes[kMaxAggs];
  for (int a = 0; a < st->naggs; a++) {
    const bool avg = st->descs[size_t(a)].func == AGG_AVG_SUM;  // merged as the f64 SUM it is
    funcs[a] = avg ? DFGPU_AGG_SUM : st->descs[size_t(a)].func;
    mtypes[a] = avg ? MT_F64 : st->descs[size_t(a)].mtype;
  }
  // per-aggregate non-null input counts travel with the accumulators: fold the host-side counts of the
  // null-free batches into the device counters, which the exchange sums over ranks
  static_assert(kMaxAggs <= SCR_AGG_NONNULL.words, "a non-null count per aggregate");
  unsigned long long* nonnull = ctx->h_scratch + SCR_AGG_NONNULL.at;  // pinned: uploaded below
  unsigned long long* rows = ctx->h_scratch + SCR_AGG_ROWS.at;
  read_words(ctx, st->d_counters + CTR_NONNULL, kMaxAggs * 8, nonnull);
  for (int a = 0; a < kMaxAggs; a++) {
    if (a < st->naggs) nonnull[a] += (unsigned long long)st->nonnull_host[size_t(a)];
    if (a < st->naggs) st->nonnull_host[size_t(a)] = 0;
  }
  *rows = (unsigned long long)st->rows_seen;
  DF_CUDA(cudaMemcpyAsync(st->d_counters + CTR_NONNULL, nonnull, kMaxAggs * 8, cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaMemcpyAsync(st->d_counters + CTR_ROWS, rows, 8, cudaMemcpyHostToDevice, ctx->stream));
  st->saw_nulls = true;
  // slot 0's accumulators (cap = 0: every accumulator in its own one-word array, contiguous)
  comm_allreduce_aggs(ctx, st->naggs, funcs, mtypes, st->t.val(0, 0), st->d_counters + CTR_NONNULL, st->d_counters + CTR_ROWS);
  st->rows_seen = (long long)read_counter(st, CTR_ROWS);
}

// GROUP BY.  Returns the global result as raw rows of (1 + naggs) words in *rows (caller frees) and their number.
constexpr int HDR = 16;  // header words: [0] typed [1] nkeys [2] naggs [3] utf8 [4] rows_seen [5] key dtypes (8 bits each) [6] arg dtypes (8 bits each)
struct GatheredSegments {
  int nseg = 0;
  long long stride = 0;
  long long n[AG_MAX_WORLD] = {0};
};
void agg_exchange_groups(dfgpu_ctx* ctx, dfgpu_aggstate* st, DevBufs& rows_buf, unsigned long long** rows_out, long long* n_out, GatheredSegments* seg,
                         bool* regroup) {
  const int W = ctx->world, me = ctx->rank;
  if (W > AG_MAX_WORLD) fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than " + std::to_string(AG_MAX_WORLD) + " ranks");
  Trace tr(ctx);
  DevBufs tmp(ctx);
  auto dalloc = [&](size_t words) { return tmp.alloc((words ? words : 1) * 8); };
  // 1. local entries, counted per owner
  unsigned long long *keys = nullptr, *vals = nullptr;
  long long n_local = 0;
  // Utf8 and wide keys do not fit the (packed key, accumulators) rows of this exchange: if any rank has them, every
  // rank leaves through the regroup merge (finish_regroup) right after the header round
  const bool special = st->typed && (st->wide || st->utf8_key);
  if (st->typed && !special) agg_export_raw(st, tmp, &keys, &vals, &n_local);
  unsigned long long* d_rec = dalloc(size_t(HDR + W));
  DF_CUDA(cudaMemsetAsync(d_rec, 0, size_t(HDR + W) * 8, ctx->stream));
  OwnerParams op;
  memset(&op, 0, sizeof(op));
  op.keys = keys;
  const size_t ln = size_t(n_local > 0 ? n_local : 1);
  for (int a = 0; a < st->naggs; a++) op.vals[a] = vals + size_t(a) * ln;
  op.n = n_local;
  op.world = W;
  op.naggs = st->naggs;
  op.counts = d_rec + HDR;
  if (n_local > 0) launch_kernel(ctx, k_owner_count, "k_owner_count", op, n_local, 256 * 4, 8);
  static_assert(HDR <= SCR_AGG_HEADER.words, "the header record fits its scratch range");
  unsigned long long* hh = ctx->h_scratch + SCR_AGG_HEADER.at;  // pinned
  memset(hh, 0, HDR * 8);
  hh[0] = st->typed ? 1 : 0;
  hh[1] = (unsigned long long)st->nkeys;
  hh[2] = (unsigned long long)(st->utf8_key ? st->naggs - 1 : st->naggs);  // user aggregates
  hh[3] = special ? 1 : 0;
  hh[7] = st->utf8_key ? 1 : 0;  // the single-Utf8-key form carries a hidden representative aggregate
  hh[4] = (unsigned long long)st->rows_seen;
  if (st->typed) {
    for (int k = 0; k < st->nkeys; k++) hh[5] |= (unsigned long long)(st->key_dtypes[size_t(k)] & 0xff) << (8 * k);
    for (int a = 0; a < (st->utf8_key ? st->naggs - 1 : st->naggs); a++) hh[6] |= (unsigned long long)(st->descs[size_t(a)].dtype & 0xff) << (8 * a);
    if (st->utf8_key) hh[5] = DFGPU_UTF8;  // the key the caller sees (internally: a UInt64 string hash)
  }
  DF_CUDA(cudaMemcpyAsync(d_rec, hh, HDR * 8, cudaMemcpyHostToDevice, ctx->stream));
  // 2. all-gather (header, counts)
  unsigned long long* d_all = dalloc(size_t(W) * size_t(HDR + W));
  comm_allgather_u64(ctx, d_rec, d_all, size_t(HDR + W));
  std::vector<unsigned long long> all(size_t(W) * size_t(HDR + W));
  DF_CUDA(cudaMemcpyAsync(all.data(), d_all, all.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  auto hdr = [&](int r, int i) { return all[size_t(r) * size_t(HDR + W) + size_t(i)]; };
  auto cnt = [&](int from, int to) { return (size_t)all[size_t(from) * size_t(HDR + W) + size_t(HDR + to)]; };
  // 3. agree on types; adopt them on a rank that saw no batch
  int typed_rank = -1;
  long long total_rows = 0;
  for (int r = 0; r < W; r++) {
    total_rows += (long long)hdr(r, 4);
    if ((int)hdr(r, 1) != st->nkeys) fail(DFGPU_ERR_GENERAL, "ranks disagree on the GROUP BY expressions");
    if (hdr(r, 3)) *regroup = true;
    if (hdr(r, 0)) {
      if (typed_rank < 0) typed_rank = r;
      else if (hdr(r, 5) != hdr(typed_rank, 5) || hdr(r, 6) != hdr(typed_rank, 6) || hdr(r, 2) != hdr(typed_rank, 2) || hdr(r, 3) != hdr(typed_rank, 3))
        fail(DFGPU_ERR_GENERAL, "ranks disagree on GROUP BY key / aggregate argument types");
    }
  }
  st->rows_seen = total_rows;
  if (!st->typed) {
    st->key_dtypes.clear();
    st->descs.clear();
    for (int k = 0; k < st->nkeys; k++) st->key_dtypes.push_back(typed_rank >= 0 ? int((hdr(typed_rank, 5) >> (8 * k)) & 0xff) : DFGPU_INT64);
    for (int a = 0; a < st->naggs; a++) {
      int dt = typed_rank >= 0 ? int((hdr(typed_rank, 6) >> (8 * a)) & 0xff) : st->out_dtypes[size_t(a)];
      if (!is_numeric(dt)) dt = DFGPU_FLOAT64;
      AggDesc d;
      d.func = uint8_t(st->funcs[size_t(a)]);
      d.dtype = uint8_t(dt);
      d.mtype = mtype_of(dt);
      d.out_dtype = uint8_t(d.func == DFGPU_AGG_COUNT ? DFGPU_UINT64 : (d.func == AGG_AVG_SUM ? DFGPU_FLOAT64 : dt));
      st->descs.push_back(d);
    }
    if (!*regroup) pack_keys(st);  // (the regroup merge never packs keys)
    st->typed = true;
  }
  if (*regroup) {
    *rows_out = nullptr;
    *n_out = -1;
    return;
  }
  const size_t E = size_t(1 + st->naggs);
  // 4. scatter the local entries into per-owner segments
  std::vector<size_t> s_off(size_t(W), 0), s_cnt(size_t(W), 0), r_off(size_t(W), 0), r_cnt(size_t(W), 0);
  size_t total_send = 0, total_recv = 0;
  for (int r = 0; r < W; r++) {
    s_off[size_t(r)] = total_send * E;
    s_cnt[size_t(r)] = cnt(me, r) * E;
    total_send += cnt(me, r);
    r_off[size_t(r)] = total_recv * E;
    r_cnt[size_t(r)] = cnt(r, me) * E;
    total_recv += cnt(r, me);
  }
  if ((long long)total_send != n_local) fail(DFGPU_ERR_INTERNAL, "owner counts do not add up to the local groups");
  size_t max_recv = 1;  // the most entries any rank receives (column sums of the count matrix)
  for (int r = 0; r < W; r++) {
    size_t col = 0;
    for (int q = 0; q < W; q++) col += cnt(q, r);
    max_recv = std::max(max_recv, col);
  }
  unsigned long long* d_send = dalloc(total_send * E);
  if (n_local > 0) {
    unsigned long long* d_cursor = dalloc(size_t(W));
    DF_CUDA(cudaMemsetAsync(d_cursor, 0, size_t(W) * 8, ctx->stream));
    op.cursor = d_cursor;
    op.rows = d_send;
    for (int r = 0; r < W; r++) op.seg_off[r] = s_off[size_t(r)] / E;
    launch_kernel(ctx, k_owner_scatter, "k_owner_scatter", op, n_local, 256 * 4, 8);
  }
  // 5. all-to-all: every entry goes to its owner
  unsigned long long* d_recv = dalloc(total_recv * E);
  comm_exchange_v(ctx, d_send, s_off.data(), s_cnt.data(), d_recv, r_off.data(), r_cnt.data());
  tr.mark("exchange: export + all-to-all");
  // 6. merge what this rank owns into a fresh table
  long long n_owned = 0;
  unsigned long long* d_owned = nullptr;
  if (total_recv > 0) {
    const bool oaos = want_aos((long long)total_recv, st->descs, st->naggs);
    TableLayout ot = table_alloc(ctx, st->naggs, st->nkeys, st->descs, table_cap((long long)total_recv, 1024), oaos);
    tmp.blocks.push_back(ot.base);
    MergeParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.in_keys = d_recv;
    for (int a = 0; a < st->naggs; a++) {
      mp.in_vals[a] = d_recv + 1 + a;
      mp.aggs[a] = st->descs[size_t(a)];
    }
    mp.in_stride = (long long)E;
    mp.n = (long long)total_recv;
    mp.t = ot;
    mp.naggs = st->naggs;
    DF_CUDA(cudaMemsetAsync(st->d_counters, 0, (CTR_ERROR + 1) * 8, ctx->stream));  // slots CTR_GROUPS .. CTR_ERROR
    mp.counters = st->d_counters;
    launch_kernel(ctx, k_merge, "k_merge", mp, mp.n, 256, 8);
    // compact what this rank owns without a host round trip in between: the buffer has room for the largest
    // number of entries any rank receives (known to all from the count matrix), which also makes it a valid send
    // buffer of the padded all-gather below; the sentinel slot's use and the count stay on the device
    d_owned = dalloc(max_recv * E);
    compact_raw(st, ot, 0, st->d_counters + CTR_SENTINEL, d_owned, d_owned + 1, 1, (long long)E);
  } else {
    DF_CUDA(cudaMemsetAsync(st->d_counters, 0, CTR_NONNULL * 8, ctx->stream));  // no entries, no merge error
  }
  // 7. every rank gathers the owned segments: sizes first ([owned entries, merge error flag] per rank)
  unsigned long long* d_n = dalloc(size_t(2 + 2 * W));
  DF_CUDA(cudaMemcpyAsync(d_n, st->d_counters + CTR_COMPACT, 8, cudaMemcpyDeviceToDevice, ctx->stream));
  DF_CUDA(cudaMemcpyAsync(d_n + 1, st->d_counters + CTR_ERROR, 8, cudaMemcpyDeviceToDevice, ctx->stream));
  comm_allgather_u64(ctx, d_n, d_n + 2, 2);
  std::vector<unsigned long long> owned_n2(size_t(2 * W), 0);
  DF_CUDA(cudaMemcpyAsync(owned_n2.data(), d_n + 2, size_t(2 * W) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<unsigned long long> owned_n(size_t(W), 0);
  for (int r = 0; r < W; r++) {
    if (owned_n2[size_t(2 * r + 1)]) fail(DFGPU_ERR_INTERNAL, "partial-aggregate merge failed on rank " + std::to_string(r));
    owned_n[size_t(r)] = owned_n2[size_t(2 * r)];
  }
  n_owned = (long long)owned_n[size_t(me)];
  // one fixed-size all-gather of max_owned entries per rank (owners are a hash of the key, so the segments are
  // within a few percent of each other): one collective instead of one broadcast per rank
  size_t max_owned = 0, G = 0;
  for (int r = 0; r < W; r++) {
    max_owned = std::max(max_owned, size_t(owned_n[size_t(r)]));
    G += size_t(owned_n[size_t(r)]);
  }
  if (max_owned > max_recv) fail(DFGPU_ERR_INTERNAL, "owned groups exceed the received entries");
  unsigned long long* d_final = rows_buf.alloc((max_owned ? size_t(W) * max_owned * E : 1) * 8);
  if (max_owned > 0) {
    if (!d_owned) d_owned = dalloc(max_recv * E);  // a rank that owns nothing still contributes its (empty) segment
    comm_allgather_u64(ctx, d_owned, d_final, max_owned * E);
  }
  DF_CUDA(cudaStreamSynchronize(ctx->stream));  // the temporaries above are released on return
  tr.mark("exchange: owner merge + gather");
  *rows_out = d_final;
  *n_out = (long long)G;
  seg->nseg = W;
  seg->stride = (long long)max_owned;
  for (int r = 0; r < W; r++) seg->n[r] = (long long)owned_n[size_t(r)];
}

}  // namespace

// Multi-GPU merge for key shapes whose groups cannot travel as (packed key, accumulators) rows — Utf8 keys and
// wide composite keys: every rank finishes locally, the ranks all-gather their LOCAL key and table-word columns
// (strings included), and every rank aggregates the concatenation once more with the merge function of each word
// (SUM -> SUM, COUNT -> SUM of counts, AVG's sum -> SUM, MIN -> MIN, MAX -> MAX) through the same single-GPU
// operator.  O(W x G) work
// per rank instead of the owner-partitioned O(G): accepted for these shapes.  Results agree across ranks bit for
// bit except Float64 SUMs (order of the second aggregation's reductions: <= 1e-9 relative).
namespace {
struct WorldGuard {  // run a stretch of the operator as if no communicator were attached
  dfgpu_ctx* c;
  int world;
  explicit WorldGuard(dfgpu_ctx* ctx) : c(ctx), world(ctx->world) { c->world = 1; }
  ~WorldGuard() { c->world = world; }
};

// The merge works on table words, not on the caller's columns: an AVG travels as its sum and count words, which are
// merged with SUM and divided only after the merge (k_avg_finish, in finish).  Returns keys + one column per word.
std::unique_ptr<dfgpu_result> finish_regroup(dfgpu_ctx* ctx, dfgpu_aggstate* st) {
  const int W = ctx->world;
  const int nwords = st->utf8_key ? st->naggs - 1 : st->naggs;
  const int ncols = st->nkeys + nwords;
  // 1. this rank's own words (an empty result when it saw no batch: types were adopted from the header)
  std::unique_ptr<dfgpu_result> local;
  if (st->t.base) {
    WorldGuard g(ctx);
    dfgpu_result* r = nullptr;
    st->emit_words = true;
    const int rc = dfgpu_aggregate_finish(st, &r);
    if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
    local.reset(r);
  } else {
    local = std::make_unique<dfgpu_result>();
    local->ctx = ctx;
    local->nrows = 0;
    for (int k = 0; k < st->nkeys; k++) {
      DevColumn c;
      c.dtype = st->key_dtypes[size_t(k)];
      if (c.dtype == DFGPU_UTF8) {
        c.offsets = (int32_t*)ctx->alloc(4);
        DF_CUDA(cudaMemsetAsync(c.offsets, 0, 4, ctx->stream));
      }
      local->cols.push_back(c);
    }
    for (int a = 0; a < nwords; a++) {
      DevColumn c;
      c.dtype = st->descs[size_t(a)].out_dtype;
      local->cols.push_back(c);
    }
  }
  if (int(local->cols.size()) != ncols) fail(DFGPU_ERR_INTERNAL, "regroup merge: unexpected local result shape");
  // 2. sizes: [rows, bytes of every Utf8 column] per rank
  const int NH = 1 + kMaxKeys;
  DevBufs tmp(ctx);
  unsigned long long* d_h = tmp.alloc(size_t(NH) * 8 * size_t(W + 1));
  static_assert(NH <= SCR_AGG_HEADER.words, "the size record fits its scratch range");
  unsigned long long* hh = ctx->h_scratch + SCR_AGG_HEADER.at;  // pinned
  memset(hh, 0, size_t(NH) * 8);
  hh[0] = (unsigned long long)local->nrows;
  for (int k = 0; k < st->nkeys; k++)
    if (local->cols[size_t(k)].dtype == DFGPU_UTF8) hh[1 + k] = (unsigned long long)local->cols[size_t(k)].values_bytes;
  DF_CUDA(cudaMemcpyAsync(d_h, hh, size_t(NH) * 8, cudaMemcpyHostToDevice, ctx->stream));
  comm_allgather_u64(ctx, d_h, d_h + NH, size_t(NH));
  std::vector<unsigned long long> all(size_t(NH) * size_t(W));
  DF_CUDA(cudaMemcpyAsync(all.data(), d_h + NH, all.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  long long N = 0;
  std::vector<long long> row_base(size_t(W), 0);
  for (int r = 0; r < W; r++) {
    row_base[size_t(r)] = N;
    N += (long long)all[size_t(r) * NH];
  }
  if (N >= (1ll << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "regroup merge of 2^31 or more partial groups");
  // 3. gather every result column
  auto gathered = std::make_unique<dfgpu_batch>();
  gathered->ctx = ctx;
  gathered->nrows = N;
  std::vector<size_t> off(size_t(W), 0), cnt(size_t(W), 0);
  for (int c = 0; c < ncols; c++) {
    const DevColumn& lc = local->cols[size_t(c)];
    DevColumn gc;
    gc.dtype = lc.dtype;
    if (lc.dtype == DFGPU_UTF8) {
      // bytes
      size_t total_b = 0;
      std::vector<size_t> bbase(size_t(W), 0);
      for (int r = 0; r < W; r++) {
        bbase[size_t(r)] = total_b;
        off[size_t(r)] = total_b;
        cnt[size_t(r)] = size_t(all[size_t(r) * NH + 1 + size_t(c)]);
        total_b += cnt[size_t(r)];
      }
      if (total_b >= (1ull << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "regroup merge of 2 GiB or more of key strings");
      gc.values_bytes = total_b;
      gc.values = ctx->alloc(total_b ? total_b : 1);
      comm_allgather_bytes_v(ctx, lc.values, gc.values, off.data(), cnt.data());
      // offsets: every rank's (rows + 1) array, spliced with its byte base
      int* raw = tmp.alloc<int>(size_t(N + W) * 4);
      for (int r = 0; r < W; r++) {
        off[size_t(r)] = size_t(row_base[size_t(r)] + r) * 4;
        cnt[size_t(r)] = size_t(all[size_t(r) * NH] + 1) * 4;
      }
      comm_allgather_bytes_v(ctx, lc.offsets, raw, off.data(), cnt.data());
      gc.offsets = (int32_t*)ctx->alloc(size_t(N + 1) * 4);
      for (int r = 0; r < W; r++)
        shift_copy_i32(ctx, gc.offsets + row_base[size_t(r)], raw + row_base[size_t(r)] + r, (long long)all[size_t(r) * NH], int(bbase[size_t(r)]));
      const int last = int(total_b);
      DF_CUDA(cudaMemcpyAsync(gc.offsets + N, &last, 4, cudaMemcpyHostToDevice, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));  // `last` is a stack variable
    } else {
      const size_t w = size_t(dtype_width(lc.dtype));
      for (int r = 0; r < W; r++) {
        off[size_t(r)] = size_t(row_base[size_t(r)]) * w;
        cnt[size_t(r)] = size_t(all[size_t(r) * NH]) * w;
      }
      gc.values_bytes = size_t(N) * w;
      gc.values = ctx->alloc(gc.values_bytes ? gc.values_bytes : 8);
      comm_allgather_bytes_v(ctx, lc.values, gc.values, off.data(), cnt.data());
    }
    gathered->cols.push_back(gc);
  }
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  // 4. aggregate the partial results once more, with each aggregate's merge function
  const size_t nk = size_t(st->nkeys), na = size_t(nwords);
  std::vector<dfgpu_insn> kprog(nk), aprog(na);
  std::vector<const dfgpu_insn*> kptr;
  std::vector<int> klen;
  for (int k = 0; k < st->nkeys; k++) {
    memset(&kprog[size_t(k)], 0, sizeof(dfgpu_insn));
    kprog[size_t(k)].op = DFGPU_OP_COL;
    kprog[size_t(k)].col = k;
    kprog[size_t(k)].dtype = gathered->cols[size_t(k)].dtype;
    kptr.push_back(&kprog[size_t(k)]);
    klen.push_back(1);
  }
  std::vector<dfgpu_agg> aggs(na);
  for (int a = 0; a < nwords; a++) {
    memset(&aprog[size_t(a)], 0, sizeof(dfgpu_insn));
    aprog[size_t(a)].op = DFGPU_OP_COL;
    aprog[size_t(a)].col = st->nkeys + a;
    aprog[size_t(a)].dtype = gathered->cols[size_t(st->nkeys + a)].dtype;
    const int f = st->descs[size_t(a)].func;
    aggs[size_t(a)].func = f == DFGPU_AGG_COUNT || f == AGG_AVG_SUM ? DFGPU_AGG_SUM : f;  // AVG's sum word: a Float64 column
    aggs[size_t(a)].arg = &aprog[size_t(a)];
    aggs[size_t(a)].arg_len = 1;
    aggs[size_t(a)].out_dtype = gathered->cols[size_t(st->nkeys + a)].dtype;
    aggs[size_t(a)]._pad = 0;
  }
  WorldGuard g(ctx);
  dfgpu_aggstate* st2 = nullptr;
  int rc = dfgpu_aggregate_create(ctx, kptr.data(), klen.data(), st->nkeys, aggs.data(), nwords, N / W + 1, &st2);
  if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
  struct StFree { dfgpu_aggstate* s; ~StFree() { dfgpu_aggregate_free(s); } } stfree{st2};
  dfgpu_result* res = nullptr;
  if (N > 0) {
    rc = dfgpu_aggregate_update(st2, gathered.get());
    if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
    rc = dfgpu_aggregate_finish(st2, &res);
    if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
    return std::unique_ptr<dfgpu_result>(res);
  }
  return local;  // nobody had a group: the (empty) local result has the right columns
}

// The caller's aggregate columns from a result that holds the key columns and then one column per table word: the
// COUNT(DISTINCT) words are put in the caller's order, and each AVG is computed from its sum and count words, which
// are then freed like every word no output uses.
void assemble_outputs(dfgpu_aggstate* st, dfgpu_result* res) {
  dfgpu_ctx* ctx = st->ctx;
  const size_t nk = size_t(st->nkeys);
  const long long n = res->nrows;
  dfgpu_result spare;  // RAII: the word columns that are not outputs
  spare.ctx = ctx;
  spare.cols.assign(res->cols.begin() + nk, res->cols.end());
  res->cols.resize(nk);
  bool any_avg = false;
  for (char a : st->out_is_avg) any_avg = any_avg || a;
  if (!any_avg) {  // a reordering only: no device work, no synchronisation
    for (int w : st->out_word) {
      res->cols.push_back(spare.cols[size_t(w)]);
      spare.cols[size_t(w)] = DevColumn{};
    }
    return;
  }
  DevBufs tmp(ctx);
  unsigned long long* d_nulls = tmp.alloc(kMaxAggs * 8);
  DF_CUDA(cudaMemsetAsync(d_nulls, 0, kMaxAggs * 8, ctx->stream));
  for (size_t i = 0; i < st->out_word.size(); i++) {
    const size_t w = size_t(st->out_word[i]);
    if (!st->out_is_avg[i]) {
      res->cols.push_back(spare.cols[w]);
      spare.cols[w] = DevColumn{};
      continue;
    }
    DevColumn c;
    c.dtype = DFGPU_FLOAT64;
    c.values_bytes = size_t(n) * 8;
    c.values = ctx->alloc(size_t(n > 0 ? n : 1) * 8);
    res->cols.push_back(c);
    if (n == 0) continue;
    res->cols.back().validity = (uint8_t*)ctx->alloc(size_t((n + 31) / 32) * 4);
    AvgFinishParams ap;
    ap.sum = (const double*)spare.cols[w].values;
    ap.cnt = (const unsigned long long*)spare.cols[w + 1].values;
    ap.n = n;
    ap.out = (double*)res->cols.back().values;
    ap.validity = (unsigned*)res->cols.back().validity;
    ap.nulls = d_nulls + i;
    launch_kernel(ctx, k_avg_finish, "k_avg_finish", ap, n, 256 * 4, 8);
  }
  unsigned long long h[kMaxAggs];
  read_words(ctx, d_nulls, sizeof(h), h);
  for (size_t i = 0; i < st->out_word.size(); i++) {
    if (st->out_is_avg[i]) set_null_count(ctx, res->cols[nk + i], (int64_t)h[i]);
  }
}
}  // namespace

extern "C" int dfgpu_aggregate_finish(dfgpu_aggstate* st, dfgpu_result** out) {
  return guarded([&] {
    if (!st || !out) fail(DFGPU_ERR_GENERAL, "dfgpu_aggregate_finish: null argument");
    if (st->finished) fail(DFGPU_ERR_GENERAL, "aggregate already finished");  // one-shot (aggregate.rs:616-619)
    dfgpu_ctx* ctx = st->ctx;
    ctx->use();
    Trace tr(ctx);
    if (ctx->world > 1 && !st->dist_progs.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT) with a communicator attached");
    if (!st->typed && !(st->nkeys > 0 && ctx->world > 1)) {
      // no batch was ever seen: resolve types from the declared output types (an AVG's words: Float64 and UInt64)
      if (st->nkeys > 0) {
        // an empty GROUP BY input yields an empty batch; key types are unknown -> need a batch
        fail(DFGPU_ERR_GENERAL, "aggregate finished before any input batch was provided");
      }
      for (int a = 0; a < st->nscan; a++) {
        AggDesc d;
        int odt = st->out_dtypes[size_t(a)];
        if (!is_numeric(odt)) fail(DFGPU_ERR_GENERAL, "aggregate output type must be given when there is no input");
        d.func = uint8_t(st->funcs[size_t(a)]);
        d.dtype = uint8_t(odt);
        d.mtype = mtype_of(odt);
        d.out_dtype = uint8_t(odt);
        st->descs.push_back(d);
      }
      for (size_t j = 0; j < st->dist_set.size(); j++) st->descs.push_back(AggDesc{DFGPU_AGG_COUNT, MT_U, DFGPU_UINT64, DFGPU_UINT64});
      st->typed = true;
      st->t = table_alloc(ctx, st->naggs, st->nkeys, st->descs, 0, false);
    }
    // multi-GPU: every rank must take part (also one that saw no batch), and every rank gets the global result
    unsigned long long* xrows = nullptr;
    long long xn = -1;
    GatheredSegments xseg;
    bool regroup = false;
    DevBufs xbuf(ctx);
    if (ctx->world > 1) {
      if (st->nkeys == 0) agg_exchange_scalars(ctx, st);
      else agg_exchange_groups(ctx, st, xbuf, &xrows, &xn, &xseg, &regroup);
      if (regroup) {
        std::unique_ptr<dfgpu_result> res = finish_regroup(ctx, st);
        assemble_outputs(st, res.get());
        st->finished = true;
        *out = res.release();
        return;
      }
    }
    if (!st->dist_progs.empty()) {  // the COUNT(DISTINCT) words (single GPU: the exchange is refused above)
      if (st->nkeys == 0) distinct_count_scalar(st);
      else distinct_count(st, st->t, st->sentinel_used ? 1 : 0);
    }
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    const long long cnt = xn >= 0 ? xn : (st->nkeys == 0 ? 1 : st->ngroups + (st->sentinel_used ? 1 : 0));
    const size_t alloc_n = size_t(cnt > 0 ? cnt : 1);
    CompactParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.t = st->t;
    cp.sentinel_used = st->nkeys == 0 ? 1 : (st->sentinel_used ? 1 : 0);
    cp.nkeys = st->nkeys;
    cp.naggs = st->naggs;
    cp.raw = 0;
    cp.wide_kw = st->wide ? st->nkeys : 0;
    for (int k = 0; k < st->nkeys && st->wide; k++) cp.key_is_utf8[k] = st->key_is_utf8[size_t(k)];
    dfgpu_result hidden;  // RAII: hash-key and representative columns of a Utf8-keyed aggregate
    hidden.ctx = ctx;
    std::vector<std::pair<int, size_t>> wide_refs;  // wide keys: (key part, index of its reference column in `hidden`)
    for (int k = 0; k < st->nkeys; k++) {  // group columns first (aggregate.rs:890-925)
      DevColumn c;
      c.dtype = st->key_dtypes[size_t(k)];
      if (st->wide && st->key_is_utf8[size_t(k)]) {
        // references to the groups' strings come out of the compaction; the strings are gathered below
        c.dtype = DFGPU_UINT64;
        c.values_bytes = alloc_n * 8;
        c.values = ctx->alloc(c.values_bytes);
        wide_refs.push_back({k, hidden.cols.size()});
        hidden.cols.push_back(c);
        DevColumn u;
        u.dtype = DFGPU_UTF8;
        res->cols.push_back(u);
        cp.out_keys[k] = c.values;
        cp.key_dtype[k] = DFGPU_UINT64;
        continue;
      }
      c.values_bytes = alloc_n * size_t(dtype_width(c.dtype));
      c.values = ctx->alloc(c.values_bytes);
      if (st->utf8_key) {
        hidden.cols.push_back(c);
        DevColumn u;
        u.dtype = DFGPU_UTF8;  // filled by the gather below
        res->cols.push_back(u);
      } else {
        res->cols.push_back(c);
      }
      cp.out_keys[k] = c.values;
      cp.key_dtype[k] = c.dtype;
      cp.key_mask[k] = st->key_mask[size_t(k)];
      cp.key_shift[k] = st->key_shift[size_t(k)];
    }
    for (int a = 0; a < st->naggs; a++) {  // then aggregate columns (aggregate.rs:928-949)
      DevColumn c;
      c.dtype = st->descs[size_t(a)].out_dtype;
      c.values_bytes = alloc_n * size_t(dtype_width(c.dtype));
      c.values = ctx->alloc(c.values_bytes);
      if (st->utf8_key && a == st->naggs - 1) hidden.cols.push_back(c);  // representative rows: not a result column
      else res->cols.push_back(c);
      cp.out_vals[a] = c.values;
      cp.aggs[a] = st->descs[size_t(a)];
    }
    if (xn >= 0) {
      // the merged global rows came back from the exchange: decode them (same rows, same order on every rank)
      DecodeParams dp;
      memset(&dp, 0, sizeof(dp));
      dp.rows = xrows;
      dp.n = xn;
      dp.nseg = xseg.nseg;
      dp.seg_stride = xseg.stride;
      for (int r = 0; r < xseg.nseg; r++) dp.seg_n[r] = xseg.n[r];
      dp.nkeys = st->nkeys;
      dp.naggs = st->naggs;
      for (int k = 0; k < st->nkeys; k++) {
        dp.key_mask[k] = cp.key_mask[k];
        dp.key_shift[k] = cp.key_shift[k];
        dp.key_dtype[k] = cp.key_dtype[k];
        dp.out_keys[k] = cp.out_keys[k];
      }
      for (int a = 0; a < st->naggs; a++) {
        dp.aggs[a] = cp.aggs[a];
        dp.out_vals[a] = cp.out_vals[a];
      }
      if (xn > 0) launch_kernel(ctx, k_decode_rows, "k_decode_rows", dp, xn, 256, 8);
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
    } else {
      DF_CUDA(cudaMemsetAsync(st->d_counters + CTR_COMPACT, 0, 8, ctx->stream));
      cp.counter = st->d_counters + CTR_COMPACT;
      launch_kernel(ctx, k_compact, "k_compact", cp, st->t.cap + 1, 256, 8);
      if ((long long)read_counter(st, CTR_COMPACT) != cnt) fail(DFGPU_ERR_INTERNAL, "table compaction count mismatch");
    }
    res->nrows = cnt;
    for (auto& wr : wide_refs)  // wide keys: the Utf8 parts' strings, in output order
      gather_utf8_multi(ctx, st->d_utf8_srcs, (const unsigned long long*)hidden.cols[wr.second].values, cnt, &res->cols[size_t(wr.first)]);
    if (st->utf8_key)  // key strings = the representatives' strings, in output order
      gather_utf8_multi(ctx, st->d_utf8_srcs, (const unsigned long long*)hidden.cols[1].values, cnt, &res->cols[0]);
    if (st->nkeys == 0) {
      // an aggregate that saw no non-null input is null (array_from_scalar!, aggregate.rs:641-643)
      std::vector<long long> nonnull = st->nonnull_host;
      if (st->saw_nulls) {
        unsigned long long d[kMaxAggs];
        read_words(ctx, st->d_counters + CTR_NONNULL, sizeof(d), d);
        for (int a = 0; a < st->naggs; a++) nonnull[size_t(a)] += (long long)d[a];
      }
      std::vector<char> avg_word(size_t(st->naggs), 0);  // an AVG's validity comes from its count word (k_avg_finish)
      for (size_t i = 0; i < st->out_word.size(); i++)
        if (st->out_is_avg[i]) avg_word[size_t(st->out_word[i])] = avg_word[size_t(st->out_word[i]) + 1] = 1;
      for (int a = 0; a < st->naggs; a++) {
        if (avg_word[size_t(a)] || nonnull[size_t(a)] > 0 || (st->rows_seen > 0 && st->descs[size_t(a)].func == DFGPU_AGG_COUNT)) continue;
        DevColumn& c = res->cols[size_t(a)];
        c.validity = (uint8_t*)ctx->alloc(1);
        DF_CUDA(cudaMemsetAsync(c.validity, 0, 1, ctx->stream));
        c.null_count = 1;
      }
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (!st->emit_words) assemble_outputs(st, res.get());
    tr.mark("finish (compact + outputs)");
    st->finished = true;
    *out = res.release();
  });
}

extern "C" int dfgpu_aggregate_free(dfgpu_aggstate* st) {
  return guarded([&] {
    if (st) st->ctx->use();
    delete st;
  });
}
