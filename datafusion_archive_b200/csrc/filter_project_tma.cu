// filter_project_tma.cu — the production filter+project kernel: persistent, warp-specialised,
// fed by the TMA engine, with the predicate running far ahead of the projection.
//
// Roles inside one CTA (one CTA per SM, cooperative launch, tiles assigned round-robin: in "wave"
// `it` CTA c owns tile it*G + c):
//
//   producer A (1 warp) : one elected lane streams the PREDICATE columns of tile it into ring A with
//                         cp.async.bulk (SASS UBLKCP), completion tracked by mbarrier tx counts
//   producer B (1 warp) : streams the PROJECTION columns of tile it-LAG into ring B the same way —
//                         a re-read of bytes fetched LAG tiles earlier, served by the 50 MB L2
//   16 consumer warps   : phase 1 = predicate of tile it over ring A -> K flag bits per lane, kept in
//                         a 64-bit shift register; phase 2 = projections of tile it-LAG over ring B,
//                         selected rows stored at their compacted global position
//   1 scan warp         : turns the per-warp counts of a tile into global output offsets, one wave per
//                         step, a fixed delay behind publishing the counts
//
// Why the lag: order-preserving compaction needs, per tile, the number of selected rows in ALL
// earlier tiles.  Under a bandwidth-saturating stream every dependent global round trip costs
// microseconds, far longer than a tile's HBM time (~0.5 us), and a tile cannot wait in shared
// memory that long (bandwidth x latency exceeds the SM's storage).  So the predicate pass, which
// only produces 1 bit per row, runs LAG tiles ahead; by the time the projection pass reaches a
// tile its offset has long been resolved, and the tile's bytes come back from L2, not HBM.
//
// Offsets: in step w the scan warp publishes the count of its tile of wave w to tile_status, then
// RESOLVES wave w - D: it gathers the counts of all G tiles of that wave (offset = base + sum(counts
// of lower CTAs) + the warp's offset inside the tile); base advances by the wave total, computed
// redundantly by every CTA (nothing is forwarded between waves through memory).  The status loads
// of wave w - D are issued before the step waits for the counts of wave w, so their L2 round trip
// overlaps the predicate pass; every CTA published wave w - D about D waves earlier, so a re-poll
// of a status not yet written is rare.  The offsets of wave j are ready right after the counts of
// wave j + D, so the lag must be >= D (the consumers reach the projection pass of wave j right
// after the predicate pass of wave j + LAG), and every wave gets the same slack.
//
// Nothing in the CTA executes __syncthreads in the steady state; all hand-offs are mbarriers.
// Reference path replaced: src/execution/filter.rs:46-110 + src/execution/projection.rs:46-66.
#include "filter_project.cuh"

namespace dfgpu {

constexpr int TM_CWARPS = 16;  // consumer warps
// one scan warp: its status loads fly while it waits for the next tile's counts, so a second warp taking every
// other wave was 2-8 % slower on H100 (C2, C3).  19 warps leave 96 registers per thread, as 20 did.
constexpr int TM_WARPS = TM_CWARPS + 2 + 1;
constexpr int TM_THREADS = TM_WARPS * 32;
constexpr int TM_MAX_STAGES = 8;
constexpr int TM_MAX_LAG = 24;
constexpr int TM_MAX_DELAY = 8;
// slots of the count/offset hand-off rings.  The slot of wave w is reused by wave w + TM_RING, whose publish
// rewrites s_off; that publish waits for the counts of wave w + TM_RING, which the consumers only report after
// reading the offsets of wave w + TM_RING - 1 - lag.  So TM_RING >= lag + 1 keeps every slot alive until read.
constexpr int TM_RING = 32;
static_assert(TM_RING >= TM_MAX_LAG + 1, "hand-off ring too short for the longest lag");
constexpr int TM_MAX_GRID = 160;  // CTAs (= SMs) the wave gather is written for (H100 SXM: 132)
constexpr int TM_HDR_BYTES = 8192;
constexpr int TM_SMEM_BUDGET = 200 * 1024;
// upper bound of one hardware suspension in mbarrier.try_wait: a waiting warp sleeps until the phase
// completes (or this long) instead of re-issuing the poll; ncu showed 22 % of all issued instructions in
// the poll loop with the default (short) limit
constexpr unsigned TM_WAIT_HINT_NS = 4000;

// ---- mbarrier / bulk-copy PTX ----------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n"
      "@P1 bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity), "r"(TM_WAIT_HINT_NS)
      : "memory");
}
// the same on 32-bit shared-window addresses kept in registers (the lean consumer loop: no generic -> shared
// conversion, S2UR SR_CgaCtaId + ULEA, in front of every barrier operation)
__device__ __forceinline__ void mbar_arrive_a(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n"
      "@P1 bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(bar), "r"(parity), "r"(TM_WAIT_HINT_NS)
      : "memory");
}
// 1-D bulk async copy global -> shared, completion reported to an mbarrier (TMA engine; UBLKCP),
// with an L2 eviction-priority hint: the predicate stream marks bytes that the projection stream
// will re-read LAG tiles later as evict_last; the projection stream (and bytes read once) use
// evict_first so they do not push the pending re-reads out of L2.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar,
                                            unsigned long long policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

struct TmaShared {
  unsigned long long fullA[TM_MAX_STAGES], emptyA[TM_MAX_STAGES];  // ring A (predicate columns)
  unsigned long long fullB[TM_MAX_STAGES], emptyB[TM_MAX_STAGES];  // ring B (projection columns)
  unsigned long long cnt_ready[TM_RING];   // consumers -> scan warp: per-warp counts of a tile are in s_cnt
  unsigned long long pfx_ready[TM_RING];   // scan warp -> consumers: global offsets of a tile are in s_off
  unsigned long long s_off[TM_RING][TM_CWARPS];
  unsigned s_cnt[TM_RING][TM_CWARPS];
};
static_assert(sizeof(TmaShared) <= TM_HDR_BYTES, "shared header too large");

// One producer warp: stream the `ncols` columns listed in `slots` of every tile this CTA owns into
// a ring of S stages.
__device__ __forceinline__ void producer_loop(const FPParams& p, int tile_rows, const int* col_off, const int* reread_off, unsigned char* ring,
                                              int S, int stage_bytes, unsigned long long* full, unsigned long long* empty, int lane) {
  const unsigned long long keep = l2_policy_evict_last(), stream = l2_policy_evict_first();
  int s = 0;
  unsigned ph = 1;  // first pass over the ring returns immediately
  for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
    mbar_wait(&empty[s], ph);
    unsigned char* dst = ring + (size_t)s * stage_bytes;
    const long long row0 = (long long)tile * tile_rows;
    const long long left = p.nrows - row0;
    if (left >= tile_rows) {
      if (lane == 0) {
        unsigned total = 0;
        for (int c = 0; c < p.ps.ncols; c++)
          if (col_off[c] >= 0) total += (unsigned)(tile_rows * p.col_w[c]);
        mbar_arrive_expect_tx(&full[s], total);
        for (int c = 0; c < p.ps.ncols; c++)
          if (col_off[c] >= 0)
            tma_load_1d(dst + col_off[c], (const unsigned char*)p.ps.cols[c].ptr + row0 * p.col_w[c], (unsigned)(tile_rows * p.col_w[c]),
                        &full[s], (reread_off && reread_off[c] >= 0) ? keep : stream);
      }
    } else {
      // ragged last tile: sizes need not be 16-byte multiples, so the warp copies it by hand
      for (int c = 0; c < p.ps.ncols; c++) {
        if (col_off[c] < 0) continue;
        const unsigned char* src = (const unsigned char*)p.ps.cols[c].ptr + row0 * p.col_w[c];
        const long long nb = left * p.col_w[c];
        for (long long b = lane; b < nb; b += 32) dst[col_off[c] + b] = src[b];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[s]);
    }
    if (++s == S) { s = 0; ph ^= 1u; }
  }
}

// one comparison over the K rows of this lane -> K flag bits (operands straight from the staged tile)
template <int K, class T>
__device__ __forceinline__ unsigned cmp_term_t(const Leaf& t, const unsigned char* stage, const int* col_off, int lrow0, T imm) {
  const T* A = (const T*)(stage + col_off[t.a]) + lrow0;
  const bool bcol = t.kind == 2;
  const T* B = bcol ? (const T*)(stage + col_off[t.b]) + lrow0 : A;
  unsigned flags = 0;
#define DF_CMP(OPR)                                                                                    \
  if (bcol) {                                                                                          \
    _Pragma("unroll") for (int k = 0; k < K; k++) flags |= (unsigned)(A[k * 32] OPR B[k * 32]) << k;   \
  } else {                                                                                             \
    _Pragma("unroll") for (int k = 0; k < K; k++) flags |= (unsigned)(A[k * 32] OPR imm) << k;         \
  }
  switch (t.op) {
    case V_EQ: DF_CMP(==) break;
    case V_NE: DF_CMP(!=) break;
    case V_LT: DF_CMP(<) break;
    case V_LE: DF_CMP(<=) break;
    case V_GT: DF_CMP(>) break;
    default: DF_CMP(>=) break;
  }
#undef DF_CMP
  return flags;
}
template <int K, bool F64>
__device__ __forceinline__ unsigned cmp_term(const Leaf& t, const unsigned char* stage, const int* col_off, int lrow0) {
  if (F64) return cmp_term_t<K, double>(t, stage, col_off, lrow0, u2d(t.imm));
  switch (t.dtype) {
    case DFGPU_FLOAT64: return cmp_term_t<K, double>(t, stage, col_off, lrow0, u2d(t.imm));
    case DFGPU_INT64: return cmp_term_t<K, long long>(t, stage, col_off, lrow0, (long long)t.imm);
    case DFGPU_UINT64: return cmp_term_t<K, unsigned long long>(t, stage, col_off, lrow0, t.imm);
    case DFGPU_FLOAT32: return cmp_term_t<K, float>(t, stage, col_off, lrow0, u2f(t.imm));
    case DFGPU_INT32: return cmp_term_t<K, int>(t, stage, col_off, lrow0, (int)(long long)t.imm);
    default: return cmp_term_t<K, unsigned>(t, stage, col_off, lrow0, (unsigned)t.imm);
  }
}

// one arithmetic operation over the K rows of this lane (Float64 / Float32 / 64-bit integers)
template <int K, class T>
__device__ __forceinline__ void arith_term_t(const Leaf& t, const unsigned char* stage, const int* col_off, int lrow0, T imm, unsigned flags,
                                             bool& bad, T (&out)[K]) {
  const T* A = (const T*)(stage + col_off[t.a]) + lrow0;
  const bool bcol = t.kind == 2;
  const T* B = bcol ? (const T*)(stage + col_off[t.b]) + lrow0 : A;
  T y[K];
#pragma unroll
  for (int k = 0; k < K; k++) y[k] = bcol ? B[k * 32] : imm;
  switch (t.op) {
    case V_ADD:
#pragma unroll
      for (int k = 0; k < K; k++) out[k] = A[k * 32] + y[k];
      break;
    case V_SUB:
#pragma unroll
      for (int k = 0; k < K; k++) out[k] = A[k * 32] - y[k];
      break;
    case V_MUL:
#pragma unroll
      for (int k = 0; k < K; k++) out[k] = A[k * 32] * y[k];
      break;
    default:  // V_DIV: floating point only (the host does not select integer division as a fast shape)
#pragma unroll
      for (int k = 0; k < K; k++) {
        if (y[k] == T(0) && ((flags >> k) & 1u)) bad = true;  // DivideByZero on a surviving row
        out[k] = A[k * 32] / y[k];
      }
      break;
  }
}

// ---- lean consumer loop ---------------------------------------------------------------------------
// The shapes the headline configurations have (C2: SELECT a WHERE a > c; C3: SELECT a+b, a*b WHERE b < a): ONE
// Float64 comparison as the predicate and one or two projections that copy an 8-byte column or combine Float64
// operands.  In the generic FAST loop most instructions per warp-tile re-derive per-tile invariants — indexed
// constant-bank loads of the column offsets behind the term's column index, a jump table on the comparison
// operator, generic -> shared address conversions in front of every mbarrier operation — and their dependent
// latencies are what the 4 consumer warps per scheduler cannot hide.  Here the comparison operator and the operand kind are template
// parameters, every offset, pointer and barrier address is computed once before the loop, and the loop body is
// waits + loads + compares + the ballot-compacted store.  Protocol (barriers, rings, scan warp) unchanged.
template <int CMP, class T>
__device__ __forceinline__ bool lean_cmp_t(T a, T b) {
  if (CMP == V_EQ) return a == b;
  if (CMP == V_NE) return a != b;
  if (CMP == V_LT) return a < b;
  if (CMP == V_LE) return a <= b;
  if (CMP == V_GT) return a > b;
  return a >= b;
}
// TY: 0 = Float64, 1 = Int64, 2 = UInt64 (operands as raw 8-byte words)
template <int CMP, int TY>
__device__ __forceinline__ bool lean_cmp(unsigned long long a, unsigned long long b) {
  if (TY == 0) return lean_cmp_t<CMP, double>(u2d(a), u2d(b));
  if (TY == 1) return lean_cmp_t<CMP, long long>((long long)a, (long long)b);
  return lean_cmp_t<CMP, unsigned long long>(a, b);
}

// predicated 8-byte store (the compiler turns `if (selected) out[pos] = v` into a divergent branch per row when the
// value's load can be sunk into it; the compacted store wants @P STG)
__device__ __forceinline__ void st_if(unsigned cond, unsigned long long* dst, unsigned long long v) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.u32 p, %0, 0;\n"
      "@p st.global.b64 [%1], %2;\n"
      "}\n" ::"r"(cond), "l"(dst), "l"(v)
      : "memory");
}

// 8-byte load from a 32-bit shared-window address (ordered with the mbarrier operations around it: volatile + memory)
__device__ __forceinline__ unsigned long long lds64(unsigned addr) {
  unsigned long long v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
  return v;
}

// One row slot of the ballot compaction, fused: p = (flags & bit) != 0; m = ballot(p); pos = run + popc(m & lanes
// below); @p store v at o[pos]; run += popc(m).  One predicate feeds the vote and the store (the C++ form costs a
// shift + and + compare for the vote and an and + compare again for the store).
__device__ __forceinline__ unsigned compact_store(unsigned flags, unsigned bit, unsigned lt_mask, unsigned& run, unsigned long long* o, unsigned long long v) {
  unsigned pos;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .b32 m, t;\n"
      ".reg .b64 a;\n"
      "and.b32 t, %2, %3;\n"
      "setp.ne.u32 p, t, 0;\n"
      "vote.sync.ballot.b32 m, p, 0xffffffff;\n"
      "and.b32 t, m, %4;\n"
      "popc.b32 t, t;\n"
      "add.u32 %1, t, %0;\n"
      "mad.wide.u32 a, %1, 8, %5;\n"
      "@p st.global.b64 [a], %6;\n"
      "popc.b32 m, m;\n"
      "add.u32 %0, %0, m;\n"
      "}\n"
      : "+r"(run), "=&r"(pos)
      : "r"(flags), "r"(bit), "r"(lt_mask), "l"(o), "l"(v)
      : "memory");
  return pos;
}

constexpr int LEAN_MAX_PROJ = 2;

template <int K, int CMP, bool PB, int NP, int TY>
__device__ __forceinline__ void consumer_lean(const FPParams& p, int warp, int lane) {
  extern __shared__ __align__(128) unsigned char smem_raw[];  // the kernel's dynamic shared memory: 32-bit shared-window arithmetic below
  TmaShared& sh = *reinterpret_cast<TmaShared*>(smem_raw);
  constexpr int TILE = TM_CWARPS * 32 * K;
  constexpr unsigned KMASK = (1u << K) - 1u;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int first = blockIdx.x, step = gridDim.x;
  const int nloc = first < p.ntiles ? (p.ntiles - first + step - 1) / step : 0;
  const int SA = p.nstagesA, SB = p.nstagesB, LAG = p.lag;
  const int last_it = (p.ntiles - 1 - first) % step == 0 ? (p.ntiles - 1 - first) / step : -1;  // the only ragged tile, if this CTA owns it
  unsigned sh0 = smem_u32(smem_raw);
  asm volatile("" : "+r"(sh0));  // one register for every barrier address: do not re-derive the shared-window base at every use
  constexpr unsigned b_fullA = (unsigned)offsetof(TmaShared, fullA), b_emptyA = (unsigned)offsetof(TmaShared, emptyA);
  constexpr unsigned b_fullB = (unsigned)offsetof(TmaShared, fullB), b_emptyB = (unsigned)offsetof(TmaShared, emptyB);
  constexpr unsigned b_cnt = (unsigned)offsetof(TmaShared, cnt_ready), b_pfx = (unsigned)offsetof(TmaShared, pfx_ready);
  // operand offsets (bytes from the start of shared memory) in stage 0
  const int lrow0 = warp * 32 * K + lane;
  const Leaf& pt = p.pred_fast.term[0];
  const unsigned long long pimm = pt.imm;
  const int ringA_off = TM_HDR_BYTES, stageA = p.stage_bytesA;
  const int ringB_off = TM_HDR_BYTES + SA * stageA, stageB = p.stage_bytesB;
  const unsigned a1 = sh0 + (unsigned)(ringA_off + p.col_offA[pt.a] + lrow0 * 8);  // shared-window addresses: LDS [R + imm], nothing to derive per tile
  const unsigned b1 = PB ? sh0 + (unsigned)(ringA_off + p.col_offA[pt.b] + lrow0 * 8) : a1;
  unsigned a2[NP], b2[NP];
  int kop2[NP];
  unsigned long long imm2[NP];
  unsigned long long* out2[NP];
#pragma unroll
  for (int q = 0; q < NP; q++) {
    const Leaf& fo = p.proj_fast[q];
    // -1 copy; op (+0x100: the right operand is the immediate; +0x200: 64-bit integer arithmetic, two's complement wrap-around)
    kop2[q] = fo.kind == 1 ? -1 : ((fo.kind == 2 ? fo.op : fo.op | 0x100) | (fo.dtype == DFGPU_FLOAT64 ? 0 : 0x200));
    imm2[q] = fo.imm;
    a2[q] = sh0 + (unsigned)(ringB_off + p.col_offB[fo.a] + lrow0 * 8);
    b2[q] = fo.kind == 2 ? sh0 + (unsigned)(ringB_off + p.col_offB[fo.b] + lrow0 * 8) : a2[q];
    out2[q] = (unsigned long long*)p.out[q];
  }
  bool bad = false;
  unsigned __int128 fl = 0;  // flag bits of the last LAG+1 tiles, K per tile
  int sa = 0, sb = 0;
  unsigned pha = 0, phb = 0;
  for (int it = 0; it < nloc + LAG; it++) {
    unsigned f0 = 0;
    if (it < nloc) {
      // ---- predicate of tile `it` -> K flag bits, the warp's count to the scan warp
      mbar_wait_a(sh0 + b_fullA + 8u * sa, pha);
      const unsigned A = a1 + (unsigned)(sa * stageA), B = b1 + (unsigned)(sa * stageA);
      unsigned long long x[K], y[K];
#pragma unroll
      for (int k = 0; k < K; k++) x[k] = lds64(A + k * 256);
#pragma unroll
      for (int k = 0; k < K; k++) y[k] = PB ? lds64(B + k * 256) : pimm;
#pragma unroll
      for (int k = 0; k < K; k++) f0 |= (unsigned)lean_cmp<CMP, TY>(x[k], y[k]) << k;
      if (it == last_it) {
        const long long row0 = ((long long)first + (long long)it * step) * TILE + lrow0;
        unsigned valid = 0;
#pragma unroll
        for (int k = 0; k < K; k++)
          if (row0 + k * 32 < p.nrows) valid |= 1u << k;
        f0 &= valid;
      }
      const unsigned cnt = __reduce_add_sync(0xffffffffu, (unsigned)__popc(f0));
      if (lane == 0) {
        mbar_arrive_a(sh0 + b_emptyA + 8u * sa);  // this warp is done reading the stage
        sh.s_cnt[it % TM_RING][warp] = cnt;
        mbar_arrive_a(sh0 + b_cnt + 8u * (it % TM_RING));
      }
      if (++sa == SA) { sa = 0; pha ^= 1u; }
    }
    fl = (fl << K) | (unsigned __int128)f0;
    if (it >= LAG) {
      // ---- projections of tile it - LAG: selected rows go to their compacted global position
      const int j = it - LAG;
      const unsigned flags = (unsigned)(fl >> (K * LAG)) & KMASK;
      mbar_wait_a(sh0 + b_pfx + 8u * (j % TM_RING), (j / TM_RING) & 1);
      const unsigned long long base = sh.s_off[j % TM_RING][warp];
      mbar_wait_a(sh0 + b_fullB + 8u * sb, phb);
      // projection values of the K rows of this lane, then the ballot compaction: the rank of a selected row inside the
      // warp's slice (row order: k major, lane minor) is computed while the first projection is stored
      unsigned pos[K];
#pragma unroll
      for (int q = 0; q < NP; q++) {
        const unsigned A = a2[q] + (unsigned)(sb * stageB);
        unsigned long long* o = out2[q] + base;
        unsigned long long v[K];
        if (kop2[q] < 0) {
#pragma unroll
          for (int k = 0; k < K; k++) v[k] = lds64(A + k * 256);
        } else {
          const unsigned B = b2[q] + (unsigned)(sb * stageB);
          const bool rimm = (kop2[q] & 0x100) != 0;
          const int op = kop2[q] & 0xff;
          unsigned long long y[K];
#pragma unroll
          for (int k = 0; k < K; k++) v[k] = lds64(A + k * 256);
#pragma unroll
          for (int k = 0; k < K; k++) y[k] = rimm ? imm2[q] : lds64(B + k * 256);
          if (kop2[q] & 0x200) {  // Int64 / UInt64: + - * (the host keeps integer division out of the fast shapes)
            if (op == V_ADD) {
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = v[k] + y[k];
            } else if (op == V_MUL) {
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = v[k] * y[k];
            } else {
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = v[k] - y[k];
            }
          } else if (op == V_ADD) {
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = d2u(u2d(v[k]) + u2d(y[k]));
          } else if (op == V_MUL) {
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = d2u(u2d(v[k]) * u2d(y[k]));
          } else if (op == V_SUB) {
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = d2u(u2d(v[k]) - u2d(y[k]));
          } else {  // V_DIV
#pragma unroll
            for (int k = 0; k < K; k++) {
              if (u2d(y[k]) == 0.0 && (flags & (1u << k))) bad = true;  // DivideByZero on a surviving row
              v[k] = d2u(u2d(v[k]) / u2d(y[k]));
            }
          }
        }
        if (q == 0) {
          unsigned run = 0;
#pragma unroll
          for (int k = 0; k < K; k++) pos[k] = compact_store(flags, 1u << k, lt_mask, run, o, v[k]);
        } else {
#pragma unroll
          for (int k = 0; k < K; k++) st_if(flags & (1u << k), o + pos[k], v[k]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_a(sh0 + b_emptyB + 8u * sb);
      if (++sb == SB) { sb = 0; phb ^= 1u; }
    }
  }
  if (bad) *p.err_flag = 1u;
}

template <int K, int NP, int TY>
__device__ __forceinline__ void consumer_lean_ops(const FPParams& p, int warp, int lane) {
  const int op = p.pred_fast.term[0].op;
  const bool pb = p.pred_fast.term[0].kind == 2;
#define DF_LEAN(OP)                                                \
  case OP:                                                         \
    if (pb) consumer_lean<K, OP, true, NP, TY>(p, warp, lane);     \
    else consumer_lean<K, OP, false, NP, TY>(p, warp, lane);       \
    break;
  switch (op) {
    DF_LEAN(V_EQ)
    DF_LEAN(V_NE)
    DF_LEAN(V_LT)
    DF_LEAN(V_LE)
    DF_LEAN(V_GT)
    default:
      if (pb) consumer_lean<K, V_GE, true, NP, TY>(p, warp, lane);
      else consumer_lean<K, V_GE, false, NP, TY>(p, warp, lane);
      break;
  }
#undef DF_LEAN
}
template <int K, int NP>
__device__ __forceinline__ void consumer_lean_dispatch(const FPParams& p, int warp, int lane) {
  const int ty = p.pred_fast.term[0].dtype;
  if (ty == DFGPU_FLOAT64) consumer_lean_ops<K, NP, 0>(p, warp, lane);
  else if (ty == DFGPU_INT64) consumer_lean_ops<K, NP, 1>(p, warp, lane);
  else consumer_lean_ops<K, NP, 2>(p, warp, lane);
}

// FAST: every program of the query is a fast shape, so the interpreter is not even compiled into
// this instantiation (fewer registers, smaller code).  FAST + F64ONLY: additionally every operand is
// Float64, and the per-type dispatch of the fast shapes disappears too (the C2 / C3 kernels).
template <int DEPTH, int K, bool F64ONLY, bool FAST, int LEAN = 0>  // LEAN = number of projections of a lean shape
__global__ void __launch_bounds__(TM_THREADS, 1) k_filter_project_tma(const __grid_constant__ FPParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int TILE = TM_CWARPS * 32 * K;
  TmaShared& sh = *reinterpret_cast<TmaShared*>(smem_raw);
  unsigned char* ringA = smem_raw + TM_HDR_BYTES;
  unsigned char* ringB = ringA + (size_t)p.nstagesA * p.stage_bytesA;
  const int SA = p.nstagesA, SB = p.nstagesB;
  const int LAG = p.lag;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < TM_MAX_STAGES; s++) {
      mbar_init(&sh.fullA[s], 1);
      mbar_init(&sh.emptyA[s], TM_CWARPS);
      mbar_init(&sh.fullB[s], 1);
      mbar_init(&sh.emptyB[s], TM_CWARPS);
    }
    for (int i = 0; i < TM_RING; i++) {
      mbar_init(&sh.cnt_ready[i], TM_CWARPS);
      mbar_init(&sh.pfx_ready[i], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int first = blockIdx.x, step = gridDim.x;

  if (warp == TM_CWARPS) {
    // ================================ producer A: predicate columns ============================
    if (p.has_pred) producer_loop(p, TILE, p.col_offA, p.col_offB, ringA, SA, p.stage_bytesA, sh.fullA, sh.emptyA, lane);
  } else if (warp == TM_CWARPS + 1) {
    // ================================ producer B: projection columns ===========================
    // Runs as far ahead as ring B allows; the consumers reach these tiles LAG iterations after the
    // predicate pass touched the same rows, so the bytes are L2 hits.
    producer_loop(p, TILE, p.col_offB, nullptr, ringB, SB, p.stage_bytesB, sh.fullB, sh.emptyB, lane);
  } else if (warp == TM_CWARPS + 2) {
    // ================================ scan warp =================================================
    if (!p.has_pred) return;  // nothing is dropped: output positions are the row numbers
    const int D = p.delay;
    int nloc = 0;
    for (int tile = first; tile < p.ntiles; tile += step) nloc++;
    unsigned long long base = 0;  // selected rows in all waves before the one being resolved
    // Step w publishes wave w and resolves wave w - D; the last D steps only resolve.
    for (int w = 0; w < nloc + D; w++) {
      const int v = w - D;  // the wave this step resolves
      const long long wave0 = (long long)v * step;
      // 1. the statuses of every tile of wave v, all loads issued before this step waits for its own counts:
      //    the L2 round trip overlaps the predicate pass of wave w
      unsigned long long sv[TM_MAX_GRID / 32];
#pragma unroll
      for (int g = 0; g < TM_MAX_GRID / 32; g++) {
        const int j = g * 32 + lane;
        sv[g] = (v >= 0 && j < step && wave0 + j < p.ntiles) ? ld_relaxed(&p.tile_status[wave0 + j]) : ST_AGG;
      }
      // 2. publish wave w: per-warp counts -> exclusive offsets inside the tile, parked in s_off until the wave is
      //    resolved; the tile total goes to tile_status
      if (w < nloc) {
        const int b = w % TM_RING;
        mbar_wait(&sh.cnt_ready[b], (w / TM_RING) & 1);
        const unsigned c = lane < TM_CWARPS ? sh.s_cnt[b][lane] : 0u;
        unsigned incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
        if (lane == 0) st_relaxed(&p.tile_status[first + w * step], ST_AGG | total);
        if (lane < TM_CWARPS) sh.s_off[b][lane] = incl - c;
      }
      if (v < 0) continue;
      // 3. resolve wave v: re-poll only the statuses that were still unpublished, all of them at once
      for (;;) {
        bool missing = false;
#pragma unroll
        for (int g = 0; g < TM_MAX_GRID / 32; g++) {
          if ((sv[g] >> 62) == 0) {
            missing = true;
            sv[g] = ld_relaxed(&p.tile_status[wave0 + g * 32 + lane]);
          }
        }
        if (!__any_sync(0xffffffffu, missing)) break;
      }
      unsigned long long bf = 0, wt = 0;
#pragma unroll
      for (int g = 0; g < TM_MAX_GRID / 32; g++) {
        const unsigned long long c = sv[g] & ST_MASK;
        wt += c;
        if (g * 32 + lane < (int)blockIdx.x) bf += c;
      }
      const unsigned long long before = warp_sum64(bf), wave_total = warp_sum64(wt);
      const int b = v % TM_RING;
      if (lane < TM_CWARPS) sh.s_off[b][lane] += base + before;
      base += wave_total;
      // the last tile is the highest of its wave: everything up to and including it is the new base
      if (lane == 0 && first + v * step == p.ntiles - 1) *p.out_count = base;
      __syncwarp();
      if (lane == 0) mbar_arrive(&sh.pfx_ready[b]);
    }
  } else if constexpr (LEAN > 0) {
    // ================================ consumer warps, lean shapes ================================
    consumer_lean_dispatch<K, LEAN>(p, warp, lane);
  } else {
    // ================================ consumer warps ============================================
    const unsigned lt_mask = (1u << lane) - 1u;
    constexpr unsigned KMASK = (1u << K) - 1u;
    bool bad = false;

    // predicate of local iteration `it` -> K flag bits (bit k = row warp*32*K + k*32 + lane of the tile)
    auto phase1 = [&](int it, int tile, int s, unsigned ph) -> unsigned {
      mbar_wait(&sh.fullA[s], ph);
      StagedTile<K> src;
      src.stage = ringA + (size_t)s * p.stage_bytesA;
      src.col_off = p.col_offA;
      src.lrow0 = warp * 32 * K + lane;
      src.row0 = (long long)tile * TILE + src.lrow0;
      src.valid = KMASK;
      if (tile == p.ntiles - 1) {  // only the last tile can be ragged
        const long long row0 = src.row0;
        src.valid = 0;
#pragma unroll
        for (int k = 0; k < K; k++)
          if (row0 + k * 32 < p.nrows) src.valid |= 1u << k;
      }
      unsigned flags;
      if (FAST || p.pred_fast.nterms > 0) {
        // fast shape: Float64 comparisons straight from the staged tile, joined by AND / OR
        flags = cmp_term<K, FAST && F64ONLY>(p.pred_fast.term[0], src.stage, p.col_offA, src.lrow0);
        for (int t = 1; t < p.pred_fast.nterms; t++) {
          const unsigned ft = cmp_term<K, FAST && F64ONLY>(p.pred_fast.term[t], src.stage, p.col_offA, src.lrow0);
          flags = p.pred_fast.term[t].conn ? (flags | ft) : (flags & ft);
        }
      } else if constexpr (!FAST) {
        unsigned long long v[K];
        const unsigned b = eval_program<DEPTH, K, F64ONLY>(p.ps, 0, src, v);
        bad = bad || (b != 0);
        flags = 0;
#pragma unroll
        for (int k = 0; k < K; k++) flags |= (unsigned)(v[k] & 1ull) << k;
      }
      flags &= src.valid;
      // rows this warp selected in the tile: one population count per lane, one warp reduction (REDUX)
      const unsigned cnt = __reduce_add_sync(0xffffffffu, (unsigned)__popc(flags));
      if (lane == 0) {
        mbar_arrive(&sh.emptyA[s]);  // this warp is done reading the stage
        sh.s_cnt[it % TM_RING][warp] = cnt;
        mbar_arrive(&sh.cnt_ready[it % TM_RING]);
      }
      return flags;
    };

    // projections of local iteration `it`: selected rows go to their compacted global position
    auto phase2 = [&](int it, int tile, unsigned flags, int s, unsigned ph) {
      unsigned long long base;
      if (p.has_pred) {
        mbar_wait(&sh.pfx_ready[it % TM_RING], (it / TM_RING) & 1);
        base = sh.s_off[it % TM_RING][warp];
      } else {
        base = (unsigned long long)tile * TILE + (unsigned long long)warp * 32 * K;
      }
      StagedTile<K> src;
      mbar_wait(&sh.fullB[s], ph);
      src.stage = ringB + (size_t)s * p.stage_bytesB;
      src.col_off = p.col_offB;
      src.lrow0 = warp * 32 * K + lane;
      src.row0 = (long long)tile * TILE + src.lrow0;
      src.valid = flags;  // a zero divisor only matters on rows that survive the filter
      for (int q = 0; q < p.nproj; q++) {
        const int prog = q + p.has_pred;
        unsigned long long v[K];
        const Leaf& fo = p.proj_fast[q];
        if (fo.kind == 1 || (FAST && fo.kind < 2)) {
          if (FAST && F64ONLY) {
            const unsigned long long* A = (const unsigned long long*)(src.stage + p.col_offB[fo.a]) + src.lrow0;
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = A[k * 32];
          } else {
            src.load_rows(p.ps, fo.a, v);
          }
        } else if (fo.kind >= 2) {
          switch ((FAST && F64ONLY) ? (int)DFGPU_FLOAT64 : fo.dtype) {
            case DFGPU_FLOAT64: {
              double o[K];
              arith_term_t<K, double>(fo, src.stage, p.col_offB, src.lrow0, u2d(fo.imm), flags, bad, o);
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = d2u(o[k]);
              break;
            }
            case DFGPU_FLOAT32: {
              float o[K];
              arith_term_t<K, float>(fo, src.stage, p.col_offB, src.lrow0, u2f(fo.imm), flags, bad, o);
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = f2u(o[k]);
              break;
            }
            default: {  // Int64 / UInt64: two's complement wrap-around is the natural 64-bit result
              unsigned long long o[K];
              arith_term_t<K, unsigned long long>(fo, src.stage, p.col_offB, src.lrow0, fo.imm, flags, bad, o);
#pragma unroll
              for (int k = 0; k < K; k++) v[k] = o[k];
              break;
            }
          }
        } else if constexpr (!FAST) {
          const unsigned b = eval_program<DEPTH, K, F64ONLY>(p.ps, prog, src, v);
          bad = bad || (b != 0);
        }
        const int odt = p.ps.out_dtype[prog];
        const bool wide = (FAST && F64ONLY) || dtype_width_dev(odt) == 8;
        // warp-local base pointer once (64-bit), then 32-bit running offsets
        unsigned char* o = (unsigned char*)p.out[q] + base * (unsigned long long)(wide ? 8 : dtype_width_dev(odt));
        // compacted store; the element-width dispatch is warp-uniform and hoisted out of the row loop
#define DF_STORE_LOOP(TYPE)                                                        \
  {                                                                                \
    unsigned run = 0;                                                              \
    _Pragma("unroll") for (int k = 0; k < K; k++) {                                \
      const bool f = (flags >> k) & 1u;                                            \
      const unsigned m = __ballot_sync(0xffffffffu, f);                            \
      if (f) ((TYPE*)o)[run + __popc(m & lt_mask)] = (TYPE)v[k];                   \
      run += __popc(m);                                                            \
    }                                                                              \
  }
        if (wide) DF_STORE_LOOP(unsigned long long)
        else switch (dtype_width_dev(odt)) {
          case 4: DF_STORE_LOOP(unsigned) break;
          case 2: DF_STORE_LOOP(unsigned short) break;
          case 1: DF_STORE_LOOP(unsigned char) break;
          default: DF_STORE_LOOP(unsigned long long) break;
        }
#undef DF_STORE_LOOP
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sh.emptyB[s]);
    };

    int nloc = 0;
    for (int tile = first; tile < p.ntiles; tile += step) nloc++;
    int sb = 0;
    unsigned phb = 0;
    if (!p.has_pred) {
      // pure projection: no predicate pass, no lag
      for (int it = 0; it < nloc; it++) {
        const int tile = first + it * step;
        unsigned valid = KMASK;
        if (tile == p.ntiles - 1) {
          const long long row0 = (long long)tile * TILE + warp * 32 * K + lane;
          valid = 0;
#pragma unroll
          for (int k = 0; k < K; k++)
            if (row0 + k * 32 < p.nrows) valid |= 1u << k;
        }
        phase2(it, tile, valid, sb, phb);
        if (++sb == SB) { sb = 0; phb ^= 1u; }
      }
    } else {
      // software pipeline: predicate of tile it, projections of tile it - LAG; the flag bits of the
      // last LAG+1 tiles live in a 128-bit shift register (K bits per tile: up to 15 tiles of lag at K = 8)
      unsigned __int128 fl = 0;
      int sa = 0;
      unsigned pha = 0;
      for (int it = 0; it < nloc + LAG; it++) {
        unsigned f0 = 0;
        if (it < nloc) {
          f0 = phase1(it, first + it * step, sa, pha);
          if (++sa == SA) { sa = 0; pha ^= 1u; }
        }
        fl = (fl << K) | (unsigned __int128)f0;
        if (it >= LAG) {
          phase2(it - LAG, first + (it - LAG) * step, (unsigned)(fl >> (K * LAG)) & KMASK, sb, phb);
          if (++sb == SB) { sb = 0; phb ^= 1u; }
        }
      }
    }
    if (bad) *p.err_flag = 1u;
  }
}

template <int DEPTH, int K, bool F64ONLY, bool FAST, int LEAN = 0>
static void launch_one(dfgpu_ctx* ctx, const FPParams& p, size_t smem) {
  auto kern = k_filter_project_tma<DEPTH, K, F64ONLY, FAST, LEAN>;
  if (ctx->first_use((const void*)kern))
    DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TM_SMEM_BUDGET + 16384 + TM_HDR_BYTES));
  const int grid = std::min(std::min(ctx->sm_count, TM_MAX_GRID), p.ntiles);  // one persistent CTA per SM
  static const std::string name = "k_filter_project_tma<" + depth_arg(DEPTH) + ", " + std::to_string(K) + (F64ONLY ? ", true" : ", false") +
                                  (FAST ? ", true, " : ", false, ") + std::to_string(LEAN) + ">";
  // cooperative launch: the wave-synchronous scan needs every CTA of the grid resident at once
  launch(ctx, name.c_str(), kern, grid, TM_THREADS, LaunchOpts{smem, true, true}, p);
}

template <int DEPTH, int K>
static void launch_k(dfgpu_ctx* ctx, const FPParams& p, size_t smem) {
  bool fast = !p.has_pred || p.pred_fast.nterms > 0;
  for (int q = 0; q < p.nproj; q++) fast = fast && p.proj_fast[q].kind > 0;
  bool all_f64 = true;
  for (int c = 0; c < p.ps.ncols; c++) all_f64 = all_f64 && p.ps.cols[c].dtype == DFGPU_FLOAT64;
  // lean shapes: one comparison over 8-byte operands (Float64 / Int64 / UInt64), one or two copy / arithmetic projections over 8-byte columns (DFGPU_FP_LEAN=0: A/B switch)
  bool lean = fast && p.has_pred && p.pred_fast.nterms == 1 && is_numeric8(p.pred_fast.term[0].dtype) && p.nproj >= 1 && p.nproj <= LEAN_MAX_PROJ;
  for (int q = 0; lean && q < p.nproj; q++) lean = is_numeric8(p.proj_fast[q].dtype);  // copies and arithmetic over 8-byte columns only
  if (const char* e = getenv("DFGPU_FP_LEAN")) lean = lean && atoi(e) != 0;
  if (lean && p.nproj == 1) launch_one<1, K, true, true, 1>(ctx, p, smem);
  else if (lean) launch_one<1, K, true, true, 2>(ctx, p, smem);
  else if (fast && all_f64) launch_one<1, K, true, true>(ctx, p, smem);
  else if (fast) launch_one<1, K, false, true>(ctx, p, smem);
  else if (p.ps.f64_only) launch_one<DEPTH, K, true, false>(ctx, p, smem);
  else launch_one<DEPTH, K, false, false>(ctx, p, smem);
}

bool launch_fp_tma(dfgpu_ctx* ctx, FPParams& p) {
  if (p.ps.max_depth > 4 || p.ps.ncols < 1) return false;
  // which column slots does the predicate read, which do the projections read?
  bool inA[kMaxCols] = {}, inB[kMaxCols] = {};
  for (int prog = 0; prog < p.ps.nprog; prog++) {
    bool* dst = (p.has_pred && prog == 0) ? inA : inB;
    for (int pc = p.ps.start[prog]; pc < p.ps.start[prog + 1]; pc++) {
      const DevInsn& di = p.ps.insn[pc];
      if (di.op == V_PUSH_COL || (di.op > V_CAST && di.mode == RHS_COL)) dst[di.slot] = true;
    }
  }
  int rowA = 0, rowB = 0;
  for (int c = 0; c < p.ps.ncols; c++) {
    p.col_w[c] = dtype_width(p.ps.cols[c].dtype);
    if (p.col_w[c] <= 0) return false;
    if (inA[c]) rowA += p.col_w[c];
    if (inB[c]) rowB += p.col_w[c];
  }
  // projections of literals only, or a predicate over literals only: leave to the direct kernel
  if (rowB == 0 || (p.has_pred && rowA == 0)) return false;
  // Layout: ring A holds the predicate's columns, ring B the projections' columns.  A column in both rings is
  // loaded evict_last by producer A and re-read from L2 by producer B LAG tiles later; every other load is
  // evict_first.  Any width; the lag can be long.
  // Rows per lane K in {8,4,2}: the biggest tile that still gives both rings 3 stages.  Per-tile fixed
  // costs (barrier hand-offs, offset gather) outweigh deeper prefetch, so bigger tiles with few stages
  // beat smaller tiles with many.
  int K = 0;
  for (int k : {8, 4, 2}) {
    if (k == 8 && p.ps.max_depth > 2) continue;  // deep register stacks spill at 8 rows per lane
    const long long tile = (long long)TM_CWARPS * 32 * k;
    if (tile * (rowA + rowB) * 3 <= TM_SMEM_BUDGET) { K = k; break; }
  }
  if (const char* e = getenv("DFGPU_FP_K")) {  // experiment knob
    const int k = atoi(e);
    if ((k == 8 || k == 4 || k == 2) && (long long)TM_CWARPS * 32 * k * (rowA + rowB) * 2 <= TM_SMEM_BUDGET && !(k == 8 && p.ps.max_depth > 2)) K = k;
  }
  // program sets with scalar functions take one tile shape, 4 rows per lane: K = 8 holds too many live rows across the
  // function calls, and a set whose columns leave room for 2 rows only takes the direct kernel
  const bool fn = has_fn(p.ps);
  if (fn && K == 8) K = 4;
  if (!K || (fn && K != 4)) return false;
  const int tile = TM_CWARPS * 32 * K;
  int offA = 0, offB = 0;
  for (int c = 0; c < p.ps.ncols; c++) {
    // tile is a multiple of 512 rows: every column slice stays 128-B aligned
    p.col_offA[c] = inA[c] ? offA : -1;
    if (inA[c]) offA += tile * p.col_w[c];
    p.col_offB[c] = inB[c] ? offB : -1;
    if (inB[c]) offB += tile * p.col_w[c];
  }
  p.stage_bytesA = offA;
  p.stage_bytesB = offB;
  const int S = std::min(TM_MAX_STAGES, TM_SMEM_BUDGET / (offA + offB));
  p.nstagesA = offA ? S : 0;
  p.nstagesB = S;
  if (!p.has_pred) p.nstagesB = std::min(TM_MAX_STAGES, TM_SMEM_BUDGET / offB);
  if (const char* e = getenv("DFGPU_FP_STAGES")) {  // experiment knob: "A,B"
    int sa = 0, sb = 0;
    if (sscanf(e, "%d,%d", &sa, &sb) == 2 && sa >= 1 && sb >= 1 && sa <= TM_MAX_STAGES && sb <= TM_MAX_STAGES &&
        (long long)sa * offA + (long long)sb * offB <= TM_SMEM_BUDGET + 16384 && p.has_pred) {
      p.nstagesA = sa;
      p.nstagesB = sb;
    }
  }
  // delay: the scan warp resolves wave w - delay right after publishing wave w.  Its status loads are issued one
  // wave-time after the wave was published locally, so at delay 2 the other CTAs have published it too and the
  // re-poll is rare; delay 1 reads statuses the slower CTAs have not written yet (C3: 0.90 -> 0.86 ms at 2).
  // lag: at least the delay (the consumers wait for the offsets of tile it - lag right after reporting the
  // counts of tile it, and those are resolved in the scan step of tile it - lag + delay), as large as the flag
  // shift register allows (K bits per tile in 128 bits), but the bytes the projection stream will re-read
  // (lag x grid x stage B) must still be in L2 when it gets there.  On H100 (132 SMs, 50 MB L2) lag = delay = 2
  // was fastest for C2 and C3, whose projection stages re-read about 4.3 MB per wave; every extra wave of lag
  // cost 5-15 % (profiles/sweep_fp_lean.sh).
  p.lag = 0;
  p.delay = 2;
  if (const char* e = getenv("DFGPU_FP_DELAY")) {  // experiment knob
    const int d = atoi(e);
    if (d >= 1 && d <= TM_MAX_DELAY) p.delay = d;
  }
  const int max_lag = std::min(TM_MAX_LAG, 128 / K - 1);
  if (p.has_pred) {
    const long long l2_budget = 12ll << 20;  // a quarter of the 50 MB L2
    const long long per_tile = (long long)std::min(ctx->sm_count, TM_MAX_GRID) * offB;
    p.lag = (int)std::min<long long>(max_lag, std::max<long long>(p.delay, l2_budget / per_tile));
  }
  if (const char* e = getenv("DFGPU_FP_LAG")) {  // experiment knob
    const int l = atoi(e);
    if (p.has_pred && l >= p.delay && l <= max_lag) p.lag = l;
  }
  p.ntiles = int((p.nrows + tile - 1) / tile);
  const size_t smem = TM_HDR_BYTES + (size_t)p.nstagesA * p.stage_bytesA + (size_t)p.nstagesB * p.stage_bytesB;
  const int d = p.ps.max_depth;
  if (has_case(p.ps)) {
    if (p.ps.f64_only) launch_one<kCaseDepth, 4, true, false>(ctx, p, smem);
    else launch_one<kCaseDepth, 4, false, false>(ctx, p, smem);
  } else if (fn) {
    if (p.ps.f64_only) launch_one<kFnDepth, 4, true, false>(ctx, p, smem);
    else launch_one<kFnDepth, 4, false, false>(ctx, p, smem);
  } else if (K == 8) launch_k<2, 8>(ctx, p, smem);
  else if (K == 4) { if (d <= 2) launch_k<2, 4>(ctx, p, smem); else launch_k<4, 4>(ctx, p, smem); }
  else { if (d <= 2) launch_k<2, 2>(ctx, p, smem); else launch_k<4, 2>(ctx, p, smem); }
  return true;
}

}  // namespace dfgpu
