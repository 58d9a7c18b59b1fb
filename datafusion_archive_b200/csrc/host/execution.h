// execution.h — C++ mirror of the reference's operator API on the hot path:
//   trait Relation            src/execution/relation.rs:27-32
//   trait DataSource          src/execution/datasource.rs:27-30   (+ CsvDataSource :33-58)
//   DataSourceRelation        src/execution/relation.rs:34-54
//   FilterRelation/ProjectRelation/AggregateRelation -> GPU relations calling the C ABI
//   ExecutionContext          src/execution/context.rs:33-197
#pragma once
#include <fstream>
#include <map>
#include <optional>
#include <set>

#include "sqlplanner.h"

namespace dfhost {

// ---- host-side Arrow arrays (what Relation::next hands to its consumer) -----------------------------
struct Array {
  DataType data_type = 0;
  int64_t len = 0;
  int64_t offset = 0;      // element offset into the buffers (ArrayData.offset)
  int64_t null_count = 0;
  // buffers: either owned (vectors) or borrowed (raw pointers into caller memory)
  std::vector<uint8_t> own_values, own_validity;
  std::vector<int32_t> own_offsets;
  const void* values = nullptr;
  const uint8_t* validity = nullptr;
  const int32_t* offsets = nullptr;
  int64_t values_bytes = 0;  // Utf8 byte buffer size
  std::shared_ptr<void> owner;  // keeps library-owned (pinned) result memory alive for zero-copy columns
  dfgpu_col view() const;    // borrowed Arrow view for the C ABI
};
using ArrayRef = std::shared_ptr<Array>;

struct RecordBatch {
  SchemaRef schema;
  std::vector<ArrayRef> columns;
  int64_t num_rows = 0;
};

struct Relation {
  virtual ~Relation() {}
  virtual std::optional<RecordBatch> next() = 0;
  virtual const SchemaRef& schema() const = 0;
};
using RelationRef = std::shared_ptr<Relation>;

struct DataSource {
  virtual ~DataSource() {}
  virtual const SchemaRef& schema() const = 0;
  virtual std::optional<RecordBatch> next() = 0;
};
using DataSourceRef = std::shared_ptr<DataSource>;

// CsvDataSource::new(filename, schema, batch_size): has_headers is hard-wired to true, exactly as
// the reference does (datasource.rs:41) — the first line is always dropped.
class CsvDataSource : public DataSource {
 public:
  CsvDataSource(const std::string& filename, SchemaRef schema, size_t batch_size);
  const SchemaRef& schema() const override { return schema_; }
  std::optional<RecordBatch> next() override;
 private:
  SchemaRef schema_;
  std::ifstream file_;
  size_t batch_size_;
  bool header_skipped_ = false;
  size_t line_no_ = 0;
};

// In-memory source over borrowed Arrow buffers, yielding batch_size-row slices (zero copy).
class MemoryDataSource : public DataSource {
 public:
  MemoryDataSource(SchemaRef schema, std::vector<ArrayRef> cols, size_t batch_size);
  const SchemaRef& schema() const override { return schema_; }
  std::optional<RecordBatch> next() override;
 private:
  SchemaRef schema_;
  std::vector<ArrayRef> cols_;
  int64_t nrows_ = 0, pos_ = 0, batch_size_ = 0;
};

class DataSourceRelation : public Relation {
 public:
  explicit DataSourceRelation(DataSourceRef ds) : schema_(ds->schema()), ds_(std::move(ds)) {}
  std::optional<RecordBatch> next() override { return ds_->next(); }
  const SchemaRef& schema() const override { return schema_; }
 private:
  SchemaRef schema_;
  DataSourceRef ds_;
};

// FilterRelation (+ ProjectRelation fused): src/execution/filter.rs:29-110, projection.rs:29-74
class GpuFilterProjectRelation : public Relation {
 public:
  // predicate may be null (projection only); proj empty = all input columns (FilterRelation alone)
  GpuFilterProjectRelation(dfgpu_ctx* gpu, RelationRef input, ExprRef predicate, std::vector<ExprRef> proj, SchemaRef schema);
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return schema_; }
 private:
  RecordBatch process(const RecordBatch& batch, const std::vector<ExprRef>& proj, const SchemaRef& out_schema);
  dfgpu_ctx* gpu_;
  RelationRef input_;
  ExprRef predicate_;
  std::vector<ExprRef> proj_;
  SchemaRef schema_;
};

// Row-range shard of a relation for one-process-per-GPU execution: rank g of G passes on rows
// [g*ceil(n/G), min(n, (g+1)*ceil(n/G))) of every batch (zero copy: Array offset / len).  Inserted above the
// TableScan by ExecutionContext::execute when a partition is set (SURVEY.md §8e).
class ShardRelation : public Relation {
 public:
  ShardRelation(RelationRef input, int rank, int world) : input_(std::move(input)), rank_(rank), world_(world) {}
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return input_->schema(); }
 private:
  RelationRef input_;
  int rank_, world_;
};

// AggregateRelation: src/execution/aggregate.rs:38-61, 615-631.  `predicate` (may be null) is the expression
// of a Selection directly under the Aggregate (context.rs:126-139 builds FilterRelation there): it is fused
// into the scan kernel instead of materialising the filtered batch.
// A result stage (the Selection / Sort / Limit / Projection the planner puts over the Aggregate of a query with HAVING,
// ORDER BY or LIMIT) runs on the aggregate's device result through dfgpu_sort: the rows where `keep` is true, ordered
// by `sort`, then by the GROUP BY keys ascending when `ordered`, the first `limit`, and the first `visible` columns.
class GpuAggregateRelation : public Relation {
 public:
  struct ResultStage {
    ExprRef keep;               // HAVING over the aggregate's output, or null
    std::vector<ExprRef> sort;  // Expr::Sort over the aggregate's output
    bool ordered = false;       // a Sort or a Limit: the GROUP BY keys break the remaining ties
    int64_t limit = -1;         // < 0: no LIMIT
    SchemaRef aggregate_schema;  // the aggregate's own output: GROUP BY keys, then every aggregate, hidden ones included
  };
  GpuAggregateRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef input, std::vector<ExprRef> group_expr, std::vector<ExprRef> aggr_expr,
                       ExprRef predicate = nullptr, std::optional<ResultStage> stage = std::nullopt);
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return schema_; }
 private:
  RecordBatch finish(dfgpu_aggstate* st);  // dfgpu_aggregate_finish, the result stage and the download
  dfgpu_ctx* gpu_;
  SchemaRef schema_;
  RelationRef input_;
  std::vector<ExprRef> group_expr_, aggr_expr_;
  ExprRef predicate_;
  std::optional<ResultStage> stage_;
  bool end_of_results_ = false;
};

// Window (LogicalPlan::Window; the reference has no window functions).  On the first next() it drains its input and
// concatenates the batches on the host, uploads the columns the window calls read once and calls dfgpu_window once per
// distinct OVER specification; it returns one batch: the input columns in `cols` (the input's batches hold exactly those,
// in that order, when `projected`; else they hold every input column), every other input column as an empty placeholder,
// then one column per window call.  With a communicator attached every rank calls dfgpu_window, a rank without rows with
// an empty batch, and gets its own rows back.
class GpuWindowRelation : public Relation {
 public:
  GpuWindowRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef input, std::vector<size_t> cols, bool projected, std::vector<ExprRef> window_expr);
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return schema_; }
 private:
  dfgpu_ctx* gpu_;
  SchemaRef schema_;
  RelationRef input_;
  std::vector<size_t> cols_;
  bool projected_;
  std::vector<ExprRef> window_expr_;
  bool done_ = false;
};

// Inner equi-join (LogicalPlan::Join; the reference has no join relation).  On the first next() it drains the build
// (right) relation, concatenates its batches on the host and builds the GPU hash table (dfgpu_join_build); then each
// batch of the probe (left) relation gives one output batch (dfgpu_join_probe).  `left_keys` are over the left schema,
// `right_keys` over the right schema.
// A semi / anti join (`kind`) keeps the probe rows that pass (dfgpu_join_semi): its schema is the left schema, and
// `right_cols` is empty.
// Output batches have the joined schema's column positions, but only the columns in `left_cols` / `right_cols` (the ones
// the plan above references) are materialised: every other column is an empty placeholder (its dtype and length, no
// buffers), which no relation above reads.  So no unreferenced column is ever gathered or copied.
// The join's device state lives from the first next() until the probe side is exhausted.  A relation dropped before
// that holds it until release(): ExecutionContext releases every join it created before it shuts the GPU context
// down, so a relation that outlives its context never touches a freed one (its next() then returns nothing).
class GpuHashJoinRelation : public Relation {
 public:
  GpuHashJoinRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef left, RelationRef right, std::vector<ExprRef> left_keys,
                      std::vector<ExprRef> right_keys, std::vector<size_t> left_cols, std::vector<size_t> right_cols,
                      LogicalPlan::JoinKind kind = LogicalPlan::JoinKind::Inner);
  ~GpuHashJoinRelation() override;
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return schema_; }
  void release();  // frees the device state; next() returns nothing afterwards
 private:
  void build();
  dfgpu_ctx* gpu_;
  SchemaRef schema_;
  RelationRef left_, right_;
  std::vector<ExprRef> left_keys_, right_keys_;
  std::vector<size_t> left_cols_, right_cols_;
  LogicalPlan::JoinKind kind_;
  dfgpu_join* join_ = nullptr;
  bool released_ = false;
  std::vector<int> build_out_;  // right_cols_ as columns of the uploaded build batch
};

// The batches of one DataSource, drained on first use and replayed to each scan of a query that reads the table more
// than once (a self-join, a subquery over an outer table): a DataSource is one-pass.
class SharedScan {
 public:
  explicit SharedScan(DataSourceRef ds) : ds_(std::move(ds)) {}
  const SchemaRef& schema() const { return ds_->schema(); }
  const std::vector<RecordBatch>& batches();
 private:
  DataSourceRef ds_;
  std::vector<RecordBatch> batches_;
  bool drained_ = false;
};

// One scan of a SharedScan, with its own cursor
class SharedScanRelation : public Relation {
 public:
  explicit SharedScanRelation(std::shared_ptr<SharedScan> scan) : scan_(std::move(scan)) {}
  std::optional<RecordBatch> next() override;
  const SchemaRef& schema() const override { return scan_->schema(); }
 private:
  std::shared_ptr<SharedScan> scan_;
  size_t pos_ = 0;
};

class ExecutionContext {
 public:
  explicit ExecutionContext(int device);  // ExecutionContext::new() + dfgpu_init
  ~ExecutionContext();
  RelationRef sql(const std::string& sql);                                    // context.rs:44-98
  void register_datasource(const std::string& name, DataSourceRef ds);        // context.rs:100-102
  RelationRef execute(const PlanRef& plan);                                   // context.rs:104-196
  PlanRef plan(const std::string& sql);                                       // parse + plan only
  dfgpu_ctx* gpu() const { return gpu_; }
  // One process (ExecutionContext) per GPU: attach this context to an NCCL communicator and make it work on
  // its row range of every table.  Aggregates then return the GLOBAL result on every rank (partial-aggregate
  // merge inside dfgpu_aggregate_finish); filter / project relations return this rank's rows, and the
  // rank-ordered concatenation of all ranks' outputs is the global output.  `nccl_unique_id`: 128 bytes from
  // dfgpu_comm_unique_id on rank 0.
  void set_partition(int rank, int world, const uint8_t* nccl_unique_id);
  int rank() const { return rank_; }
  int world() const { return world_; }
  bool verbose = false;  // the reference prints "Logical plan: ..." on every execute (context.rs:105)
 private:
  // `needed`: the columns of the plan's output that the relations above read (null: all).  `shard`: whether a
  // TableScan is cut to this rank's row range (not under a join's build side: every rank builds from the whole table).
  RelationRef execute_node(const PlanRef& plan, const std::set<size_t>* needed, bool shard);
  std::shared_ptr<std::map<std::string, DataSourceRef>> datasources_;
  std::vector<std::weak_ptr<GpuHashJoinRelation>> joins_;  // released before gpu_ is shut down
  std::map<std::string, std::shared_ptr<SharedScan>> shared_;  // the tables the query being executed scans more than once
  dfgpu_ctx* gpu_ = nullptr;
  int rank_ = 0, world_ = 1;
};

// ---- built-in scalar functions ---------------------------------------------------------------------------
// The catalogue of functions ExecutionContext plans and runs on the GPU (DFGPU_OP_FN of include/dfgpu.h).  The reference
// only plans Expr::ScalarFunction; its console registers one `sqrt` UDF (src/bin/console/main.rs:123-125).  No function
// can be registered by the user: the GPU cannot run an arbitrary closure.
struct BuiltinFunction {
  const char* name;  // lower case; SQL names match in any letter case
  int op;            // DFGPU_OP_FN (Float64 math) or DFGPU_OP_UTF8_FN
  int code;          // DFGPU_FN_* or DFGPU_UTF8FN_*
  int min_arity, arity;  // arguments: min_arity .. arity (the planner's extra-argument check uses arity)
  DataType arg_types[3], return_type;
};
const std::vector<BuiltinFunction>& builtin_functions();
const BuiltinFunction* find_builtin_function(const std::string& name);      // nullptr for an unknown name
std::shared_ptr<FunctionMeta> builtin_function_meta(const std::string& name);  // FunctionMeta for the planner, or nullptr

// Expr name as RuntimeExpr::get_name reports it (expression.rs:230,312,322,407)
std::string runtime_expr_name(const Expr& e, const Schema& input_schema);

}  // namespace dfhost
