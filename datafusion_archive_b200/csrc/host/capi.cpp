// capi.cpp — C API over the C++ host mirror, for harnesses that cannot link C++ (the Python tests
// and bench).  A Rust build of the reference would not use this file: it binds include/dfgpu.h
// directly (INTEGRATION.md); this layer exists because the reference's own host language has no
// toolchain in this image.
#include <cstring>

#include "execution.h"
#include "../../../include/dfhost.h"  // the declarations this file defines (signature check)

using namespace dfhost;

namespace {
thread_local std::string g_err;
template <class Fn>
int guarded(Fn&& fn) {
  try {
    fn();
    return 0;
  } catch (const ExecutionError& e) {
    g_err = e.msg;
    return e.code ? e.code : DFGPU_ERR_GENERAL;
  } catch (const std::exception& e) {
    g_err = std::string("internal: ") + e.what();
    return DFGPU_ERR_INTERNAL;
  }
}

struct Catalog : SchemaProvider {
  std::map<std::string, SchemaRef> tables;
  std::map<std::string, std::shared_ptr<FunctionMeta>> functions;
  bool builtins = false;  // dfhost_catalog_add_builtin_functions: ExecutionContext's catalogue, behind `functions`
  SchemaRef get_table_meta(const std::string& name) const override {
    auto it = tables.find(name);
    return it == tables.end() ? nullptr : it->second;
  }
  std::shared_ptr<FunctionMeta> get_function_meta(const std::string& name) const override {
    auto it = functions.find(name);
    if (it != functions.end()) return it->second;
    return builtins ? builtin_function_meta(name) : nullptr;
  }
};

SchemaRef make_schema(int ncols, const char* const* names, const int32_t* dtypes) {
  auto s = std::make_shared<Schema>();
  for (int i = 0; i < ncols; i++) s->fields.push_back(Field{names[i], dtypes[i], false});
  return s;
}

char* dup_str(const std::string& s) {
  char* p = static_cast<char*>(malloc(s.size() + 1));
  memcpy(p, s.c_str(), s.size() + 1);
  return p;
}
}  // namespace

struct dfhost_catalog { std::shared_ptr<Catalog> c = std::make_shared<Catalog>(); };
struct dfhost_context { std::unique_ptr<ExecutionContext> ctx; };
struct dfhost_relation { RelationRef rel; };
struct dfhost_batch { RecordBatch b; };
struct dfhost_datasource { DataSourceRef ds; };

extern "C" {

const char* dfhost_last_error(void) { return g_err.c_str(); }
void dfhost_free_string(char* s) { free(s); }

// ---- planner only (no GPU needed): MockSchemaProvider-style catalogs -----------------------------------
int dfhost_catalog_new(dfhost_catalog** out) { return guarded([&] { *out = new dfhost_catalog(); }); }
void dfhost_catalog_free(dfhost_catalog* c) { delete c; }
int dfhost_catalog_add_table(dfhost_catalog* c, const char* name, int ncols, const char* const* names, const int32_t* dtypes) {
  return guarded([&] { c->c->tables[name] = make_schema(ncols, names, dtypes); });
}
int dfhost_catalog_add_function(dfhost_catalog* c, const char* name, int nargs, const int32_t* arg_dtypes, int32_t return_dtype) {
  return guarded([&] {
    auto fm = std::make_shared<FunctionMeta>();
    fm->name = name;
    for (int i = 0; i < nargs; i++) fm->args.push_back(Field{"n", arg_dtypes[i], false});
    fm->return_type = return_dtype;
    c->c->functions[name] = fm;
  });
}
int dfhost_catalog_add_builtin_functions(dfhost_catalog* c) { return guarded([&] { c->c->builtins = true; }); }
// SQL -> `format!("{:?}", plan)` of the reference's LogicalPlan
int dfhost_plan_sql(dfhost_catalog* c, const char* sql, char** out_debug) {
  return guarded([&] {
    PlanRef plan = SqlToRel(c->c).sql_to_rel(parse_sql(sql));
    *out_debug = dup_str(plan->debug());
  });
}
int dfhost_supertype(int32_t l, int32_t r, int32_t* out) {
  DataType t = 0;
  bool ok = get_supertype(l, r, &t);
  *out = ok ? t : 0;
  return 0;
}
int dfhost_debug_f64(double x, char** out) { return guarded([&] { *out = dup_str(rust_debug_f64(x)); }); }

// ---- DataSource on its own (no GPU needed): CsvDataSource::new + next (datasource.rs:33-58) ---------------
int dfhost_csv_open(const char* filename, int ncols, const char* const* names, const int32_t* dtypes, int64_t batch_size, dfhost_datasource** out) {
  return guarded([&] {
    auto d = std::make_unique<dfhost_datasource>();
    d->ds = std::make_shared<CsvDataSource>(filename, make_schema(ncols, names, dtypes), size_t(batch_size));
    *out = d.release();
  });
}
int dfhost_datasource_next(dfhost_datasource* d, dfhost_batch** out) {
  return guarded([&] {
    *out = nullptr;
    auto b = d->ds->next();
    if (!b) return;
    auto hb = std::make_unique<dfhost_batch>();
    hb->b = std::move(*b);
    *out = hb.release();
  });
}
void dfhost_datasource_free(dfhost_datasource* d) { delete d; }

// ---- ExecutionContext -----------------------------------------------------------------------------------
int dfhost_context_new(int device, dfhost_context** out) {
  return guarded([&] {
    auto c = std::make_unique<dfhost_context>();
    c->ctx = std::make_unique<ExecutionContext>(device);
    *out = c.release();
  });
}
void dfhost_context_free(dfhost_context* c) { delete c; }
int dfhost_context_set_verbose(dfhost_context* c, int on) { c->ctx->verbose = on != 0; return 0; }
int dfhost_context_set_partition(dfhost_context* c, int rank, int world, const uint8_t* nccl_unique_id) {
  return guarded([&] { c->ctx->set_partition(rank, world, nccl_unique_id); });
}

int dfhost_register_csv(dfhost_context* c, const char* table, const char* filename, int ncols, const char* const* names,
                        const int32_t* dtypes, int64_t batch_size) {
  return guarded([&] {
    c->ctx->register_datasource(table, std::make_shared<CsvDataSource>(filename, make_schema(ncols, names, dtypes), size_t(batch_size)));
  });
}
// Borrowed Arrow buffers (must outlive every relation created over the table).
int dfhost_register_memory(dfhost_context* c, const char* table, int ncols, const char* const* names, const dfgpu_col* cols, int64_t batch_size) {
  return guarded([&] {
    auto schema = std::make_shared<Schema>();
    std::vector<ArrayRef> arrays;
    for (int i = 0; i < ncols; i++) {
      schema->fields.push_back(Field{names[i], cols[i].dtype, cols[i].validity != nullptr});
      auto a = std::make_shared<Array>();
      a->data_type = cols[i].dtype;
      a->len = cols[i].len;
      a->offset = cols[i].offset;
      a->values = cols[i].values;
      a->validity = cols[i].validity;
      a->offsets = cols[i].offsets;
      a->values_bytes = cols[i].values_bytes;
      if (cols[i].validity) {
        int64_t nulls = 0;
        for (int64_t r = 0; r < a->len; r++) nulls += !((cols[i].validity[(a->offset + r) >> 3] >> ((a->offset + r) & 7)) & 1);
        a->null_count = nulls;
      }
      arrays.push_back(a);
    }
    c->ctx->register_datasource(table, std::make_shared<MemoryDataSource>(schema, arrays, size_t(batch_size)));
  });
}

int dfhost_sql(dfhost_context* c, const char* sql, dfhost_relation** out) {
  return guarded([&] {
    auto r = std::make_unique<dfhost_relation>();
    r->rel = c->ctx->sql(sql);
    *out = r.release();
  });
}
int dfhost_plan_debug(dfhost_context* c, const char* sql, char** out_debug) {
  return guarded([&] { *out_debug = dup_str(c->ctx->plan(sql)->debug()); });
}
void dfhost_relation_free(dfhost_relation* r) { delete r; }
int dfhost_relation_schema(dfhost_relation* r, int* nfields) {
  *nfields = int(r->rel->schema()->fields.size());
  return 0;
}
int dfhost_relation_field(dfhost_relation* r, int i, char** name, int32_t* dtype) {
  return guarded([&] {
    const auto& f = r->rel->schema()->fields.at(size_t(i));
    *name = dup_str(f.name);
    *dtype = f.data_type;
  });
}
// Relation::next(): *out = NULL when exhausted
int dfhost_relation_next(dfhost_relation* r, dfhost_batch** out) {
  return guarded([&] {
    *out = nullptr;
    auto b = r->rel->next();
    if (!b) return;
    auto hb = std::make_unique<dfhost_batch>();
    hb->b = std::move(*b);
    *out = hb.release();
  });
}
void dfhost_batch_free(dfhost_batch* b) { delete b; }
int dfhost_batch_shape(const dfhost_batch* b, int64_t* nrows, int* ncols) {
  *nrows = b->b.num_rows;
  *ncols = int(b->b.columns.size());
  return 0;
}
int dfhost_batch_col(const dfhost_batch* b, int i, dfgpu_col* out, int64_t* null_count) {
  return guarded([&] {
    const Array& a = *b->b.columns.at(size_t(i));
    *out = a.view();
    *null_count = a.null_count;
  });
}

}  // extern "C"
