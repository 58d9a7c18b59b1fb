/* dfhost.h — C API of libdfhost.so, the C++ mirror of the reference's HOST layer above the operator
 * boundary (ExecutionContext / Relation / DataSource / SQL planner), for harnesses that cannot link
 * C++ (the Python tests and bench).
 *
 * This is NOT the drop-in boundary: a Rust build of the reference binds include/dfgpu.h directly
 * (INTEGRATION.md) and keeps its own host layer.  This layer exists because the reference's host
 * language has no toolchain in the build image; it mirrors, name for name:
 *   ExecutionContext::{new, register_datasource, sql}   src/execution/context.rs:38-102
 *   Relation::{next, schema}                            src/execution/relation.rs:27-32
 *   CsvDataSource::{new, next}                          src/execution/datasource.rs:33-58
 *   SqlToRel::sql_to_rel + SchemaProvider               src/sqlplanner.rs:27-375
 *   get_supertype                                       src/logicalplan.rs:446-548
 * Conventions: every function returns 0 or a DFGPU_ERR_* code (include/dfgpu.h) with the message in
 * dfhost_last_error() (thread-local); strings returned through `char**` are released with
 * dfhost_free_string; dtypes are the dfgpu_dtype codes. */
#ifndef DFHOST_H
#define DFHOST_H

#include "dfgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dfhost_catalog dfhost_catalog;       /* SchemaProvider: tables + scalar functions (planner only) */
typedef struct dfhost_context dfhost_context;       /* ExecutionContext bound to one GPU */
typedef struct dfhost_relation dfhost_relation;     /* Rc<RefCell<Relation>> */
typedef struct dfhost_batch dfhost_batch;           /* RecordBatch in host memory */
typedef struct dfhost_datasource dfhost_datasource; /* Rc<RefCell<DataSource>> */

const char* dfhost_last_error(void);
void dfhost_free_string(char* s);

/* ---- planner only (no GPU): SqlToRel over a SchemaProvider, plan printed with Rust's {:?} ---- */
int dfhost_catalog_new(dfhost_catalog** out);
void dfhost_catalog_free(dfhost_catalog* c);
int dfhost_catalog_add_table(dfhost_catalog* c, const char* name, int ncols, const char* const* names, const int32_t* dtypes);
int dfhost_catalog_add_function(dfhost_catalog* c, const char* name, int nargs, const int32_t* arg_dtypes, int32_t return_dtype);
/* the built-in scalar functions ExecutionContext plans and runs (sqrt, abs, power, ...: DFGPU_FN_* of dfgpu.h), matched in
 * any letter case; functions added by name take precedence */
int dfhost_catalog_add_builtin_functions(dfhost_catalog* c);
int dfhost_plan_sql(dfhost_catalog* c, const char* sql, char** out_debug);
int dfhost_supertype(int32_t l, int32_t r, int32_t* out); /* get_supertype; *out = 0 when there is none */
int dfhost_debug_f64(double x, char** out);               /* format!("{:?}", x) */

/* ---- data sources (no GPU) ---- */
int dfhost_csv_open(const char* filename, int ncols, const char* const* names, const int32_t* dtypes, int64_t batch_size,
                    dfhost_datasource** out);
int dfhost_datasource_next(dfhost_datasource* d, dfhost_batch** out); /* *out = NULL when exhausted */
void dfhost_datasource_free(dfhost_datasource* d);

/* ---- ExecutionContext (needs a GPU: dfgpu_init) ---- */
int dfhost_context_new(int device, dfhost_context** out);
void dfhost_context_free(dfhost_context* c);
int dfhost_context_set_verbose(dfhost_context* c, int on); /* the reference's `println!("Logical plan: ..")` */
/* one process per GPU: join an NCCL communicator (128-byte id from dfgpu_comm_unique_id on rank 0) and work on
 * this rank's row range of every table; aggregates return the global result on every rank */
int dfhost_context_set_partition(dfhost_context* c, int rank, int world, const uint8_t* nccl_unique_id);
int dfhost_register_csv(dfhost_context* c, const char* table, const char* filename, int ncols, const char* const* names,
                        const int32_t* dtypes, int64_t batch_size);
/* in-memory table over borrowed Arrow buffers (must outlive the relation), sliced into batch_size rows */
int dfhost_register_memory(dfhost_context* c, const char* table, int ncols, const char* const* names, const dfgpu_col* cols,
                           int64_t batch_size);
int dfhost_sql(dfhost_context* c, const char* sql, dfhost_relation** out);
int dfhost_plan_debug(dfhost_context* c, const char* sql, char** out_debug);

/* ---- Relation ---- */
void dfhost_relation_free(dfhost_relation* r);
int dfhost_relation_schema(dfhost_relation* r, int* nfields);
int dfhost_relation_field(dfhost_relation* r, int i, char** name, int32_t* dtype);
int dfhost_relation_next(dfhost_relation* r, dfhost_batch** out); /* *out = NULL when exhausted */

/* ---- RecordBatch ---- */
void dfhost_batch_free(dfhost_batch* b);
int dfhost_batch_shape(const dfhost_batch* b, int64_t* nrows, int* ncols);
int dfhost_batch_col(const dfhost_batch* b, int i, dfgpu_col* out, int64_t* null_count); /* borrowed view, valid until batch_free */

#ifdef __cplusplus
}
#endif
#endif /* DFHOST_H */
