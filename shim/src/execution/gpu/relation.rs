//! `impl Relation` for the GPU operators (src/execution/relation.rs:27-32).
//!   GpuFilterProjectRelation = FilterRelation (+ ProjectRelation fused): filter.rs:29-110, projection.rs:29-74
//!   GpuAggregateRelation     = AggregateRelation: aggregate.rs:38-61, 615-631, 703-952
//! Inputs are borrowed views of the Arrow buffers for the duration of a call; outputs are copied into
//! freshly allocated Arrow buffers; opaque handles are freed with their `*_free`.  Everything is `!Send`
//! like the rest of the reference (`Rc<RefCell<..>>`): one host thread per dfgpu_ctx.
use std::cell::RefCell;
use std::os::raw::{c_int, c_void};
use std::ptr;
use std::rc::Rc;
use std::sync::Arc;

use arrow::array::{Array, ArrayData, ArrayRef, BinaryArray, BooleanArray, PrimitiveArray};
use arrow::buffer::MutableBuffer;
use arrow::datatypes::*;
use arrow::record_batch::RecordBatch;

use super::super::super::logicalplan::Expr;
use super::super::error::{ExecutionError, Result};
use super::super::relation::Relation;
use super::ffi::*;
use super::lower::{collect_columns, dtype_code, lower};

/// Owner of the dfgpu_ctx; created once by ExecutionContext::new() (src/execution/context.rs:38).
pub struct GpuContext {
    pub raw: *mut dfgpu_ctx,
}
impl GpuContext {
    pub fn new(device: i32) -> Result<Rc<GpuContext>> {
        let mut raw = ptr::null_mut();
        check(unsafe { dfgpu_init(device as c_int, &mut raw) })?;
        Ok(Rc::new(GpuContext { raw }))
    }
    /// one process per GPU: join the NCCL communicator (id from dfgpu_comm_unique_id on rank 0)
    pub fn join(&self, rank: i32, world: i32, id: &[u8; 128]) -> Result<()> {
        check(unsafe { dfgpu_comm_init(self.raw, rank, world, id.as_ptr()) })
    }
}
impl Drop for GpuContext {
    fn drop(&mut self) {
        unsafe { dfgpu_shutdown(self.raw) };
    }
}

/// Borrowed view of one Arrow array: values buffer, len, offset, null bitmap; Utf8 = BinaryArray
/// (offsets buffer + byte buffer), as in src/execution/filter.rs:93-103.
fn col_view(a: &ArrayRef) -> Result<dfgpu_col> {
    let d = a.data();
    let dt = dtype_code(a.data_type())?;
    let validity = d.null_bitmap().as_ref().map(|b| b.raw_data()).unwrap_or(ptr::null());
    let mut c = dfgpu_col {
        dtype: dt, _pad: 0, len: d.len() as i64, offset: d.offset() as i64,
        values: ptr::null(), validity, offsets: ptr::null(), values_bytes: 0,
    };
    if dt == DT_UTF8 {
        c.offsets = d.buffers()[0].raw_data() as *const i32;
        c.values = d.buffers()[1].raw_data() as *const c_void;
        c.values_bytes = d.buffers()[1].len() as i64;
    } else {
        c.values = d.buffers()[0].raw_data() as *const c_void;
    }
    Ok(c)
}

fn arrow_type(code: i32) -> DataType {
    match code {
        DT_BOOL => DataType::Boolean, DT_INT8 => DataType::Int8, DT_INT16 => DataType::Int16, DT_INT32 => DataType::Int32,
        DT_INT64 => DataType::Int64, DT_UINT8 => DataType::UInt8, DT_UINT16 => DataType::UInt16, DT_UINT32 => DataType::UInt32,
        DT_UINT64 => DataType::UInt64, DT_FLOAT32 => DataType::Float32, DT_FLOAT64 => DataType::Float64, _ => DataType::Utf8,
    }
}

/// Copy a device result into a RecordBatch: size query, MutableBuffer per buffer, dfgpu_result_copy_col,
/// ArrayData::builder (the builder calls of projection.rs:59-60 / aggregate.rs:890-949 without the per-row appends).
fn download(res: *mut dfgpu_result, schema: &Arc<Schema>) -> Result<RecordBatch> {
    let (mut nrows, mut ncols) = (0i64, 0 as c_int);
    check(unsafe { dfgpu_result_shape(res, &mut nrows, &mut ncols) })?;
    let n = nrows as usize;
    let mut columns: Vec<ArrayRef> = Vec::with_capacity(ncols as usize);
    for i in 0..ncols {
        let (mut dt, mut nulls, mut nbytes) = (0i32, 0i64, 0i64);
        unsafe {
            check(dfgpu_result_col_dtype(res, i, &mut dt))?;
            check(dfgpu_result_col_nulls(res, i, &mut nulls))?;
            check(dfgpu_result_col_bytes(res, i, &mut nbytes))?;
        }
        let mut values = MutableBuffer::new(nbytes.max(1) as usize);
        values.resize(nbytes as usize)?;
        let mut validity = MutableBuffer::new((n + 7) / 8 + 1);
        validity.resize((n + 7) / 8)?;
        let mut offsets = MutableBuffer::new((n + 1) * 4);
        offsets.resize((n + 1) * 4)?;
        let want_validity = nulls > 0;
        check(unsafe {
            dfgpu_result_copy_col(
                res, i, values.raw_data() as *mut c_void,
                if want_validity { validity.raw_data() as *mut u8 } else { ptr::null_mut() },
                if dt == DT_UTF8 { offsets.raw_data() as *mut i32 } else { ptr::null_mut() },
            )
        })?;
        let mut b = ArrayData::builder(arrow_type(dt)).len(n);
        if dt == DT_UTF8 {
            b = b.add_buffer(offsets.freeze());
        }
        b = b.add_buffer(values.freeze());
        if want_validity {
            b = b.null_count(nulls as usize).null_bit_buffer(validity.freeze());
        }
        let data = b.build();
        columns.push(match dt {
            DT_BOOL => Arc::new(BooleanArray::from(data)) as ArrayRef,
            DT_INT8 => Arc::new(PrimitiveArray::<Int8Type>::from(data)),
            DT_INT16 => Arc::new(PrimitiveArray::<Int16Type>::from(data)),
            DT_INT32 => Arc::new(PrimitiveArray::<Int32Type>::from(data)),
            DT_INT64 => Arc::new(PrimitiveArray::<Int64Type>::from(data)),
            DT_UINT8 => Arc::new(PrimitiveArray::<UInt8Type>::from(data)),
            DT_UINT16 => Arc::new(PrimitiveArray::<UInt16Type>::from(data)),
            DT_UINT32 => Arc::new(PrimitiveArray::<UInt32Type>::from(data)),
            DT_UINT64 => Arc::new(PrimitiveArray::<UInt64Type>::from(data)),
            DT_FLOAT32 => Arc::new(PrimitiveArray::<Float32Type>::from(data)),
            DT_FLOAT64 => Arc::new(PrimitiveArray::<Float64Type>::from(data)),
            _ => Arc::new(BinaryArray::from(data)),
        });
    }
    Ok(RecordBatch::new(schema.clone(), columns))
}

/// Prune the upload to the columns the expressions read: (uploaded column indices, input index -> uploaded index).
fn prune(exprs: &[&Expr], ncols: usize, all: bool) -> (Vec<usize>, Vec<Option<usize>>) {
    let mut used: Vec<usize> = if all { (0..ncols).collect() } else { vec![] };
    for e in exprs {
        collect_columns(e, &mut used);
    }
    used.sort();
    used.dedup();
    let mut remap = vec![None; ncols];
    for (k, c) in used.iter().enumerate() {
        if *c < ncols {
            remap[*c] = Some(k);
        }
    }
    (used, remap)
}

// ---------------------------------------------------------------------------------------------------------
pub struct GpuFilterProjectRelation {
    gpu: Rc<GpuContext>,
    schema: Arc<Schema>,
    input: Rc<RefCell<Relation>>,
    predicate: Option<Expr>,
    proj: Vec<Expr>, // empty = FilterRelation alone: every input column (filter.rs:55-57)
}

impl GpuFilterProjectRelation {
    pub fn new(gpu: Rc<GpuContext>, input: Rc<RefCell<Relation>>, predicate: Option<Expr>, proj: Vec<Expr>, schema: Arc<Schema>) -> Self {
        GpuFilterProjectRelation { gpu, schema, input, predicate, proj }
    }
}

impl Relation for GpuFilterProjectRelation {
    fn next(&mut self) -> Result<Option<RecordBatch>> {
        let batch = match self.input.borrow_mut().next()? {
            Some(b) => b,
            None => return Ok(None),
        };
        let in_schema = self.input.borrow().schema().clone();
        let all_cols: Vec<Expr> = (0..batch.num_columns()).map(Expr::Column).collect();
        let exprs: &[Expr] = if self.proj.is_empty() { &all_cols } else { &self.proj };
        let mut reads: Vec<&Expr> = exprs.iter().collect();
        if let Some(p) = &self.predicate {
            reads.push(p);
        }
        let (used, remap) = prune(&reads, batch.num_columns(), false);
        let mut pred = vec![];
        if let Some(p) = &self.predicate {
            lower(p, &in_schema, &remap, &mut pred)?;
        }
        let mut progs: Vec<Vec<dfgpu_insn>> = vec![];
        for e in exprs {
            let mut v = vec![];
            lower(e, &in_schema, &remap, &mut v)?;
            progs.push(v);
        }
        let cols = used.iter().map(|c| col_view(batch.column(*c))).collect::<Result<Vec<_>>>()?;
        let ptrs: Vec<*const dfgpu_insn> = progs.iter().map(|p| p.as_ptr()).collect();
        let lens: Vec<c_int> = progs.iter().map(|p| p.len() as c_int).collect();
        let (mut dbatch, mut res) = (ptr::null_mut(), ptr::null_mut());
        unsafe {
            check(dfgpu_batch_upload(self.gpu.raw, cols.as_ptr(), cols.len() as c_int, &mut dbatch))?;
            let rc = dfgpu_filter_project(self.gpu.raw, dbatch, pred.as_ptr(), pred.len() as c_int, ptrs.as_ptr(), lens.as_ptr(), ptrs.len() as c_int, &mut res);
            dfgpu_batch_free(dbatch);
            check(rc)?;
        }
        // (batches of millions of rows: dfgpu_filter_project_host overlaps PCIe and the kernel chunk by chunk and
        // returns pinned host columns — see csrc/host/execution.cpp GpuFilterProjectRelation::process)
        let out = download(res, &self.schema);
        unsafe { dfgpu_result_free(res) };
        out.map(Some)
    }
    fn schema(&self) -> &Arc<Schema> {
        &self.schema
    }
}

// ---------------------------------------------------------------------------------------------------------
pub struct GpuAggregateRelation {
    gpu: Rc<GpuContext>,
    schema: Arc<Schema>,
    input: Rc<RefCell<Relation>>,
    group_expr: Vec<Expr>,
    aggr_expr: Vec<Expr>,
    predicate: Option<Expr>, // Selection directly under the Aggregate: fused into the scan kernel
    end_of_results: bool,
}

impl GpuAggregateRelation {
    pub fn new(gpu: Rc<GpuContext>, schema: Arc<Schema>, input: Rc<RefCell<Relation>>, group_expr: Vec<Expr>, aggr_expr: Vec<Expr>, predicate: Option<Expr>) -> Self {
        GpuAggregateRelation { gpu, schema, input, group_expr, aggr_expr, predicate, end_of_results: false }
    }
}

fn agg_func(name: &str) -> Result<i32> {
    match name.to_lowercase().as_ref() {
        "min" => Ok(AGG_MIN),
        "max" => Ok(AGG_MAX),
        "sum" => Ok(AGG_SUM),
        "count" => Ok(AGG_COUNT),
        "avg" => Ok(AGG_AVG),
        _ => Err(ExecutionError::General(format!("Unsupported aggregate function '{}'", name))), // expression.rs:103-106
    }
}

impl Relation for GpuAggregateRelation {
    fn next(&mut self) -> Result<Option<RecordBatch>> {
        if self.end_of_results {
            return Ok(None); // aggregate.rs:616-619
        }
        self.end_of_results = true;
        let in_schema = self.input.borrow().schema().clone();
        let mut args: Vec<(i32, &Expr, i32)> = vec![];
        for a in &self.aggr_expr {
            match a {
                Expr::AggregateFunction { name, args: fargs, return_type } => {
                    assert_eq!(1, fargs.len()); // expression.rs:91
                    args.push((agg_func(name)?, &fargs[0], dtype_code(return_type)?));
                }
                _ => return Err(ExecutionError::General("Invalid aggregate expression".to_string())),
            }
        }
        let mut reads: Vec<&Expr> = self.group_expr.iter().collect();
        reads.extend(args.iter().map(|a| a.1));
        if let Some(p) = &self.predicate {
            reads.push(p);
        }
        let mut st: *mut dfgpu_aggstate = ptr::null_mut();
        let mut used: Vec<usize> = vec![];
        let result = (|| -> Result<RecordBatch> {
            while let Some(batch) = self.input.borrow_mut().next()? {
                // aggregate.rs:707 / :796
                if st.is_null() {
                    let (u, remap) = prune(&reads, batch.num_columns(), false);
                    used = u;
                    let mut keys: Vec<Vec<dfgpu_insn>> = vec![];
                    for k in &self.group_expr {
                        let mut v = vec![];
                        lower(k, &in_schema, &remap, &mut v)?;
                        keys.push(v);
                    }
                    let mut arg_progs: Vec<Vec<dfgpu_insn>> = vec![];
                    for a in &args {
                        let mut v = vec![];
                        lower(a.1, &in_schema, &remap, &mut v)?;
                        arg_progs.push(v);
                    }
                    let kptr: Vec<*const dfgpu_insn> = keys.iter().map(|p| p.as_ptr()).collect();
                    let klen: Vec<c_int> = keys.iter().map(|p| p.len() as c_int).collect();
                    let aggs: Vec<dfgpu_agg> = args.iter().zip(arg_progs.iter())
                        .map(|(a, p)| dfgpu_agg { func: a.0, arg_len: p.len() as i32, arg: p.as_ptr(), out_dtype: a.2, _pad: 0 })
                        .collect();
                    check(unsafe { dfgpu_aggregate_create(self.gpu.raw, kptr.as_ptr(), klen.as_ptr(), kptr.len() as c_int, aggs.as_ptr(), aggs.len() as c_int, 0, &mut st) })?;
                    if let Some(p) = &self.predicate {
                        let mut v = vec![];
                        lower(p, &in_schema, &remap, &mut v)?;
                        check(unsafe { dfgpu_aggregate_set_predicate(st, v.as_ptr(), v.len() as c_int) })?;
                    }
                }
                let cols = used.iter().map(|c| col_view(batch.column(*c))).collect::<Result<Vec<_>>>()?;
                check(unsafe { dfgpu_aggregate_update_host(st, cols.as_ptr(), cols.len() as c_int, 0) })?;
            }
            if st.is_null() {
                // empty input: GROUP BY -> empty batch; no GROUP BY -> one row of nulls (array_from_scalar!, aggregate.rs:641-643)
                if !self.group_expr.is_empty() {
                    let mut world: i64 = 1;
                    check(unsafe { dfgpu_comm_world(self.gpu.raw, &mut world) })?;
                    if world <= 1 {
                        return Ok(RecordBatch::new(self.schema.clone(), vec![]));
                    }
                    // a communicator is attached: this rank saw no batch but still has to join the merge of
                    // dfgpu_aggregate_finish with an empty state (it adopts the key / argument types from the other ranks)
                    let (_, remap) = prune(&reads, in_schema.fields().len(), false);
                    let mut keys: Vec<Vec<dfgpu_insn>> = vec![];
                    for k in &self.group_expr {
                        let mut v = vec![];
                        lower(k, &in_schema, &remap, &mut v)?;
                        keys.push(v);
                    }
                    let mut arg_progs: Vec<Vec<dfgpu_insn>> = vec![];
                    for a in &args {
                        let mut v = vec![];
                        lower(a.1, &in_schema, &remap, &mut v)?;
                        arg_progs.push(v);
                    }
                    let kptr: Vec<*const dfgpu_insn> = keys.iter().map(|p| p.as_ptr()).collect();
                    let klen: Vec<c_int> = keys.iter().map(|p| p.len() as c_int).collect();
                    let aggs: Vec<dfgpu_agg> = args.iter().zip(arg_progs.iter())
                        .map(|(a, p)| dfgpu_agg { func: a.0, arg_len: p.len() as i32, arg: p.as_ptr(), out_dtype: a.2, _pad: 0 })
                        .collect();
                    check(unsafe { dfgpu_aggregate_create(self.gpu.raw, kptr.as_ptr(), klen.as_ptr(), kptr.len() as c_int, aggs.as_ptr(), aggs.len() as c_int, 0, &mut st) })?;
                    let mut res = ptr::null_mut();
                    check(unsafe { dfgpu_aggregate_finish(st, &mut res) })?;
                    let out = download(res, &self.schema);
                    unsafe { dfgpu_result_free(res) };
                    return out;
                }
                let lit = [dfgpu_insn { op: OP_COL, col: 0, dtype: 0, _pad: 0, lit: 0 }];
                let aggs: Vec<dfgpu_agg> = args.iter().map(|a| dfgpu_agg { func: a.0, arg_len: 1, arg: lit.as_ptr(), out_dtype: a.2, _pad: 0 }).collect();
                check(unsafe { dfgpu_aggregate_create(self.gpu.raw, ptr::null(), ptr::null(), 0, aggs.as_ptr(), aggs.len() as c_int, 0, &mut st) })?;
            }
            let mut res = ptr::null_mut();
            check(unsafe { dfgpu_aggregate_finish(st, &mut res) })?; // + the multi-GPU merge when a communicator is attached
            let out = download(res, &self.schema); // group columns then aggregate columns (aggregate.rs:890-949)
            unsafe { dfgpu_result_free(res) };
            out
        })();
        if !st.is_null() {
            unsafe { dfgpu_aggregate_free(st) };
        }
        result.map(Some)
    }
    fn schema(&self) -> &Arc<Schema> {
        &self.schema
    }
}
