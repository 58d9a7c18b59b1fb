//! H100 (sm_90a) execution of the Arrow-batch hot path: FilterRelation, ProjectRelation and
//! AggregateRelation behind the `Relation` trait, calling libdfgpu.so (include/dfgpu.h).
pub mod ffi;
pub mod lower;
pub mod relation;

pub use self::relation::{GpuAggregateRelation, GpuContext, GpuFilterProjectRelation};
