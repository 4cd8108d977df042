//! Raw bindings of include/flockgpu.h.  Batches cross the boundary through the Arrow C Data Interface
//! (`arrow::ffi::{FFI_ArrowArray, FFI_ArrowSchema}` are layout-compatible with `struct ArrowArray` /
//! `struct ArrowSchema`).
#![allow(non_camel_case_types)]
use datafusion::arrow::ffi::{FFI_ArrowArray, FFI_ArrowSchema};
use std::os::raw::{c_char, c_int, c_void};

#[repr(C)]
pub struct flockgpu_ctx {
    _private: [u8; 0],
}
#[repr(C)]
pub struct flockgpu_table {
    _private: [u8; 0],
}
#[repr(C)]
pub struct flockgpu_payload {
    _private: [u8; 0],
}
#[repr(C)]
pub struct flock_context {
    _private: [u8; 0],
}

pub const FLOCKGPU_OK: c_int = 0;
pub const FLOCKGPU_ERR_INVALID: c_int = -1;
pub const FLOCKGPU_ERR_UNSUPPORTED: c_int = -2;

extern "C" {
    pub fn flockgpu_open(device: c_int, out: *mut *mut flockgpu_ctx) -> c_int;
    pub fn flockgpu_close(ctx: *mut flockgpu_ctx) -> c_int;
    pub fn flockgpu_last_error() -> *const c_char;
    /// "feed_zero_copy" (0/1): page-locked, uniformly batched fixed-width columns stay in host memory and are read in place.
    pub fn flockgpu_set_option(ctx: *mut flockgpu_ctx, name: *const c_char, value: i64) -> c_int;
    /// Page-locked host memory for record-batch buffers (256-byte aligned, carved out of 64 MB slabs).
    pub fn flockgpu_host_alloc(ctx: *mut flockgpu_ctx, bytes: i64, out: *mut *mut c_void) -> c_int;
    pub fn flockgpu_host_free(ctx: *mut flockgpu_ctx, ptr: *mut c_void) -> c_int;

    pub fn flockgpu_table_export(
        ctx: *mut flockgpu_ctx,
        table: *const flockgpu_table,
        row_begin: i64,
        row_count: i64,
        out_schema: *mut FFI_ArrowSchema,
        out_array: *mut FFI_ArrowArray,
    ) -> c_int;
    pub fn flockgpu_table_release(table: *mut flockgpu_table) -> c_int;
    /// Payload frames (FlightData.data_header / data_body, Encoding::None) straight to a device table and back.
    pub fn flockgpu_table_import_ipc(
        ctx: *mut flockgpu_ctx,
        schema: *const FFI_ArrowSchema,
        headers: *const *const u8,
        header_lens: *const i64,
        bodies: *const *const u8,
        body_lens: *const i64,
        n_frames: i32,
        projection: *const i32,
        n_projection: i32,
        out: *mut *mut flockgpu_table,
    ) -> c_int;
    /// Payload frames as they arrive, compressed with `encoding` (Flock's `Encoding` discriminant, `payload.encoding as
    /// i32`): Zstd bodies are decoded on the GPU, None is flockgpu_table_import_ipc, Snappy / Lz4 / Zlib return
    /// FLOCKGPU_ERR_UNSUPPORTED.  header_lens / body_lens are the compressed lengths.
    pub fn flockgpu_table_import_payload(
        ctx: *mut flockgpu_ctx,
        schema: *const FFI_ArrowSchema,
        encoding: i32,
        headers: *const *const u8,
        header_lens: *const i64,
        bodies: *const *const u8,
        body_lens: *const i64,
        n_frames: i32,
        projection: *const i32,
        n_projection: i32,
        out: *mut *mut flockgpu_table,
    ) -> c_int;
    pub fn flockgpu_table_export_ipc(
        ctx: *mut flockgpu_ctx,
        table: *const flockgpu_table,
        row_begin: i64,
        row_count: i64,
        out_header: *mut *mut u8,
        out_header_len: *mut i64,
        out_body: *mut *mut u8,
        out_body_len: *mut i64,
    ) -> c_int;
    pub fn flockgpu_ipc_free(block: *mut u8);
    /// HBM -> a payload's DataFrames, rows_per_frame rows each; ZSTD bodies are compressed on the GPU.
    pub fn flockgpu_table_export_payload(
        ctx: *mut flockgpu_ctx,
        table: *const flockgpu_table,
        encoding: i32,
        rows_per_frame: i64,
        out: *mut *mut flockgpu_payload,
    ) -> c_int;
    pub fn flockgpu_payload_num_frames(p: *const flockgpu_payload) -> i32;
    pub fn flockgpu_payload_frame(
        p: *const flockgpu_payload,
        i: i32,
        header: *mut *const u8,
        header_len: *mut i64,
        body: *mut *const u8,
        body_len: *mut i64,
    ) -> c_int;
    pub fn flockgpu_payload_free(p: *mut flockgpu_payload);
    pub fn flock_context_feed_tables(ec: *mut flock_context, tables: *const *mut flockgpu_table, n_sources: i32) -> c_int;
    pub fn flockgpu_table_num_rows(table: *const flockgpu_table) -> i64;
    pub fn flockgpu_table_nbytes(table: *const flockgpu_table) -> i64;

    // flock::runtime::context::ExecutionContext on the GPU
    pub fn flock_context_unmarshal(ctx: *mut flockgpu_ctx, plans_json: *const c_char, out: *mut *mut flock_context) -> c_int;
    pub fn flock_context_free(ec: *mut flock_context) -> c_int;
    pub fn flock_context_num_plans(ec: *const flock_context) -> i32;
    pub fn flock_context_feed_data_sources(
        ec: *mut flock_context,
        schemas: *const *const FFI_ArrowSchema,
        batches: *const *const *const FFI_ArrowArray,
        n_batches: *const i32,
        n_sources: i32,
    ) -> c_int;
    pub fn flock_context_execute(ec: *mut flock_context, plan_index: i32, out: *mut *mut flockgpu_table) -> c_int;
    pub fn flock_context_execute_partitioned(
        ec: *mut flock_context,
        plan_index: i32,
        out_parts: *mut *mut flockgpu_table,
        max_parts: i32,
        n_parts: *mut i32,
    ) -> c_int;
    pub fn flock_context_clean_data_sources(ec: *mut flock_context) -> c_int;
}
