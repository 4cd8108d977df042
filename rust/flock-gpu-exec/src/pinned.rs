//! Page-locked Arrow buffers: the allocator hook behind `feed_zero_copy` (INTEGRATION.md section 4).
//!
//! arrow-rs 6 (the fork's version) has no pluggable allocator, but it does accept FOREIGN memory: a buffer imported
//! through the C Data Interface is `Deallocation::Foreign(Arc<FFI_ArrowArray>)` and is released through the array's
//! `release` callback.  So record batches whose buffers live in `flockgpu_host_alloc` memory are built as FFI arrays
//! with a release callback that calls `flockgpu_host_free`, and imported with `make_array_from_raw`.  The two places
//! that create the batches a worker function executes on are `Payload::to_record_batch` (flock/src/runtime/
//! payload.rs:161-192) and `Arena::take` (flock/src/runtime/arena/mod.rs:114-169): both decode (and, with
//! Encoding::Zstd, decompress) into freshly allocated memory anyway, so decoding INTO page-locked memory costs
//! nothing extra -- `pinned_batch` below is the copy form for batches that already exist.  `frames_to_table` skips
//! host batches altogether: zstd frames are decompressed on the GPU; `table_to_frames` is its inverse, compressing on
//! the GPU.
//!
//! SOURCE ONLY (no cargo / rustc in the build image): never compiled.
use crate::ffi;
use datafusion::arrow::array::{make_array_from_raw, Array, ArrayRef, StructArray};
use datafusion::arrow::error::Result as ArrowResult;
use datafusion::arrow::ffi::{FFI_ArrowArray, FFI_ArrowSchema};
use datafusion::arrow::record_batch::RecordBatch;
use std::os::raw::c_void;

/// One page-locked block; freed through the library when the last Arrow buffer that points into it goes away.
struct PinnedBlock {
    ctx: *mut ffi::flockgpu_ctx,
    ptr: *mut c_void,
}
unsafe impl Send for PinnedBlock {}
unsafe impl Sync for PinnedBlock {}
impl Drop for PinnedBlock {
    fn drop(&mut self) {
        unsafe { ffi::flockgpu_host_free(self.ctx, self.ptr) };
    }
}

fn pinned_bytes(ctx: *mut ffi::flockgpu_ctx, src: &[u8]) -> Option<PinnedBlock> {
    let mut p: *mut c_void = std::ptr::null_mut();
    if unsafe { ffi::flockgpu_host_alloc(ctx, src.len().max(8) as i64, &mut p) } != ffi::FLOCKGPU_OK {
        return None;
    }
    unsafe { std::ptr::copy_nonoverlapping(src.as_ptr(), p as *mut u8, src.len()) };
    Some(PinnedBlock { ctx, ptr: p })
}

/// Private data of an exported array: the blocks its buffer pointers refer to.
struct Exported {
    blocks: Vec<PinnedBlock>,
    buffers: Vec<*const c_void>,
}

unsafe extern "C" fn release_exported(array: *mut FFI_ArrowArray) {
    // the layout of FFI_ArrowArray is the C struct ArrowArray: private_data is ours
    let a = &mut *(array as *mut RawArrowArray);
    drop(Box::from_raw(a.private_data as *mut Exported)); // frees the page-locked blocks
    a.release = None;
}

/// `struct ArrowArray` (arrow/c/abi.h), field for field.
#[repr(C)]
struct RawArrowArray {
    length: i64,
    null_count: i64,
    offset: i64,
    n_buffers: i64,
    n_children: i64,
    buffers: *mut *const c_void,
    children: *mut *mut RawArrowArray,
    dictionary: *mut RawArrowArray,
    release: Option<unsafe extern "C" fn(*mut FFI_ArrowArray)>,
    private_data: *mut c_void,
}

/// A copy of `column` whose buffers are page-locked (fixed-width and Utf8 columns; validity included).
pub fn pinned_column(ctx: *mut ffi::flockgpu_ctx, column: &ArrayRef) -> ArrowResult<ArrayRef> {
    let data = column.data();
    let mut exported = Box::new(Exported { blocks: vec![], buffers: vec![] });
    // buffer 0 of the C Data Interface is the validity bitmap (NULL when there is none)
    match data.null_buffer() {
        Some(b) => {
            let blk = pinned_bytes(ctx, b.as_slice()).expect("flockgpu_host_alloc");
            exported.buffers.push(blk.ptr as *const c_void);
            exported.blocks.push(blk);
        }
        None => exported.buffers.push(std::ptr::null()),
    }
    for b in data.buffers() {
        let blk = pinned_bytes(ctx, b.as_slice()).expect("flockgpu_host_alloc");
        exported.buffers.push(blk.ptr as *const c_void);
        exported.blocks.push(blk);
    }
    let raw = Box::new(RawArrowArray {
        length: data.len() as i64,
        null_count: data.null_count() as i64,
        offset: data.offset() as i64,
        n_buffers: exported.buffers.len() as i64,
        n_children: 0,
        buffers: exported.buffers.as_mut_ptr(),
        children: std::ptr::null_mut(),
        dictionary: std::ptr::null_mut(),
        release: Some(release_exported),
        private_data: Box::into_raw(exported) as *mut c_void,
    });
    let schema = FFI_ArrowSchema::try_from(data.data_type())?;
    // arrow takes ownership of both structs and calls `release` when the last buffer is dropped
    unsafe { make_array_from_raw(Box::into_raw(raw) as *const FFI_ArrowArray, Box::into_raw(Box::new(schema)) as *const FFI_ArrowSchema) }
}

/// The batch with every column in page-locked memory: what `feed_zero_copy` reads in place over PCIe.
pub fn pinned_batch(ctx: *mut ffi::flockgpu_ctx, batch: &RecordBatch) -> ArrowResult<RecordBatch> {
    let columns = batch.columns().iter().map(|c| pinned_column(ctx, c)).collect::<ArrowResult<Vec<_>>>()?;
    RecordBatch::try_new(batch.schema(), columns)
}

/// `Payload::to_record_batch` WITHOUT going through host record batches at all: the frames go straight to a device
/// table (flockgpu_table_import_payload), which `flock_context_feed_tables` hands to the plan.  `encoding` is the
/// payload's `Encoding` (`payload.encoding as i32`): Zstd frames (Flock's default) are decompressed on the GPU, so the
/// CPU decompress is gone; None frames are imported as they are.  `None` back (FLOCKGPU_ERR_UNSUPPORTED for Snappy /
/// Lz4 / Zlib, or any error): the caller keeps its CPU route for this payload.
pub fn frames_to_table(
    ctx: *mut ffi::flockgpu_ctx,
    schema: &FFI_ArrowSchema,
    encoding: i32,
    frames: &[(Vec<u8>, Vec<u8>)], // DataFrame { header, body }, as they arrived (compressed with `encoding`)
) -> Option<*mut ffi::flockgpu_table> {
    let headers: Vec<*const u8> = frames.iter().map(|f| f.0.as_ptr()).collect();
    let header_lens: Vec<i64> = frames.iter().map(|f| f.0.len() as i64).collect();
    let bodies: Vec<*const u8> = frames.iter().map(|f| f.1.as_ptr()).collect();
    let body_lens: Vec<i64> = frames.iter().map(|f| f.1.len() as i64).collect();
    let mut out = std::ptr::null_mut();
    let rc = unsafe {
        ffi::flockgpu_table_import_payload(
            ctx,
            schema,
            encoding,
            headers.as_ptr(),
            header_lens.as_ptr(),
            bodies.as_ptr(),
            body_lens.as_ptr(),
            frames.len() as i32,
            std::ptr::null(),
            0,
            &mut out,
        )
    };
    if rc == ffi::FLOCKGPU_OK {
        Some(out)
    } else {
        None
    }
}

/// `to_payload` (flock/src/transmute.rs:178-221) WITHOUT host record batches: the device table becomes the payload's
/// DataFrames { header, body } (flockgpu_table_export_payload); with Encoding::Zstd (`encoding = 3`, Flock's default)
/// the bodies are compressed on the GPU and only compressed bytes cross the link.  `rows_per_frame: None` picks a frame
/// size whose body stays within the 10 MiB Flock's receiver decompresses into (flock/src/encoding.rs:92): at most
/// 65,536 rows and about 8 MiB of the table's bytes per frame, halved while a frame is still too large.  `None` back
/// (FLOCKGPU_ERR_UNSUPPORTED for Snappy / Lz4 / Zlib, or any other error): the caller keeps its CPU route.
pub fn table_to_frames(
    ctx: *mut ffi::flockgpu_ctx,
    table: *const ffi::flockgpu_table,
    encoding: i32,
    rows_per_frame: Option<i64>,
) -> Option<Vec<(Vec<u8>, Vec<u8>)>> {
    let rows = unsafe { ffi::flockgpu_table_num_rows(table) }.max(1);
    let bytes = unsafe { ffi::flockgpu_table_nbytes(table) }.max(1);
    let mut rpf = rows_per_frame.unwrap_or_else(|| ((8i64 << 20) as i128 * rows as i128 / bytes as i128).clamp(1, 65536) as i64);
    loop {
        let mut p = std::ptr::null_mut();
        let rc = unsafe { ffi::flockgpu_table_export_payload(ctx, table, encoding, rpf, &mut p) };
        if rc == ffi::FLOCKGPU_ERR_INVALID && rows_per_frame.is_none() && rpf > 1 {
            rpf /= 2; // a frame's body is over 10 MiB: smaller frames
            continue;
        }
        if rc != ffi::FLOCKGPU_OK {
            return None;
        }
        let n = unsafe { ffi::flockgpu_payload_num_frames(p) };
        let mut frames = Vec::with_capacity(n as usize);
        for i in 0..n {
            let (mut h, mut hl, mut b, mut bl) = (std::ptr::null(), 0i64, std::ptr::null(), 0i64);
            if unsafe { ffi::flockgpu_payload_frame(p, i, &mut h, &mut hl, &mut b, &mut bl) } != ffi::FLOCKGPU_OK {
                unsafe { ffi::flockgpu_payload_free(p) };
                return None;
            }
            let copy = |ptr: *const u8, len: i64| if len == 0 { vec![] } else { unsafe { std::slice::from_raw_parts(ptr, len as usize) }.to_vec() };
            frames.push((copy(h, hl), copy(b, bl)));
        }
        unsafe { ffi::flockgpu_payload_free(p) };
        return Some(frames);
    }
}

#[allow(dead_code)]
fn _uses(_: &StructArray) {}
