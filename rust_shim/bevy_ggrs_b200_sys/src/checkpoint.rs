//! `#[repr(C)]` mirror of the world checkpoint header of `include/bevy_ggrs_b200.h` (bgr_checkpoint_save /
//! bgr_checkpoint_restore), and the batched calls over a world batch (bgr_batch_checkpoint_save /
//! bgr_batch_checkpoint_restore).  The checkpoint delta header and its safe calls (bgr_checkpoint_save_delta /
//! bgr_checkpoint_restore_delta): a frame coded against a base frame's checkpoint, restored from the two.

use crate::*;
use core::ptr;

pub const BGR_CHECKPOINT_MAGIC: u32 = 0x43524742;
pub const BGR_CHECKPOINT_VERSION: u32 = 1;
pub const BGR_CKPT_CONST: u32 = 0;
pub const BGR_CKPT_SPARSE: u32 = 1;
pub const BGR_CKPT_RAW: u32 = 2;
pub const BGR_CHECKPOINT_DELTA_MAGIC: u32 = 0x44524742;
pub const BGR_CHECKPOINT_DELTA_VERSION: u32 = 1;

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_checkpoint_header {
    pub magic: u32,
    pub version: u32,
    pub layout: u64,
    pub frame: i32,
    pub rows: u32,
    pub words: u32,
    pub n_blocks: u32,
    pub n_columns: u32,
    pub fps: u32,
    pub active: u64,
    pub elapsed_ns: u64,
    pub rng: [u64; 4],
    pub digest_root: u64,
    pub payload_bytes: u64,
}

/// 120 bytes, no padding, as in the C header
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_checkpoint_delta_header {
    pub magic: u32,
    pub version: u32,
    pub layout: u64,
    pub frame: i32,
    pub rows: u32,
    pub base_frame: i32,
    pub base_rows: u32,
    pub words: u32,
    pub n_blocks: u32,
    pub n_columns: u32,
    pub fps: u32,
    pub active: u64,
    pub elapsed_ns: u64,
    pub rng: [u64; 4],
    pub digest_root: u64,
    pub base_root: u64,
    pub payload_bytes: u64,
}

/// The checkpoint delta of `frame` against `base_frame`, sized by the call's query.  `Ok(None)` where the engine holds
/// either frame neither queued nor retained.  Err(status) when refused.
pub fn save_delta(e: *mut bgr_engine, frame: i32, base_frame: i32) -> Result<Option<Vec<u8>>, c_int> {
    let mut size = 0usize;
    let mut found = 0i32;
    let rc = unsafe { bgr_checkpoint_save_delta(e, frame, base_frame, ptr::null_mut(), 0, &mut size, &mut found) };
    if rc != BGR_OK {
        return Err(rc);
    }
    if found == 0 {
        return Ok(None);
    }
    let mut dst = vec![0u8; size]; // an upper bound: the call reports the exact size
    let rc = unsafe {
        bgr_checkpoint_save_delta(e, frame, base_frame, dst.as_mut_ptr() as *mut c_void, dst.len(), &mut size, &mut found)
    };
    if rc != BGR_OK {
        return Err(rc);
    }
    dst.truncate(size);
    Ok(Some(dst))
}

/// Restores the delta's target frame from the full checkpoint `base` it was written against.  Err(status) leaves the
/// engine as it was.
pub fn restore_delta(e: *mut bgr_engine, base: &[u8], delta: &[u8]) -> Result<(), c_int> {
    let rc = unsafe {
        bgr_checkpoint_restore_delta(e, base.as_ptr() as *const c_void, base.len(), delta.as_ptr() as *const c_void,
                                     delta.len())
    };
    if rc == BGR_OK { Ok(()) } else { Err(rc) }
}

impl Batch {
    /// The checkpoints of `frames[i]` on world `worlds[i]` in one call (one encoding pass, one copy back), sized by the
    /// call's query.  `None` where the world holds that frame neither queued nor retained.  Err(status) when refused.
    pub fn checkpoint(&mut self, worlds: &[u32], frames: &[i32]) -> Result<Vec<Option<Vec<u8>>>, c_int> {
        if worlds.len() != frames.len() {
            return Err(BGR_ERR_INVALID_ARGUMENT);
        }
        let n = worlds.len() as u32;
        let mut index = vec![bgr_keyframe::default(); worlds.len()];
        let mut status = vec![0i32; worlds.len()];
        let mut size = 0usize;
        let rc = unsafe {
            bgr_batch_checkpoint_save(self.raw, worlds.as_ptr(), n, frames.as_ptr(), ptr::null_mut(), 0, index.as_mut_ptr(),
                                      &mut size, status.as_mut_ptr())
        };
        if rc != BGR_OK {
            return Err(rc);
        }
        let mut dst = vec![0u8; size];
        let rc = unsafe {
            bgr_batch_checkpoint_save(self.raw, worlds.as_ptr(), n, frames.as_ptr(), dst.as_mut_ptr() as *mut c_void, dst.len(),
                                      index.as_mut_ptr(), &mut size, status.as_mut_ptr())
        };
        if rc != BGR_OK {
            return Err(rc);
        }
        Ok(index.iter().map(|k| if k.bytes == 0 { None } else {
            Some(dst[k.offset as usize..(k.offset + k.bytes) as usize].to_vec())
        }).collect())
    }

    /// Restores `blobs[i]` into world `worlds[i]` in one call (one decoding pass).  All or nothing: Err(status) (and
    /// bgr_last_error() naming the world) leaves every world as it was.
    pub fn restore(&mut self, worlds: &[u32], blobs: &[&[u8]]) -> Result<(), c_int> {
        if worlds.len() != blobs.len() {
            return Err(BGR_ERR_INVALID_ARGUMENT);
        }
        let ptrs: Vec<*const c_void> = blobs.iter().map(|b| b.as_ptr() as *const c_void).collect();
        let sizes: Vec<usize> = blobs.iter().map(|b| b.len()).collect();
        let mut status = vec![0i32; worlds.len()];
        let rc = unsafe {
            bgr_batch_checkpoint_restore(self.raw, worlds.as_ptr(), worlds.len() as u32, ptrs.as_ptr(), sizes.as_ptr(),
                                         status.as_mut_ptr())
        };
        if rc == BGR_OK { Ok(()) } else { Err(rc) }
    }
}
