//! `#[repr(C)]` mirrors of the host edit structs of `include/bevy_ggrs_b200.h` (bgr_apply_edits), and the batched
//! edits over a world batch (bgr_batch_apply_edits).

use crate::*;
use core::ptr;

pub const BGR_EDIT_WRITE: u32 = 0;
pub const BGR_EDIT_INSERT: u32 = 1;
pub const BGR_EDIT_REMOVE: u32 = 2;
pub const BGR_EDIT_DESPAWN: u32 = 3;
pub const BGR_EDIT_SPAWN: u32 = 4;

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_edit {
    pub kind: u32,
    pub column: u32,
    pub row: u32,
    pub count: u32,
    pub byte_offset: u32,
    pub byte_len: u32,
    pub value_offset: u32,
    pub reserved: u32,
}

/// One entry of a batched edit call: bgr_apply_edits' arguments for member `world`.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct bgr_batch_edits {
    pub world: u32,
    pub n_edits: u32,
    pub edits: *const bgr_edit,
    pub values: *const c_void,
    pub values_bytes: usize,
}

/// One world's share of `Batch::apply_edits`: its records and the bytes their WRITE / INSERT records point into.
pub struct BatchEdits<'a> {
    pub world: u32,
    pub edits: &'a [bgr_edit],
    pub values: &'a [u8],
}

impl Batch {
    /// bgr_apply_edits of every entry on its world in one queued call (at most one spawn launch and one patch launch
    /// over all of them); the slices are free on return.  All or nothing: Err(status) (and bgr_last_error() naming the
    /// world) leaves every world as it was.
    pub fn apply_edits(&mut self, entries: &[BatchEdits]) -> Result<(), c_int> {
        let raw: Vec<bgr_batch_edits> = entries.iter().map(|x| bgr_batch_edits {
            world: x.world,
            n_edits: x.edits.len() as u32,
            edits: if x.edits.is_empty() { ptr::null() } else { x.edits.as_ptr() },
            values: if x.values.is_empty() { ptr::null() } else { x.values.as_ptr() as *const c_void },
            values_bytes: x.values.len(),
        }).collect();
        let mut status = vec![0i32; entries.len()];
        let rc = unsafe { bgr_batch_apply_edits(self.raw, raw.as_ptr(), raw.len() as u32, status.as_mut_ptr()) };
        if rc == BGR_OK { Ok(()) } else { Err(rc) }
    }
}
