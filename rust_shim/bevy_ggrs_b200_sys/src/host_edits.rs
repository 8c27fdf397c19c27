//! `#[repr(C)]` mirror of the host edit record of `include/bevy_ggrs_b200.h` (bgr_apply_edits).

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
