//! `#[repr(C)]` mirror of the world checkpoint header of `include/bevy_ggrs_b200.h` (bgr_checkpoint_save /
//! bgr_checkpoint_restore).

pub const BGR_CHECKPOINT_MAGIC: u32 = 0x43524742;
pub const BGR_CHECKPOINT_VERSION: u32 = 1;
pub const BGR_CKPT_CONST: u32 = 0;
pub const BGR_CKPT_SPARSE: u32 = 1;
pub const BGR_CKPT_RAW: u32 = 2;

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
