//! `#[repr(C)]` mirrors of the P2P desync report structs of `include/bevy_ggrs_b200.h`.

pub const BGR_DIGEST_BLOCK_ROWS: u32 = 512;
pub const BGR_FRAME_BLOB_MAGIC: u32 = 0x50424752;
pub const BGR_FRAME_BLOB_VERSION: u32 = 1;

#[repr(C)]
#[derive(Clone, Copy, Default, Debug, PartialEq, Eq)]
pub struct bgr_frame_digest_header {
    pub layout: u64,
    pub frame: i32,
    pub rows: u32,
    pub n_blocks: u32,
    pub n_columns: u32,
    pub active: u64,
    pub elapsed_ns: u64,
    pub rng: [u64; 4],
    pub root: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_frame_blob_header {
    pub magic: u32,
    pub version: u32,
    pub layout: u64,
    pub frame: i32,
    pub rows: u32,
    pub words: u32,
    pub n_blocks: u32,
    pub n_exported: u32,
    pub reserved: u32,
    pub elapsed_ns: u64,
    pub rng: [u64; 4],
}
