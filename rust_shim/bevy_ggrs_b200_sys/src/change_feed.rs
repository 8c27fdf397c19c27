//! `#[repr(C)]` mirrors of the change feed structs of `include/bevy_ggrs_b200.h` (bgr_feed_*).

pub const BGR_MAX_FEEDS: u32 = 8;
pub const BGR_MAX_FEED_FIELDS: u32 = 8;

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_feed_field {
    pub column: u32,
    pub byte_offset: u32,
    pub byte_len: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_feed_info {
    pub n_records: u32,
    pub pending: u32,
    pub rows: u32,
    pub record_bytes: u32,
}
