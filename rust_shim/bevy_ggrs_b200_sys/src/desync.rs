//! `#[repr(C)]` mirrors of the desync capture structs of `include/bevy_ggrs_b200.h` (BGR_CFG_DESYNC_CAPTURE).

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_desync_column {
    pub rows: u32,
    pub rows_in_checksum: u32,
    pub presence: u32,
    pub reserved: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_desync_record {
    pub row: u32,
    pub column: u32,
    pub word: u32,
    pub first: u32,
    pub latest: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_desync_summary {
    pub frame: i32,
    pub rows_first: u32,
    pub rows_latest: u32,
    pub rows_differing: u32,
    pub existence_differing: u32,
    pub host_state_differs: u32,
    pub words_differing: u64,
    pub elapsed_ns_first: u64,
    pub elapsed_ns_latest: u64,
}
