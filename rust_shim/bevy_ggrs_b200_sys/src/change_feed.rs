//! `#[repr(C)]` mirrors of the change feed structs of `include/bevy_ggrs_b200.h` (bgr_feed_*), and the batched report
//! over a world batch (bgr_batch_feed_begin / bgr_batch_feed_wait).

use crate::*;

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

/// One entry of a batched report: feed `feed` of member `world`, at most `records_cap` records.
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct bgr_batch_feed {
    pub world: u32,
    pub feed: u32,
    pub records_cap: u32,
}

impl Batch {
    /// Starts one report of every entry into `host_dst`, page-locked memory from bgr_host_alloc holding sum(records_cap)
    /// records (null when every cap is 0); returns its ticket.  Err(status) when refused (bgr_last_error() names the
    /// world), and then no feed changed.
    ///
    /// # Safety
    /// `host_dst` must stay valid, and unread, until `feed_wait` of the ticket returns.
    pub unsafe fn feed_begin(&mut self, reports: &[bgr_batch_feed], host_dst: *mut c_void) -> Result<u32, c_int> {
        let mut ticket = 0u32;
        let mut status = vec![0i32; reports.len()];
        let rc = bgr_batch_feed_begin(self.raw, reports.as_ptr(), reports.len() as u32, host_dst, &mut ticket, status.as_mut_ptr());
        if rc != BGR_OK {
            return Err(rc);
        }
        self.feed_entries = reports.len();  // one batched report per batch is in flight
        Ok(ticket)
    }

    /// Waits for a batched report: the info of each entry in list order, as many as its `feed_begin` listed.  Entry
    /// i's records start in `host_dst` at the sum of the earlier entries' n_records.  An unknown or already-waited
    /// ticket is Err(BGR_ERR_STATE) and writes nothing.
    pub fn feed_wait(&mut self, ticket: u32) -> Result<Vec<bgr_feed_info>, c_int> {
        // room for every info the report in flight writes, whatever ticket the caller passes
        let mut infos = vec![bgr_feed_info::default(); self.feed_entries.max(1)];
        let rc = unsafe { bgr_batch_feed_wait(self.raw, ticket, infos.as_mut_ptr()) };
        if rc != BGR_OK {
            return Err(rc);
        }
        infos.truncate(self.feed_entries);
        self.feed_entries = 0;
        Ok(infos)
    }
}
