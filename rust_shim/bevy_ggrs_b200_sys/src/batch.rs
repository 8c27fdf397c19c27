//! A safe owner of a world batch (bgr_batch_create / bgr_batch_handle_requests / bgr_batch_destroy): the request
//! vectors of many engines with one registration in one kernel launch.

use crate::*;
use core::ptr;

/// One call's worth of a world: its index in the batch, its session and its request vector.
pub struct BatchCall<'a> {
    pub world: u32,
    pub session: bgr_session_info,
    pub requests: &'a [bgr_request],
}

/// Owns a `bgr_batch`; the engines it was created from must outlive it (dropping it destroys the batch first).
pub struct Batch {
    pub(crate) raw: *mut bgr_batch,
    /// entries of the batched feed report in flight (`feed_begin`): the infos its wait writes
    pub(crate) feed_entries: usize,
}

impl Batch {
    /// `engines`: built engines with one registration, created with the same non-null `bgr_config.stream`.
    pub fn new(engines: &[*mut bgr_engine]) -> Result<Batch, c_int> {
        let mut raw = ptr::null_mut();
        let rc = unsafe { bgr_batch_create(engines.as_ptr(), engines.len() as u32, &mut raw) };
        if rc != BGR_OK { Err(rc) } else { Ok(Batch { raw, feed_entries: 0 }) }
    }

    /// True when calls run as one launch; false: each world's own bgr_handle_requests runs in turn.
    pub fn specialised(&self) -> bool {
        let mut v = 0u32;
        unsafe { bgr_batch_specialised(self.raw, &mut v) };
        v != 0
    }

    /// Runs `calls` in one synchronous call.  Err(status) when the call was refused before anything executed;
    /// otherwise each world's status (what its own bgr_handle_requests would have returned) and checksums, in order.
    pub fn handle_requests(&mut self, calls: &[BatchCall]) -> Result<Vec<(c_int, Vec<bgr_checksum>)>, c_int> {
        let worlds: Vec<u32> = calls.iter().map(|c| c.world).collect();
        let sessions: Vec<bgr_session_info> = calls.iter().map(|c| c.session).collect();
        let requests: Vec<bgr_request> = calls.iter().flat_map(|c| c.requests.iter().copied()).collect();
        let n_requests: Vec<u32> = calls.iter().map(|c| c.requests.len() as u32).collect();
        let cap = requests.iter().filter(|r| r.kind == BGR_REQ_SAVE).count();
        let mut out = vec![bgr_checksum::default(); cap];
        let mut n_out = vec![0u32; calls.len()];
        let mut status = vec![0i32; calls.len()];
        let rc = unsafe {
            bgr_batch_handle_requests(self.raw, worlds.as_ptr(), calls.len() as u32, sessions.as_ptr(), requests.as_ptr(),
                                      n_requests.as_ptr(), out.as_mut_ptr(), cap as u32, n_out.as_mut_ptr(), status.as_mut_ptr())
        };
        if rc != BGR_OK && rc != BGR_ERR_NON_FINITE {
            return Err(rc);
        }
        let mut at = 0usize;
        Ok(status.iter().zip(n_out.iter()).map(|(&s, &n)| {
            let cs = out[at..at + n as usize].to_vec();
            at += n as usize;
            (s, cs)
        }).collect())
    }
}

impl Drop for Batch {
    fn drop(&mut self) {
        unsafe { bgr_batch_destroy(self.raw) };
    }
}
