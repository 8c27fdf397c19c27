//! `#[repr(C)]` mirror of `struct bgr_replay` of `include/bevy_ggrs_b200.h` and safe calls over it (bgr_replay /
//! bgr_batch_replay): a recorded input log run through a world, checksummed every `checksum_interval` frames, without
//! pushing snapshots.

use crate::*;
use core::ptr;

pub const BGR_MAX_REPLAY_FRAMES: u32 = 1 << 24;

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct bgr_replay {
    pub n_frames: u32,
    pub n_players: u32,
    pub checksum_interval: u32,
    pub reserved: u32,
    pub inputs: *const u8,
}

/// An input log: `inputs[j * n_players + h]` is player h's input of frame j.
pub struct ReplayLog<'a> {
    pub n_players: u32,
    pub inputs: &'a [u8],
    pub checksum_interval: u32,
}

impl<'a> ReplayLog<'a> {
    /// Err(BGR_ERR_INVALID_ARGUMENT) when the log is not a whole number of frames.
    fn check(&self) -> Result<(), c_int> {
        if self.n_players != 0 && self.inputs.len() % self.n_players as usize != 0 { Err(BGR_ERR_INVALID_ARGUMENT) } else { Ok(()) }
    }

    fn raw(&self) -> bgr_replay {
        let n_frames = if self.n_players == 0 { 0 } else { (self.inputs.len() / self.n_players as usize) as u32 };
        bgr_replay {
            n_frames,
            n_players: self.n_players,
            checksum_interval: self.checksum_interval,
            reserved: 0,
            inputs: if self.inputs.is_empty() { ptr::null() } else { self.inputs.as_ptr() },
        }
    }

    /// Checksum frames of the log for an engine at RollbackFrameCount `f0`.
    fn points(&self, f0: i32) -> usize {
        let (n, k) = (self.raw().n_frames as i64, self.checksum_interval as i64);
        if k == 0 || f0 < 0 { return 0; }
        let f0 = f0 as i64;
        ((f0 + n + k - 1) / k - (f0 + k - 1) / k) as usize
    }
}

/// Replays `log` on `e` from its current frame.  Ok: the checksums of the checksum frames in order; Err(status, those
/// checksums): BGR_ERR_NON_FINITE after the whole log ran, or a refusal that changed nothing (no checksums).
pub fn replay(e: *mut bgr_engine, log: &ReplayLog) -> Result<Vec<bgr_checksum>, (c_int, Vec<bgr_checksum>)> {
    log.check().map_err(|rc| (rc, Vec::new()))?;
    let mut f0 = 0i32;
    unsafe { bgr_rollback_frame_count(e, &mut f0) };
    let r = log.raw();
    let mut out = vec![bgr_checksum::default(); log.points(f0)];
    let mut n = 0u32;
    let rc = unsafe { bgr_replay(e, &r, out.as_mut_ptr(), out.len() as u32, &mut n) };
    out.truncate((n as usize).min(out.len()));
    if rc == BGR_OK { Ok(out) } else { Err((rc, out)) }
}

impl Batch {
    /// Replays `logs[i]` on world `worlds[i]` in one synchronous call.  Err(status) when the call was refused before
    /// anything executed; otherwise each world's status and checksums, in order.  `f0s[i]` is world i's
    /// RollbackFrameCount before the call (it sizes the result).
    pub fn replay(&mut self, worlds: &[u32], f0s: &[i32], logs: &[ReplayLog]) -> Result<Vec<(c_int, Vec<bgr_checksum>)>, c_int> {
        for l in logs { l.check()?; }
        let reps: Vec<bgr_replay> = logs.iter().map(|l| l.raw()).collect();
        let cap: usize = logs.iter().zip(f0s.iter()).map(|(l, &f0)| l.points(f0)).sum();
        let mut out = vec![bgr_checksum::default(); cap];
        let mut n_out = vec![0u32; worlds.len()];
        let mut status = vec![0i32; worlds.len()];
        let rc = unsafe {
            bgr_batch_replay(self.raw, worlds.as_ptr(), worlds.len() as u32, reps.as_ptr(), out.as_mut_ptr(), cap as u32,
                             n_out.as_mut_ptr(), status.as_mut_ptr())
        };
        if rc != BGR_OK && rc != BGR_ERR_NON_FINITE {
            return Err(rc);
        }
        // n_out holds each world's full count; only what fits `cap` was written (a wrong f0 sized it too small)
        let mut at = 0usize;
        Ok(status.iter().zip(n_out.iter()).map(|(&s, &n)| {
            let end = (at + n as usize).min(cap);
            let cs = out[at.min(cap)..end].to_vec();
            at += n as usize;
            (s, cs)
        }).collect())
    }
}
