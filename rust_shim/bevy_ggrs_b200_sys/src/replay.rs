//! `#[repr(C)]` mirror of `struct bgr_replay` of `include/bevy_ggrs_b200.h` and safe calls over it (bgr_replay /
//! bgr_batch_replay): a recorded input log run through a world, checksummed every `checksum_interval` frames, without
//! pushing snapshots.  With keyframes (bgr_replay_keyframes / bgr_batch_replay_keyframes) the replay also returns a
//! world checkpoint every `keyframe_interval` frames, the seek points of a recorded match.  With a trace
//! (bgr_replay_trace / bgr_batch_replay_trace) it also returns the change-feed records of a row range every
//! `interval` frames, what a replay viewer draws or a match-analytics job mines.

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

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct bgr_keyframe {
    pub frame: i32,
    pub reserved: u32,
    pub offset: u64,
    pub bytes: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct bgr_keyframes {
    pub interval: u32,
    pub index_cap: u32,
    pub reserved: u64,
    pub dst: *mut c_void,
    pub dst_cap: usize,
    pub index: *mut bgr_keyframe,
}

/// A replay's keyframes: `(frame, blob)` in frame order, each blob what `bgr_checkpoint_save` writes.
pub type Keyframes = Vec<(i32, Vec<u8>)>;

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

/// Keyframe buffers sized by a query (dst NULL) of `log` on `e`, which runs nothing.
struct KeyframeBuffers {
    dst: Vec<u8>,
    index: Vec<bgr_keyframe>,
}

impl KeyframeBuffers {
    fn query(e: *mut bgr_engine, r: &bgr_replay, interval: u32) -> Result<Self, c_int> {
        let q = bgr_keyframes { interval, index_cap: 0, reserved: 0, dst: ptr::null_mut(), dst_cap: 0, index: ptr::null_mut() };
        let (mut n_cs, mut n_kf, mut bytes) = (0u32, 0u32, 0usize);
        let rc = unsafe { bgr_replay_keyframes(e, r, &q, ptr::null_mut(), 0, &mut n_cs, &mut n_kf, &mut bytes) };
        if rc != BGR_OK { return Err(rc); }
        Ok(KeyframeBuffers { dst: vec![0u8; bytes.max(1)], index: vec![bgr_keyframe::default(); (n_kf as usize).max(1)] })
    }

    fn raw(&mut self, interval: u32) -> bgr_keyframes {
        bgr_keyframes {
            interval,
            index_cap: self.index.len() as u32,
            reserved: 0,
            dst: self.dst.as_mut_ptr() as *mut c_void,
            dst_cap: self.dst.len(),
            index: self.index.as_mut_ptr(),
        }
    }

    /// The first `n` blobs, clamped to what the buffers hold.
    fn blobs(&self, n: u32) -> Keyframes {
        self.index.iter().take((n as usize).min(self.index.len())).map(|k| {
            let a = (k.offset as usize).min(self.dst.len());
            let b = (a + k.bytes as usize).min(self.dst.len());
            (k.frame, self.dst[a..b].to_vec())
        }).collect()
    }
}

/// `replay` that also returns a keyframe every `keyframe_interval` frames.  Err(status, checksums, keyframes):
/// BGR_ERR_NON_FINITE after the whole log ran (the keyframes are written), or a refusal that changed nothing.
pub fn replay_keyframes(e: *mut bgr_engine, log: &ReplayLog, keyframe_interval: u32)
                        -> Result<(Vec<bgr_checksum>, Keyframes), (c_int, Vec<bgr_checksum>, Keyframes)> {
    log.check().map_err(|rc| (rc, Vec::new(), Vec::new()))?;
    let mut f0 = 0i32;
    unsafe { bgr_rollback_frame_count(e, &mut f0) };
    let r = log.raw();
    let mut bufs = KeyframeBuffers::query(e, &r, keyframe_interval).map_err(|rc| (rc, Vec::new(), Vec::new()))?;
    let kf = bufs.raw(keyframe_interval);
    let mut out = vec![bgr_checksum::default(); log.points(f0)];
    let (mut n, mut n_kf, mut bytes) = (0u32, 0u32, 0usize);
    let rc = unsafe { bgr_replay_keyframes(e, &r, &kf, out.as_mut_ptr(), out.len() as u32, &mut n, &mut n_kf, &mut bytes) };
    out.truncate((n as usize).min(out.len()));
    let blobs = bufs.blobs(n_kf);
    if rc == BGR_OK { Ok((out, blobs)) } else { Err((rc, out, blobs)) }
}

impl Batch {
    /// `replay` of `logs[i]` on world `worlds[i]` with keyframes every `keyframe_intervals[i]` frames, in one
    /// synchronous call.  `engines[i]` is world i's engine: its query sizes the world's buffers.  Err(status) when the
    /// call was refused before anything executed; otherwise each world's status, checksums and keyframes, in order.
    pub fn replay_keyframes(&mut self, worlds: &[u32], engines: &[*mut bgr_engine], f0s: &[i32], logs: &[ReplayLog],
                            keyframe_intervals: &[u32]) -> Result<Vec<(c_int, Vec<bgr_checksum>, Keyframes)>, c_int> {
        for l in logs { l.check()?; }
        let reps: Vec<bgr_replay> = logs.iter().map(|l| l.raw()).collect();
        let mut bufs = Vec::with_capacity(worlds.len());
        for i in 0..worlds.len() { bufs.push(KeyframeBuffers::query(engines[i], &reps[i], keyframe_intervals[i])?); }
        let kfs: Vec<bgr_keyframes> = bufs.iter_mut().zip(keyframe_intervals.iter()).map(|(b, &k)| b.raw(k)).collect();
        let cap: usize = logs.iter().zip(f0s.iter()).map(|(l, &f0)| l.points(f0)).sum();
        let mut out = vec![bgr_checksum::default(); cap];
        let mut n_out = vec![0u32; worlds.len()];
        let mut n_kf = vec![0u32; worlds.len()];
        let mut status = vec![0i32; worlds.len()];
        let rc = unsafe {
            bgr_batch_replay_keyframes(self.raw, worlds.as_ptr(), worlds.len() as u32, reps.as_ptr(), kfs.as_ptr(),
                                       out.as_mut_ptr(), cap as u32, n_out.as_mut_ptr(), n_kf.as_mut_ptr(), status.as_mut_ptr())
        };
        if rc != BGR_OK && rc != BGR_ERR_NON_FINITE {
            return Err(rc);
        }
        let mut at = 0usize;
        Ok((0..worlds.len()).map(|i| {
            let end = (at + n_out[i] as usize).min(cap);
            let cs = out[at.min(cap)..end].to_vec();
            at += n_out[i] as usize;
            (status[i], cs, bufs[i].blobs(n_kf[i]))
        }).collect())
    }
}

/// One sample of a trace: its frame and RollbackOrdered::len() there.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct bgr_trace_sample {
    pub frame: i32,
    pub rows: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct bgr_trace {
    pub interval: u32,
    pub first_row: u32,
    pub n_rows: u32,
    pub n_fields: u32,
    pub fields: *const bgr_feed_field,
    pub dst: *mut c_void,
    pub dst_cap: usize,
    pub samples: *mut bgr_trace_sample,
    pub samples_cap: u32,
    pub reserved: u32,
}

const _: () = assert!(core::mem::size_of::<bgr_trace_sample>() == 8);
const _: () = assert!(core::mem::size_of::<bgr_trace>() == 56);

/// What a trace records: every `interval` frames, rows [first_row, first_row + n_rows) as change-feed records over
/// `fields`.
pub struct TraceSpec<'a> {
    pub interval: u32,
    pub first_row: u32,
    pub n_rows: u32,
    pub fields: &'a [bgr_feed_field],
}

/// A replay's trace: the samples in frame order, and n_samples * n_rows records of `record_bytes` each, sample-major.
pub struct Trace {
    pub samples: Vec<bgr_trace_sample>,
    pub records: Vec<u8>,
}

impl<'a> TraceSpec<'a> {
    fn raw(&self, t: Option<&mut Trace>) -> bgr_trace {
        let (dst, dst_cap, samples, samples_cap) = match t {
            // never a null dst, which is the query: a log may take no sample
            Some(t) => (t.records.as_mut_ptr() as *mut c_void, t.records.len() - 1, t.samples.as_mut_ptr(), t.samples.len() as u32 - 1),
            None => (ptr::null_mut(), 0, ptr::null_mut(), 0),
        };
        bgr_trace {
            interval: self.interval,
            first_row: self.first_row,
            n_rows: self.n_rows,
            n_fields: self.fields.len() as u32,
            fields: self.fields.as_ptr(),
            dst,
            dst_cap,
            samples,
            samples_cap,
            reserved: 0,
        }
    }

    /// Buffers sized by a query (dst NULL) of `r` on `e`, which runs nothing (one spare byte and sample each).
    fn query(&self, e: *mut bgr_engine, r: &bgr_replay) -> Result<Trace, c_int> {
        let q = self.raw(None);
        let (mut n_cs, mut n_s, mut bytes) = (0u32, 0u32, 0usize);
        let rc = unsafe { bgr_replay_trace(e, r, &q, ptr::null_mut(), 0, &mut n_cs, &mut n_s, &mut bytes) };
        if rc != BGR_OK { return Err(rc); }
        Ok(Trace { samples: vec![bgr_trace_sample::default(); n_s as usize + 1], records: vec![0u8; bytes + 1] })
    }
}

impl Trace {
    fn finish(mut self, n_samples: u32) -> Trace {
        let n = (n_samples as usize).min(self.samples.len() - 1);
        let per = if self.samples.len() > 1 { (self.records.len() - 1) / (self.samples.len() - 1) } else { 0 };
        self.samples.truncate(n);
        self.records.truncate(n * per);
        self
    }
}

/// `replay` that also returns a trace.  Err(status, checksums, trace): BGR_ERR_NON_FINITE after the whole log ran
/// (every sample is written), or a refusal that changed nothing.
pub fn replay_trace(e: *mut bgr_engine, log: &ReplayLog, spec: &TraceSpec)
                    -> Result<(Vec<bgr_checksum>, Trace), (c_int, Vec<bgr_checksum>, Option<Trace>)> {
    log.check().map_err(|rc| (rc, Vec::new(), None))?;
    let mut f0 = 0i32;
    unsafe { bgr_rollback_frame_count(e, &mut f0) };
    let r = log.raw();
    let mut trace = spec.query(e, &r).map_err(|rc| (rc, Vec::new(), None))?;
    let t = spec.raw(Some(&mut trace));
    let mut out = vec![bgr_checksum::default(); log.points(f0)];
    let (mut n, mut n_s, mut bytes) = (0u32, 0u32, 0usize);
    let rc = unsafe { bgr_replay_trace(e, &r, &t, out.as_mut_ptr(), out.len() as u32, &mut n, &mut n_s, &mut bytes) };
    out.truncate((n as usize).min(out.len()));
    let trace = trace.finish(n_s);
    if rc == BGR_OK { Ok((out, trace)) } else { Err((rc, out, Some(trace))) }
}

impl Batch {
    /// `replay_trace` of `logs[i]` on world `worlds[i]` with `specs[i]` (every spec with the same field list), in one
    /// synchronous call.  `engines[i]` is world i's engine: its query sizes the world's buffers.  Err(status) when the
    /// call was refused before anything executed; otherwise each world's status, checksums and trace, in order.
    pub fn replay_trace(&mut self, worlds: &[u32], engines: &[*mut bgr_engine], f0s: &[i32], logs: &[ReplayLog],
                        specs: &[TraceSpec]) -> Result<Vec<(c_int, Vec<bgr_checksum>, Trace)>, c_int> {
        for l in logs { l.check()?; }
        let reps: Vec<bgr_replay> = logs.iter().map(|l| l.raw()).collect();
        let mut bufs = Vec::with_capacity(worlds.len());
        for i in 0..worlds.len() { bufs.push(specs[i].query(engines[i], &reps[i])?); }
        let trs: Vec<bgr_trace> = bufs.iter_mut().zip(specs.iter()).map(|(b, s)| s.raw(Some(b))).collect();
        let cap: usize = logs.iter().zip(f0s.iter()).map(|(l, &f0)| l.points(f0)).sum();
        let mut out = vec![bgr_checksum::default(); cap];
        let mut n_out = vec![0u32; worlds.len()];
        let mut n_s = vec![0u32; worlds.len()];
        let mut status = vec![0i32; worlds.len()];
        let rc = unsafe {
            bgr_batch_replay_trace(self.raw, worlds.as_ptr(), worlds.len() as u32, reps.as_ptr(), trs.as_ptr(),
                                   out.as_mut_ptr(), cap as u32, n_out.as_mut_ptr(), n_s.as_mut_ptr(), status.as_mut_ptr())
        };
        if rc != BGR_OK && rc != BGR_ERR_NON_FINITE {
            return Err(rc);
        }
        let mut at = 0usize;
        Ok(bufs.into_iter().enumerate().map(|(i, b)| {
            let end = (at + n_out[i] as usize).min(cap);
            let cs = out[at.min(cap)..end].to_vec();
            at += n_out[i] as usize;
            (status[i], cs, b.finish(n_s[i]))
        }).collect())
    }
}
