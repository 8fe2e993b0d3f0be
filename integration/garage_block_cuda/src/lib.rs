//! Safe wrapper with Garage's conventions (see INTEGRATION.md section 2).  NOT compiled here.
pub mod batch;   // the batching front-end (row f1): EcBatcher::encode / ::reconstruct are what BlockManager calls
pub mod placement;   // row f4: shard-aware nodes_of / write sets / read plan (pure Rust, belongs in garage_rpc)
pub mod sys;

use bytes::Bytes;
use garage_util::data::Hash;
use garage_util::error::Error;

pub struct ErasureCoder { pub(crate) ctx: *mut sys::garage_ec_ctx, pub k: usize, pub m: usize }
unsafe impl Send for ErasureCoder {}   // the C context is internally synchronised
unsafe impl Sync for ErasureCoder {}

pub(crate) fn check(ctx: *const sys::garage_ec_ctx, rc: i32) -> Result<(), Error> {
    if rc == sys::GARAGE_EC_OK { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::garage_ec_strerror(rc)) }.to_string_lossy();
    let det = unsafe { std::ffi::CStr::from_ptr(sys::garage_ec_last_error(ctx)) }.to_string_lossy();
    Err(Error::Message(format!("garage_ec: {} {}", msg, det)))
}

impl ErasureCoder {
    pub fn new(cuda_device: i32, k: usize, m: usize) -> Result<Self, Error> {
        let mut ctx = std::ptr::null_mut();
        let rc = unsafe { sys::garage_ec_create(&mut ctx, cuda_device, k as i32, m as i32, sys::GARAGE_EC_VANDERMONDE) };
        check(std::ptr::null(), rc)?;       // NODEVICE => node refuses to start in EC mode: no CPU fallback
        Ok(Self { ctx, k, m })
    }
    /// HOST-mode calls sleep on an event instead of spinning in the driver: for the batch dispatchers,
    /// which otherwise pin one CPU each while their batch is on the GPU.
    pub fn set_wait_blocking(&self, blocking: bool) {
        unsafe { sys::garage_ec_set_wait_mode(self.ctx, blocking as i32) };
    }
    pub fn shard_len(&self, block_len: usize) -> usize {
        unsafe { sys::garage_ec_shard_len(block_len as u32, self.k as i32) as usize }
    }

    /// Parity shards of a batch of blocks.  Data shard j of block s is the slice
    /// blocks[s][j*L..(j+1)*L] (zero padded), so only parity crosses PCIe back.
    pub fn encode_blocks(&self, blocks: &[Bytes]) -> Result<Vec<Vec<Bytes>>, Error> {
        let max = blocks.iter().map(|b| b.len()).max().unwrap_or(0);
        let stride = unsafe { sys::garage_ec_stride_for(self.shard_len(max) as u32) };
        let ptrs: Vec<*const u8> = blocks.iter().map(|b| b.as_ptr()).collect();
        let lens: Vec<u32> = blocks.iter().map(|b| b.len() as u32).collect();
        let mut parity = vec![0u8; blocks.len() * self.m * stride];
        let rc = unsafe { sys::garage_ec_encode_blocks(self.ctx, ptrs.as_ptr(), lens.as_ptr(), blocks.len(),
                                                       parity.as_mut_ptr(), stride) };
        check(self.ctx, rc)?;
        let parity = Bytes::from(parity);
        Ok(blocks.iter().enumerate().map(|(s, b)| {
            let l = self.shard_len(b.len());
            (0..self.m).map(|i| parity.slice((s * self.m + i) * stride..(s * self.m + i) * stride + l)).collect()
        }).collect())
    }

    /// GET / resync, ONE stripe per call: kept for tools and tests.  The block manager goes through
    /// batch::EcBatcher::reconstruct instead (one FFI call per stripe is the slowest way to drive the GPU).
    /// `shards[i]` is Some(bytes) for every shard that arrived.  Rebuilds the
    /// shards selected by `want` (data shards for GET, this node's index for resync).
    pub fn reconstruct(&self, hash: &Hash, block_len: usize, shards: &mut [Option<Vec<u8>>], want: &[bool])
        -> Result<(), Error>
    {
        let tot = self.k + self.m;
        let l = self.shard_len(block_len);
        let stride = unsafe { sys::garage_ec_stride_for(l as u32) };
        // the C ABI wants 16-byte aligned bases: glibc's allocator gives that for a Vec<u8> of this size;
        // production code takes these buffers from garage_ec_host_alloc (pinned, page aligned)
        let mut buf = vec![0u8; tot * stride];
        let mut present = vec![0u8; tot];
        for (i, s) in shards.iter().enumerate() {
            if let Some(s) = s { buf[i * stride..i * stride + l].copy_from_slice(&s[..l]); present[i] = 1; }
        }
        let want_u8: Vec<u8> = want.iter().map(|w| *w as u8).collect();
        let (mut status, lens) = ([0i32; 1], [l as u32; 1]);
        let rc = unsafe { sys::garage_ec_reconstruct(self.ctx, buf.as_mut_ptr(), present.as_ptr(), want_u8.as_ptr(),
                          status.as_mut_ptr(), lens.as_ptr(), stride, 1, sys::GARAGE_EC_MEM_HOST, std::ptr::null_mut()) };
        if rc == sys::GARAGE_EC_E_UNRECOVERABLE { return Err(Error::MissingBlock(*hash)); }
        check(self.ctx, rc)?;
        for i in 0..tot {
            if present[i] == 0 && want[i] { shards[i] = Some(buf[i * stride..i * stride + l].to_vec()); }
        }
        Ok(())
    }

    /// Ranged read (body_from_blocks_range; UploadPartCopy's source range), step 1: the byte runs
    /// (shard, offset, len) to fetch for bytes [offset, offset+len) of a block, and whether a touched data shard is
    /// absent (the range then needs `read_range`; otherwise it is the runs' bytes in order).  Plain blocks only: an
    /// SSE-C or `Compressed` block is decrypted / decompressed as a whole, so those keep the whole-block GET.
    pub fn range_plan(&self, hash: &Hash, present: &[bool], block_len: usize, offset: usize, len: usize)
        -> Result<(Vec<(u32, u32, u32)>, bool), Error>
    {
        assert!(present.len() == self.k + self.m);
        let pr: Vec<u8> = present.iter().map(|p| *p as u8).collect();
        let cap = (self.k + self.m) * 512;
        let mut runs: Vec<sys::garage_ec_range> = (0..cap).map(|_| sys::garage_ec_range { shard: 0, offset: 0, len: 0 }).collect();
        let (mut n, mut gpu) = (0usize, 0i32);
        let rc = unsafe { sys::garage_ec_range_plan(self.ctx, pr.as_ptr(), block_len as u32, offset as u32, len as u32,
                          runs.as_mut_ptr(), cap, &mut n, &mut gpu) };
        if rc == sys::GARAGE_EC_E_UNRECOVERABLE { return Err(Error::MissingBlock(*hash)); }
        check(self.ctx, rc)?;
        Ok((runs[..n].iter().map(|r| (r.shard, r.offset, r.len)).collect(), gpu != 0))
    }

    /// Ranged read, step 2: `stripe` holds the k+m shards `stride` apart with (at least) the planned runs filled in;
    /// returns bytes [offset, offset+len) of the block, rebuilding absent columns on the GPU.  Only the shard tags
    /// prove these bytes: the block's blake2sum needs the whole block (the deep scrub finds stale shards).
    pub fn read_range(&self, hash: &Hash, stripe: &[u8], stride: usize, present: &[bool], block_len: usize,
                      offset: usize, len: usize) -> Result<Vec<u8>, Error>
    {
        assert!(present.len() == self.k + self.m);
        let pr: Vec<u8> = present.iter().map(|p| *p as u8).collect();
        let mut out = vec![0u8; len];
        let (bl, off, ln, mut st) = ([block_len as u32], [offset as u32], [len as u32], [0i32]);
        let (sp, op) = ([stripe.as_ptr()], [out.as_mut_ptr()]);
        let rc = unsafe { sys::garage_ec_decode_range_stripes(self.ctx, sp.as_ptr(), pr.as_ptr(), bl.as_ptr(),
                          off.as_ptr(), ln.as_ptr(), stride, op.as_ptr(), st.as_mut_ptr(), 1) };
        if rc == sys::GARAGE_EC_E_UNRECOVERABLE { return Err(Error::MissingBlock(*hash)); }
        check(self.ctx, rc)?;
        Ok(out)
    }

    /// Scrub: bit i of the result set = stored parity row i disagrees with the data shards.
    pub fn verify(&self, shards_layout: &[u8], shard_len: &[u32], stride: usize) -> Result<Vec<u32>, Error> {
        let n = shard_len.len();
        let mut mm = vec![0u32; n];
        let rc = unsafe { sys::garage_ec_verify(self.ctx, shards_layout.as_ptr(), mm.as_mut_ptr(), shard_len.as_ptr(),
                          stride, n, sys::GARAGE_EC_MEM_HOST, std::ptr::null_mut()) };
        check(self.ctx, rc)?;
        Ok(mm)
    }

    /// Deep scrub of gathered stripes: per stripe, (the block read from the data shards does not hash to
    /// `hashes[s]`, the parity rows that disagree with the data shards).
    pub fn deep_check(&self, shards_layout: &[u8], block_len: &[u32], hashes: &[[u8; 32]], stride: usize)
                      -> Result<(Vec<bool>, Vec<u32>), Error> {
        let n = block_len.len();
        assert_eq!(hashes.len(), n);
        let mut bad = vec![0u8; n];
        let mut mm = vec![0u32; n];
        let rc = unsafe { sys::garage_ec_deep_check(self.ctx, shards_layout.as_ptr(), block_len.as_ptr(),
                          hashes.as_ptr() as *const u8, bad.as_mut_ptr(), mm.as_mut_ptr(), stride, n,
                          sys::GARAGE_EC_MEM_HOST, std::ptr::null_mut()) };
        check(self.ctx, rc)?;
        Ok((bad.into_iter().map(|b| b != 0).collect(), mm))
    }

    /// put.rs:441-466: seal every block (None: stored as plaintext) into the shard layout; returns the content
    /// addresses.  `keys` and `nonces` hold one entry per block.
    pub fn seal_blocks(&self, blocks: &[&[u8]], keys: Option<(&[[u8; 32]], &[[u8; 8]])>, shards_out: &mut [u8],
                       stride: usize) -> Result<Vec<[u8; 32]>, Error> {
        let n = blocks.len();
        let ptrs: Vec<*const u8> = blocks.iter().map(|b| b.as_ptr()).collect();
        let lens: Vec<u32> = blocks.iter().map(|b| b.len() as u32).collect();
        let (kp, np) = match keys {
            Some((k, nn)) => { assert!(k.len() == n && nn.len() == n); (k.as_ptr() as *const u8, nn.as_ptr() as *const u8) }
            None => (std::ptr::null(), std::ptr::null()),
        };
        let mut hashes = vec![[0u8; 32]; n];
        let rc = unsafe { sys::garage_ec_seal_blocks(self.ctx, ptrs.as_ptr(), lens.as_ptr(), kp, np,
                          shards_out.as_mut_ptr(), stride, hashes.as_mut_ptr() as *mut u8, std::ptr::null_mut(), n) };
        check(self.ctx, rc)?;
        Ok(hashes)
    }

    /// EncryptionParams::get_block for SSE-C: rebuild, check the content hash and every chunk tag, decrypt.  Per
    /// stripe: Ok(plaintext length), or the stripe's status (GARAGE_EC_E_AUTH, GARAGE_EC_E_UNRECOVERABLE, or
    /// GARAGE_EC_E_INVALID for a block that does not hash to its address).
    pub fn open_stripes(&self, stripes: &[*mut u8], present: &[u8], sealed_len: &[u32], hashes: &[[u8; 32]],
                        keys: &[[u8; 32]], outs: &[*mut u8], stride: usize) -> Result<Vec<Result<u32, i32>>, Error> {
        let n = stripes.len();
        assert!(present.len() == n * (self.k + self.m) && sealed_len.len() == n && hashes.len() == n && keys.len() == n
                && outs.len() == n);
        let (mut plen, mut bad, mut status) = (vec![0u32; n], vec![0u8; n], vec![0i32; n]);
        let rc = unsafe { sys::garage_ec_open_stripes(self.ctx, stripes.as_ptr(), present.as_ptr(), sealed_len.as_ptr(),
                          hashes.as_ptr() as *const u8, keys.as_ptr() as *const u8, outs.as_ptr(), plen.as_mut_ptr(),
                          bad.as_mut_ptr(), status.as_mut_ptr(), stride, n) };
        if rc != sys::GARAGE_EC_E_AUTH && rc != sys::GARAGE_EC_E_UNRECOVERABLE { check(self.ctx, rc)?; }
        Ok((0..n).map(|s| if status[s] == sys::GARAGE_EC_E_UNRECOVERABLE { Err(status[s]) }
                          else if bad[s] != 0 { Err(sys::GARAGE_EC_E_INVALID) }
                          else if status[s] != 0 { Err(status[s]) } else { Ok(plen[s]) }).collect())
    }

    /// A byte range of SSE-C blocks (body_from_blocks_range, UploadPartCopy with a source range): check and decrypt
    /// only the chunks plaintext bytes [offset, offset + len) touch.  `stripes` hold at least the runs of
    /// garage_ec_open_range_plan.  Per request: Ok(()) with its len bytes in outs[s], or its status
    /// (GARAGE_EC_E_AUTH, GARAGE_EC_E_UNRECOVERABLE).
    pub fn open_range_stripes(&self, stripes: &[*const u8], present: &[u8], sealed_len: &[u32], keys: &[[u8; 32]],
                              offset: &[u32], len: &[u32], outs: &[*mut u8], stride: usize)
                              -> Result<Vec<Result<(), i32>>, Error> {
        let n = stripes.len();
        assert!(present.len() == n * (self.k + self.m) && sealed_len.len() == n && keys.len() == n && offset.len() == n
                && len.len() == n && outs.len() == n);
        let mut status = vec![0i32; n];
        let rc = unsafe { sys::garage_ec_open_range_stripes(self.ctx, stripes.as_ptr(), present.as_ptr(),
                          sealed_len.as_ptr(), keys.as_ptr() as *const u8, offset.as_ptr(), len.as_ptr(), stride,
                          outs.as_ptr(), status.as_mut_ptr(), n) };
        if rc != sys::GARAGE_EC_E_AUTH && rc != sys::GARAGE_EC_E_UNRECOVERABLE { check(self.ctx, rc)?; }
        Ok(status.iter().map(|&st| if st != 0 { Err(st) } else { Ok(()) }).collect())
    }

    /// Copy with re-encryption (handle_copy_reencrypt, UploadPartCopy) into SSE-C destinations: destination d is the
    /// plaintext pieces[piece_start[d]..piece_start[d + 1]] of the sources, sealed under dst_keys[d] / dst_nonces[d]
    /// into `shards_out` (the shard layout, n_dst * (k+m) * stride bytes).  src_keys = None: plaintext sources.  Per
    /// destination: Ok((content hash, stored length)) or its status (GARAGE_EC_E_AUTH, GARAGE_EC_E_UNRECOVERABLE).
    pub fn reseal_stripes(&self, stripes: &[*mut u8], present: &[u8], src_len: &[u32], src_hashes: &[[u8; 32]],
                          src_keys: Option<&[[u8; 32]]>, pieces: &[sys::garage_ec_piece], piece_start: &[u32],
                          dst_keys: &[[u8; 32]], dst_nonces: &[[u8; 8]], shards_out: &mut [u8], stride: usize)
                          -> Result<Vec<Result<([u8; 32], u32), i32>>, Error> {
        let (n_src, n_dst) = (stripes.len(), dst_keys.len());
        assert!(present.len() == n_src * (self.k + self.m) && src_len.len() == n_src && src_hashes.len() == n_src
                && piece_start.len() == n_dst + 1 && dst_nonces.len() == n_dst
                && shards_out.len() >= n_dst * (self.k + self.m) * stride);
        assert!(piece_start[n_dst] as usize <= pieces.len());
        let kp = match src_keys { Some(k) => { assert!(k.len() == n_src); k.as_ptr() as *const u8 } None => std::ptr::null() };
        let (mut hashes, mut lens) = (vec![[0u8; 32]; n_dst], vec![0u32; n_dst]);
        let (mut bad, mut src_status, mut status) = (vec![0u8; n_src], vec![0i32; n_src], vec![0i32; n_dst]);
        let rc = unsafe { sys::garage_ec_reseal_stripes(self.ctx, stripes.as_ptr(), present.as_ptr(), src_len.as_ptr(),
                          src_hashes.as_ptr() as *const u8, kp, n_src, pieces.as_ptr(), piece_start.as_ptr(),
                          dst_keys.as_ptr() as *const u8, dst_nonces.as_ptr() as *const u8, shards_out.as_mut_ptr(),
                          hashes.as_mut_ptr() as *mut u8, std::ptr::null_mut(), lens.as_mut_ptr(), bad.as_mut_ptr(),
                          src_status.as_mut_ptr(), status.as_mut_ptr(), stride, n_dst) };
        if rc != sys::GARAGE_EC_E_AUTH && rc != sys::GARAGE_EC_E_UNRECOVERABLE { check(self.ctx, rc)?; }
        Ok((0..n_dst).map(|d| if status[d] != 0 { Err(status[d]) } else { Ok((hashes[d], lens[d])) }).collect())
    }

    /// seal_blocks, also returning each block's S3 checksum of kind crc_kind[s] (GARAGE_EC_CRC_*; 0 for
    /// GARAGE_EC_CRC_NONE): read_and_put_blocks' Checksummer for CRC32 / CRC32C, folded by crc_combine.
    pub fn seal_blocks_crc(&self, blocks: &[&[u8]], keys: Option<(&[[u8; 32]], &[[u8; 8]])>, crc_kind: &[u8],
                           shards_out: &mut [u8], stride: usize) -> Result<(Vec<[u8; 32]>, Vec<u32>), Error> {
        let n = blocks.len();
        assert!(crc_kind.len() == n);
        let ptrs: Vec<*const u8> = blocks.iter().map(|b| b.as_ptr()).collect();
        let lens: Vec<u32> = blocks.iter().map(|b| b.len() as u32).collect();
        let (kp, np) = match keys {
            Some((k, nn)) => { assert!(k.len() == n && nn.len() == n); (k.as_ptr() as *const u8, nn.as_ptr() as *const u8) }
            None => (std::ptr::null(), std::ptr::null()),
        };
        let (mut hashes, mut crcs) = (vec![[0u8; 32]; n], vec![0u32; n]);
        let rc = unsafe { sys::garage_ec_seal_blocks_crc(self.ctx, ptrs.as_ptr(), lens.as_ptr(), kp, np,
                          shards_out.as_mut_ptr(), stride, hashes.as_mut_ptr() as *mut u8, std::ptr::null_mut(),
                          crc_kind.as_ptr(), crcs.as_mut_ptr(), n) };
        check(self.ctx, rc)?;
        Ok((hashes, crcs))
    }

    /// reseal_stripes, also returning the S3 checksum of kind crc_kind[d] of each destination's plaintext (copies
    /// into a destination with a CRC32 / CRC32C checksum).
    pub fn reseal_stripes_crc(&self, stripes: &[*mut u8], present: &[u8], src_len: &[u32], src_hashes: &[[u8; 32]],
                              src_keys: Option<&[[u8; 32]]>, pieces: &[sys::garage_ec_piece], piece_start: &[u32],
                              dst_keys: &[[u8; 32]], dst_nonces: &[[u8; 8]], crc_kind: &[u8], shards_out: &mut [u8],
                              stride: usize) -> Result<Vec<Result<([u8; 32], u32, u32), i32>>, Error> {
        let (n_src, n_dst) = (stripes.len(), dst_keys.len());
        assert!(present.len() == n_src * (self.k + self.m) && src_len.len() == n_src && src_hashes.len() == n_src
                && piece_start.len() == n_dst + 1 && dst_nonces.len() == n_dst && crc_kind.len() == n_dst
                && shards_out.len() >= n_dst * (self.k + self.m) * stride);
        assert!(piece_start[n_dst] as usize <= pieces.len());
        let kp = match src_keys { Some(k) => { assert!(k.len() == n_src); k.as_ptr() as *const u8 } None => std::ptr::null() };
        let (mut hashes, mut lens, mut crcs) = (vec![[0u8; 32]; n_dst], vec![0u32; n_dst], vec![0u32; n_dst]);
        let (mut bad, mut src_status, mut status) = (vec![0u8; n_src], vec![0i32; n_src], vec![0i32; n_dst]);
        let rc = unsafe { sys::garage_ec_reseal_stripes_crc(self.ctx, stripes.as_ptr(), present.as_ptr(),
                          src_len.as_ptr(), src_hashes.as_ptr() as *const u8, kp, n_src, pieces.as_ptr(),
                          piece_start.as_ptr(), dst_keys.as_ptr() as *const u8, dst_nonces.as_ptr() as *const u8,
                          shards_out.as_mut_ptr(), hashes.as_mut_ptr() as *mut u8, std::ptr::null_mut(),
                          lens.as_mut_ptr(), bad.as_mut_ptr(), src_status.as_mut_ptr(), status.as_mut_ptr(),
                          crc_kind.as_ptr(), crcs.as_mut_ptr(), stride, n_dst) };
        if rc != sys::GARAGE_EC_E_AUTH && rc != sys::GARAGE_EC_E_UNRECOVERABLE { check(self.ctx, rc)?; }
        Ok((0..n_dst).map(|d| if status[d] != 0 { Err(status[d]) } else { Ok((hashes[d], lens[d], crcs[d])) }).collect())
    }

    /// CRC(A || B) from CRC(A), CRC(B) and |B| (host only): folds block checksums, in order, into a part's.
    pub fn crc_combine(kind: u8, crc_a: u32, crc_b: u32, len_b: u64) -> Result<u32, Error> {
        let mut out = 0u32;
        let rc = unsafe { sys::garage_ec_crc_combine(kind as i32, crc_a, crc_b, len_b, &mut out) };
        if rc != sys::GARAGE_EC_OK { return Err(Error::Message(format!("garage_ec_crc_combine: {}", rc))); }
        Ok(out)
    }
}
impl Drop for ErasureCoder { fn drop(&mut self) { unsafe { sys::garage_ec_destroy(self.ctx) } } }

/// `cuda_devices = [...]` (DESIGN.md section 5.13): one coder per listed GPU with its NUMA node, and the block
/// manager's routing rule.  The coders whose GPU is on the calling thread's node are the candidates (all of them if
/// none is); the one with the fewest calls in flight wins, ties round robin.  A batch is handed to one coder only, so
/// no batch spans GPUs; the batcher and pinned pools of each coder live next to it (one batch::EcBatcher per coder).
pub struct DeviceCoders {
    coders: Vec<(ErasureCoder, i32)>,
    in_flight: Vec<std::sync::atomic::AtomicUsize>,
    rr: std::sync::atomic::AtomicUsize,
}

extern "C" {
    fn getcpu(cpu: *mut u32, node: *mut u32) -> std::os::raw::c_int;  // glibc >= 2.29
}

pub const MAX_DEVICES: usize = 16;

/// A routed call: the coder it runs on, released (one call less in flight) when dropped.
pub struct Routed<'a> { owner: &'a DeviceCoders, i: usize }
impl<'a> std::ops::Deref for Routed<'a> {
    type Target = ErasureCoder;
    fn deref(&self) -> &ErasureCoder { &self.owner.coders[self.i].0 }
}
impl<'a> Drop for Routed<'a> {
    fn drop(&mut self) { self.owner.in_flight[self.i].fetch_sub(1, std::sync::atomic::Ordering::Relaxed); }
}

impl DeviceCoders {
    /// One coder per entry of `devices` (a device may repeat).  Refused before any context exists: an empty list, more
    /// than MAX_DEVICES entries, or a device outside 0..garage_ec_device_count().  A coder that cannot be created fails
    /// the whole call (the ones already created are dropped): a node never runs on fewer GPUs than configured.
    pub fn new(devices: &[i32], k: usize, m: usize) -> Result<Self, Error> {
        let n = unsafe { sys::garage_ec_device_count() };
        if devices.is_empty() || devices.len() > MAX_DEVICES || devices.iter().any(|&d| d < 0 || d >= n) {
            return Err(Error::Message(format!("cuda_devices {:?}: {} device(s) visible", devices, n)));
        }
        let mut coders = Vec::with_capacity(devices.len());
        for &d in devices {
            let ec = ErasureCoder::new(d, k, m)?;
            let mut node = -1;
            unsafe { sys::garage_ec_numa_info(ec.ctx, &mut node, std::ptr::null_mut()) };
            coders.push((ec, node));
        }
        let in_flight = devices.iter().map(|_| std::sync::atomic::AtomicUsize::new(0)).collect();
        Ok(Self { coders, in_flight, rr: std::sync::atomic::AtomicUsize::new(0) })
    }

    /// The coder a call from this thread runs on (see the type's documentation).
    pub fn route(&self) -> Routed<'_> {
        use std::sync::atomic::Ordering::Relaxed;
        let (mut cpu, mut node) = (0u32, 0u32);
        let here = if unsafe { getcpu(&mut cpu, &mut node) } == 0 { node as i32 } else { -1 };
        let local = here >= 0 && self.coders.iter().any(|c| c.1 == here);
        let n = self.coders.len();
        let start = self.rr.fetch_add(1, Relaxed) % n;
        let mut best: Option<usize> = None;
        for j in 0..n {
            let i = (start + j) % n;
            if local && self.coders[i].1 != here { continue; }
            if best.map_or(true, |b| self.in_flight[i].load(Relaxed) < self.in_flight[b].load(Relaxed)) { best = Some(i); }
        }
        let i = best.unwrap();
        self.in_flight[i].fetch_add(1, Relaxed);
        Routed { owner: self, i }
    }

    /// Pin the calling thread (a resync worker, an API worker) to the CPUs of coder w mod n's node, so that a pool of
    /// workers spreads over the GPUs' sockets.
    pub fn bind_worker(&self, w: usize) {
        unsafe { sys::garage_ec_bind_thread(self.coders[w % self.coders.len()].0.ctx) };
    }
}
