//! Same public surface as the `vibrato` crate for the tokenisation path, backed by libvibrato_b200.so.
use std::ffi::CStr;
use std::io::Read;
use std::os::raw::{c_char, c_void};

#[repr(C)] pub struct vbt_dict { _p: [u8; 0] }
#[repr(C)] pub struct vbt_tokenizer { _p: [u8; 0] }
#[repr(C)] pub struct vbt_result { _p: [u8; 0] }

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct vbt_token {
    pub start_char: u32, pub end_char: u32, pub start_byte: u32, pub end_byte: u32,
    pub word_idx: u32, pub total_cost: i32,
}

#[link(name = "vibrato_b200")]
extern "C" {
    fn vbt_last_error() -> *const c_char;
    fn vbt_dict_from_bytes(dic: *const u8, n: usize, out: *mut *mut vbt_dict) -> i32;
    fn vbt_dict_set_user_lexicon_csv(d: *mut vbt_dict, csv: *const c_char, n: usize) -> i32;
    fn vbt_dict_free(d: *mut vbt_dict);
    fn vbt_dict_feature(d: *const vbt_dict, word_idx: u32, p: *mut *const c_char, len: *mut usize) -> i32;
    fn vbt_dict_word_param(d: *const vbt_dict, word_idx: u32, l: *mut u16, r: *mut u16, c: *mut i16) -> i32;
    fn vbt_dict_cate_id(d: *const vbt_dict, name: *const c_char, len: usize, id: *mut i32) -> i32;
    fn vbt_tokenizer_new(d: *const vbt_dict, ignore_space: i32, max_grouping_len: u64, device: i32,
                         out: *mut *mut vbt_tokenizer) -> i32;
    fn vbt_tokenizer_new_multi(d: *const vbt_dict, ignore_space: i32, max_grouping_len: u64, devices: *const i32,
                               n_devices: i32, out: *mut *mut vbt_tokenizer) -> i32;
    fn vbt_tokenizer_free(t: *mut vbt_tokenizer);
    fn vbt_tokenize_batch(t: *mut vbt_tokenizer, utf8: *const c_char, byte_offsets: *const u64, n_sent: u64,
                          out: *mut *mut vbt_result) -> i32;
    fn vbt_result_view(r: *const vbt_result, tok_offsets: *mut *const u64, toks: *mut *const vbt_token,
                       n_sent: *mut u64, n_tokens: *mut u64) -> i32;
    fn vbt_result_free(r: *mut vbt_result);
    fn vbt_dict_from_mecab(lex: *const c_char, lex_len: usize, matrix: *const c_char, matrix_len: usize,
                           chr: *const c_char, chr_len: usize, unk: *const c_char, unk_len: usize,
                           out: *mut *mut vbt_dict) -> i32;
    fn vbt_dict_from_bigram(lex: *const c_char, lex_len: usize, right: *const c_char, right_len: usize,
                            left: *const c_char, left_len: usize, cost: *const c_char, cost_len: usize,
                            chr: *const c_char, chr_len: usize, unk: *const c_char, unk_len: usize,
                            dual_connector: i32, out: *mut *mut vbt_dict) -> i32;
    fn vbt_mecab_generate_bigram_info(feature_def: *const c_char, feature_len: usize, right_id_def: *const c_char,
                                      right_id_len: usize, left_id_def: *const c_char, left_id_len: usize,
                                      model_def: *const c_char, model_len: usize, cost_factor: f64,
                                      bigram_right: *mut *mut u8, right_n: *mut usize, bigram_left: *mut *mut u8,
                                      left_n: *mut usize, bigram_cost: *mut *mut u8, cost_n: *mut usize) -> i32;
    fn vbt_bytes_free(p: *mut u8);
    fn vbt_dict_map_connection_ids(d: *mut vbt_dict, lmap: *const u16, n_lmap: usize, rmap: *const u16,
                                   n_rmap: usize) -> i32;
    fn vbt_tokenizer_set_option(t: *mut vbt_tokenizer, name: *const c_char, value: i64) -> i32;
    fn vbt_result_text(r: *const vbt_result, text_offsets: *mut *const u64, text: *mut *const c_char,
                       n_bytes: *mut u64) -> i32;
    fn vbt_evaluate(d: *const vbt_dict, t: *mut vbt_tokenizer, corpus: *const c_char, len: usize,
                    feature_indices: *const u64, n_indices: usize, num_ref: *mut u64, num_sys: *mut u64,
                    num_cor: *mut u64) -> i32;
}

#[derive(Debug)]
pub struct VibratoError { pub code: i32, pub msg: String }   // codes 1..9 == errors.rs:11-42 variants
pub type Result<T> = std::result::Result<T, VibratoError>;
fn check(rc: i32) -> Result<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { CStr::from_ptr(vbt_last_error()) }.to_string_lossy().into_owned();
    Err(VibratoError { code: rc, msg })
}

#[derive(Clone, Copy, Debug, PartialEq, Eq)]
#[repr(u8)]
pub enum LexType { System = 0, User = 1, Unknown = 2 }                  // dictionary.rs:30-40
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub struct WordIdx { pub lex_type: LexType, pub word_id: u32 }          // word_idx.rs:5-11

pub struct Dictionary { h: *mut vbt_dict }
unsafe impl Send for Dictionary {}
unsafe impl Sync for Dictionary {}
impl Drop for Dictionary { fn drop(&mut self) { unsafe { vbt_dict_free(self.h) } } }

impl Dictionary {
    /// dictionary.rs:173 — `rdr` yields the zstd-decoded stream (tokenize/src/main.rs:59-60).
    pub fn read<R: Read>(mut rdr: R) -> Result<Self> {
        let mut buf = vec![];
        rdr.read_to_end(&mut buf).map_err(|e| VibratoError { code: 7, msg: e.to_string() })?;
        let mut h = std::ptr::null_mut();
        check(unsafe { vbt_dict_from_bytes(buf.as_ptr(), buf.len(), &mut h) })?;
        Ok(Self { h })
    }
    /// dictionary.rs:209 — consumes and returns self, like the reference.
    pub fn reset_user_lexicon_from_reader<R: Read>(self, rdr: Option<R>) -> Result<Self> {
        match rdr {
            Some(mut r) => {
                let mut buf = vec![];
                r.read_to_end(&mut buf).map_err(|e| VibratoError { code: 7, msg: e.to_string() })?;
                check(unsafe { vbt_dict_set_user_lexicon_csv(self.h, buf.as_ptr() as *const c_char, buf.len()) })?;
            }
            None => check(unsafe { vbt_dict_set_user_lexicon_csv(self.h, std::ptr::null(), 0) })?,
        }
        Ok(self)
    }
    /// dictionary.rs:245-259: `lmap` / `rmap` list the OLD ids (without 0) in their NEW order.
    pub fn map_connection_ids_from_iter<L, R>(self, lmap: L, rmap: R) -> Result<Self>
    where L: IntoIterator<Item = u16>, R: IntoIterator<Item = u16> {
        let (l, r): (Vec<u16>, Vec<u16>) = (lmap.into_iter().collect(), rmap.into_iter().collect());
        check(unsafe { vbt_dict_map_connection_ids(self.h, l.as_ptr(), l.len(), r.as_ptr(), r.len()) })?;
        Ok(self)
    }
    /// dictionary.rs:108
    pub fn word_feature(&self, w: WordIdx) -> &str {
        let (mut p, mut n) = (std::ptr::null(), 0usize);
        unsafe {
            vbt_dict_feature(self.h, (w.lex_type as u32) << 30 | w.word_id, &mut p, &mut n);
            std::str::from_utf8_unchecked(std::slice::from_raw_parts(p as *const u8, n))
        }
    }
}

fn slurp<R: Read>(mut r: R) -> Result<Vec<u8>> {
    let mut buf = vec![];
    r.read_to_end(&mut buf).map_err(|e| VibratoError { code: 7, msg: e.to_string() })?;
    Ok(buf)
}

/// dictionary/builder.rs:40-148
pub struct SystemDictionaryBuilder;
impl SystemDictionaryBuilder {
    /// builder.rs:64-89
    pub fn from_readers<S: Read, C: Read, P: Read, U: Read>(lex: S, matrix: C, chr: P, unk: U) -> Result<Dictionary> {
        let (a, b, c, d) = (slurp(lex)?, slurp(matrix)?, slurp(chr)?, slurp(unk)?);
        let mut h = std::ptr::null_mut();
        check(unsafe { vbt_dict_from_mecab(a.as_ptr() as _, a.len(), b.as_ptr() as _, b.len(), c.as_ptr() as _, c.len(),
                                           d.as_ptr() as _, d.len(), &mut h) })?;
        Ok(Dictionary { h })
    }
    /// builder.rs:111-148 (RawConnector, or DualConnector when `dual_connector`)
    pub fn from_readers_with_bigram_info<S: Read, R: Read, L: Read, C: Read, P: Read, U: Read>(
        lex: S, right: R, left: L, cost: C, chr: P, unk: U, dual_connector: bool) -> Result<Dictionary> {
        let (a, r, l, k, c, d) = (slurp(lex)?, slurp(right)?, slurp(left)?, slurp(cost)?, slurp(chr)?, slurp(unk)?);
        let mut h = std::ptr::null_mut();
        check(unsafe { vbt_dict_from_bigram(a.as_ptr() as _, a.len(), r.as_ptr() as _, r.len(), l.as_ptr() as _, l.len(),
                                            k.as_ptr() as _, k.len(), c.as_ptr() as _, c.len(), d.as_ptr() as _, d.len(),
                                            dual_connector as i32, &mut h) })?;
        Ok(Dictionary { h })
    }
}

/// mecab.rs: utilities for MeCab models.
pub mod mecab {
    use super::*;
    use std::io::Write;

    /// mecab.rs:31-181: writes the bigram.right / bigram.left / bigram.cost files of a compact dictionary made from a
    /// trained MeCab model.  Same argument order as the reference: right-id.def feeds `bigram_right_wtr`.
    #[allow(clippy::too_many_arguments)]
    pub fn generate_bigram_info(feature_def_rdr: impl Read, right_id_def_rdr: impl Read, left_id_def_rdr: impl Read,
                                model_def_rdr: impl Read, cost_factor: f64, mut bigram_right_wtr: impl Write,
                                mut bigram_left_wtr: impl Write, mut bigram_cost_wtr: impl Write) -> Result<()> {
        let (f, r, l, m) = (slurp(feature_def_rdr)?, slurp(right_id_def_rdr)?, slurp(left_id_def_rdr)?,
                            slurp(model_def_rdr)?);
        let mut p = [std::ptr::null_mut(); 3];
        let mut n = [0usize; 3];
        let [p0, p1, p2] = &mut p;
        let [n0, n1, n2] = &mut n;
        check(unsafe { vbt_mecab_generate_bigram_info(f.as_ptr() as _, f.len(), r.as_ptr() as _, r.len(),
                                                      l.as_ptr() as _, l.len(), m.as_ptr() as _, m.len(), cost_factor,
                                                      p0, n0, p1, n1, p2, n2) })?;
        let mut res = Ok(());
        let writers: [&mut dyn Write; 3] = [&mut bigram_right_wtr, &mut bigram_left_wtr, &mut bigram_cost_wtr];
        for (i, w) in writers.into_iter().enumerate() {
            let bytes = unsafe { std::slice::from_raw_parts(p[i], n[i]) };
            if res.is_ok() {
                res = w.write_all(bytes).map_err(|e| VibratoError { code: 7, msg: e.to_string() });
            }
            unsafe { vbt_bytes_free(p[i]) };
        }
        res
    }
}

/// tokenize/src/main.rs:12-29
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum OutputMode { Mecab = 1, Wakati = 2, Detail = 3 }

pub struct Tokenizer { dict: Dictionary, ignore_space: bool, max_grouping_len: usize, devices: Vec<i32>,
                       h: std::cell::OnceCell<*mut vbt_tokenizer> }
impl Tokenizer {
    pub fn new(dict: Dictionary) -> Self {                                // tokenizer.rs:26
        Self { dict, ignore_space: false, max_grouping_len: 0, devices: vec![], h: Default::default() }
    }
    /// Not in the reference (a vibrato Worker is one CPU thread): spread every batch over these GPUs of the node.
    /// The dictionary image is uploaded once and broadcast over NVLink; `tokenize_batch` still returns one result
    /// in input order.
    pub fn devices(mut self, devices: &[i32]) -> Self {
        self.devices = devices.to_vec();
        self
    }
    pub fn ignore_space(mut self, yes: bool) -> Result<Self> {             // tokenizer.rs:42-55
        if yes {
            let mut id = -1i32;
            check(unsafe { vbt_dict_cate_id(self.dict.h, b"SPACE".as_ptr() as *const c_char, 5, &mut id) })?;
            if id < 0 {
                return Err(VibratoError { code: 1,
                    msg: "SPACE is not defined in the input dictionary (i.e., char.def).".into() });
            }
        }
        self.ignore_space = yes;
        Ok(self)
    }
    pub fn max_grouping_len(mut self, n: usize) -> Self { self.max_grouping_len = n; self }   // tokenizer.rs:67
    pub fn dictionary(&self) -> &Dictionary { &self.dict }
    pub fn new_worker(&self) -> Worker<'_> { Worker { t: self, sent: String::new(), toks: vec![] } }
    fn handle(&self) -> *mut vbt_tokenizer {
        *self.h.get_or_init(|| {
            let mut h = std::ptr::null_mut();
            let rc = if self.devices.is_empty() {
                unsafe { vbt_tokenizer_new(self.dict.h, self.ignore_space as i32, self.max_grouping_len as u64, 0, &mut h) }
            } else {
                unsafe { vbt_tokenizer_new_multi(self.dict.h, self.ignore_space as i32, self.max_grouping_len as u64,
                                                 self.devices.as_ptr(), self.devices.len() as i32, &mut h) }
            };
            check(rc).expect("vibrato_b200: cannot create the device tokenizer (no CPU fallback)");
            h
        })
    }
    /// Batches tokenised afterwards also carry the text `tokenize` prints (tokenize/src/main.rs:83-127), built on the
    /// device: `BatchResult::text`.
    pub fn output_mode(&self, mode: Option<OutputMode>) -> Result<()> {
        check(unsafe { vbt_tokenizer_set_option(self.handle(), b"output_mode\0".as_ptr() as *const c_char,
                                                mode.map_or(0, |m| m as i64)) })
    }
    /// The loop of the `evaluate` tool (evaluate/src/main.rs:61-138): (num_ref, num_sys, num_cor).
    pub fn evaluate(&self, corpus: &str, feature_indices: &[usize]) -> Result<(u64, u64, u64)> {
        let idx: Vec<u64> = feature_indices.iter().map(|&i| i as u64).collect();
        let (mut a, mut b, mut c) = (0u64, 0u64, 0u64);
        check(unsafe { vbt_evaluate(self.dict.h, self.handle(), corpus.as_ptr() as *const c_char, corpus.len(),
                                    idx.as_ptr(), idx.len(), &mut a, &mut b, &mut c) })?;
        Ok((a, b, c))
    }
    /// The batched call `benchmark` should use: all lines at once.
    pub fn tokenize_batch(&self, lines: &[String]) -> Result<BatchResult> {
        let mut utf8 = Vec::new();
        let mut off = vec![0u64];
        for l in lines { utf8.extend_from_slice(l.as_bytes()); off.push(utf8.len() as u64); }
        let mut r = std::ptr::null_mut();
        check(unsafe { vbt_tokenize_batch(self.handle(), utf8.as_ptr() as *const c_char, off.as_ptr(),
                                          lines.len() as u64, &mut r) })?;
        Ok(BatchResult { r })
    }
}

pub struct BatchResult { r: *mut vbt_result }
impl Drop for BatchResult { fn drop(&mut self) { unsafe { vbt_result_free(self.r) } } }
impl BatchResult {
    /// What `tokenize` writes for the batch; sentence i is `text[offsets[i]..offsets[i + 1]]`.
    pub fn text(&self) -> Result<(&[u64], &str)> {
        let (mut o, mut t, mut n) = (std::ptr::null(), std::ptr::null(), 0u64);
        check(unsafe { vbt_result_text(self.r, &mut o, &mut t, &mut n) })?;
        let (mut to, mut tt, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut to, &mut tt, &mut ns, &mut nt);
            Ok((std::slice::from_raw_parts(o, ns as usize + 1),
                std::str::from_utf8_unchecked(std::slice::from_raw_parts(t as *const u8, n as usize))))
        }
    }
    pub fn view(&self) -> (&[u64], &[vbt_token]) {
        let (mut o, mut t, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut o, &mut t, &mut ns, &mut nt);
            (std::slice::from_raw_parts(o, ns as usize + 1), std::slice::from_raw_parts(t, nt as usize))
        }
    }
}

pub struct Worker<'t> { t: &'t Tokenizer, sent: String, toks: Vec<vbt_token> }
impl<'t> Worker<'t> {
    pub fn reset_sentence<S: AsRef<str>>(&mut self, s: S) {                 // worker.rs:34
        self.sent.clear(); self.sent.push_str(s.as_ref()); self.toks.clear();
    }
    pub fn tokenize(&mut self) {                                            // worker.rs:49 (infallible)
        if self.sent.is_empty() { return; }
        let off = [0u64, self.sent.len() as u64];
        let mut r = std::ptr::null_mut();
        let rc = unsafe { vbt_tokenize_batch(self.t.handle(), self.sent.as_ptr() as *const c_char,
                                             off.as_ptr(), 1, &mut r) };
        check(rc).expect("vibrato_b200 device error");
        let b = BatchResult { r };
        self.toks = b.view().1.to_vec();
    }
    pub fn num_tokens(&self) -> usize { self.toks.len() }                   // worker.rs:59
    pub fn token<'w>(&'w self, i: usize) -> Token<'w, 't> { Token { w: self, i } }   // already in sentence order
    pub fn token_iter<'w>(&'w self) -> impl Iterator<Item = Token<'w, 't>> + 'w {
        (0..self.toks.len()).map(move |i| Token { w: self, i })
    }
}

pub struct Token<'w, 't> { w: &'w Worker<'t>, i: usize }
impl<'w, 't> Token<'w, 't> {
    fn r(&self) -> &vbt_token { &self.w.toks[self.i] }
    pub fn range_char(&self) -> std::ops::Range<usize> { self.r().start_char as usize..self.r().end_char as usize }
    pub fn range_byte(&self) -> std::ops::Range<usize> { self.r().start_byte as usize..self.r().end_byte as usize }
    pub fn surface(&self) -> &'w str { &self.w.sent[self.range_byte()] }
    pub fn word_idx(&self) -> WordIdx {
        let w = self.r().word_idx;
        let lex_type = match w >> 30 { 0 => LexType::System, 1 => LexType::User, _ => LexType::Unknown };
        WordIdx { lex_type, word_id: w & 0x3FFF_FFFF }
    }
    pub fn lex_type(&self) -> LexType { self.word_idx().lex_type }
    pub fn feature(&self) -> &'t str { self.w.t.dict.word_feature(self.word_idx()) }
    fn param(&self) -> (u16, u16, i16) {
        let (mut l, mut r, mut c) = (0u16, 0u16, 0i16);
        unsafe { vbt_dict_word_param(self.w.t.dict.h, self.r().word_idx, &mut l, &mut r, &mut c) };
        (l, r, c)
    }
    pub fn left_id(&self) -> u16 { self.param().0 }
    pub fn right_id(&self) -> u16 { self.param().1 }
    pub fn word_cost(&self) -> i16 { self.param().2 }
    pub fn total_cost(&self) -> i32 { self.r().total_cost }
}
