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

/// Per lattice node (option "lattice"): its best predecessor in the sentence's node list (-1 for BOS) and flags.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct vbt_lattice_link { pub prev: i32, pub flags: u32 }
pub const VBT_NODE_BEST: u32 = 1;

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
    fn vbt_tokenize_batch_spans(t: *mut vbt_tokenizer, utf8: *const c_char, byte_offsets: *const u64, n_sent: u64,
                                bnd_offsets: *const u64, bnd: *const u32, span_offsets: *const u64, spans: *const Span,
                                patterns: *const c_char, pattern_offsets: *const u64, n_patterns: u64,
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
    fn vbt_tokenizer_set_output_format(t: *mut vbt_tokenizer, node: *const c_char, node_len: usize,
                                       unk: *const c_char, unk_len: usize, bos: *const c_char, bos_len: usize,
                                       eos: *const c_char, eos_len: usize) -> i32;
    fn vbt_result_text(r: *const vbt_result, text_offsets: *mut *const u64, text: *mut *const c_char,
                       n_bytes: *mut u64) -> i32;
    fn vbt_tokenizer_set_marginals(t: *mut vbt_tokenizer, theta: f64) -> i32;
    fn vbt_tokenizer_set_sampling(t: *mut vbt_tokenizer, n: u32, theta: f64, seed: u64) -> i32;
    fn vbt_result_samples(r: *const vbt_result, sample_offsets: *mut *const u64, samples: *mut *const vbt_token,
                          n_sample_tokens: *mut u64) -> i32;
    fn vbt_result_marginals(r: *const vbt_result, token_prob: *mut *const f32, path_prob: *mut *const f32) -> i32;
    fn vbt_result_lattice(r: *const vbt_result, node_offsets: *mut *const u64, nodes: *mut *const vbt_token,
                          links: *mut *const vbt_lattice_link, node_prob: *mut *const f32, n_nodes: *mut u64) -> i32;
    fn vbt_result_lattice_margins(r: *const vbt_result, node_margin: *mut *const i64) -> i32;
    fn vbt_result_uncertainty(r: *const vbt_result, entropy: *mut *const f64, log_path_prob: *mut *const f64,
                              boundary_offsets: *mut *const u64, boundary_prob: *mut *const f32) -> i32;
    fn vbt_tokenizer_set_posterior(t: *mut vbt_tokenizer, on: i32, gamma: f64) -> i32;
    fn vbt_result_posterior(r: *const vbt_result, posterior_offsets: *mut *const u64,
                            posterior_tokens: *mut *const vbt_token, posterior_probs: *mut *const f32,
                            posterior_gains: *mut *const f64, n_posterior_tokens: *mut u64) -> i32;
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
                       h: std::cell::OnceCell<*mut vbt_tokenizer>, samples: std::cell::Cell<u32> }
impl Tokenizer {
    pub fn new(dict: Dictionary) -> Self {                                // tokenizer.rs:26
        Self { dict, ignore_space: false, max_grouping_len: 0, devices: vec![], h: Default::default(),
               samples: Default::default() }
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
    /// MeCab-style output formats (node / unk / BOS / EOS format strings, as `tokenize -F`), rendered on the device
    /// in place of `output_mode`: `BatchResult::text`.  `node == None` switches the format off; `unk == None` prints
    /// Unknown tokens with `node`, `bos` / `eos == None` print "" / "EOS\n".
    pub fn output_format(&self, node: Option<&str>, unk: Option<&str>, bos: Option<&str>, eos: Option<&str>)
                         -> Result<()> {
        let p = |x: Option<&str>| x.map_or((std::ptr::null(), 0), |s| (s.as_ptr() as *const c_char, s.len()));
        let (n, u, b, e) = (p(node), p(unk), p(bos), p(eos));
        check(unsafe { vbt_tokenizer_set_output_format(self.handle(), n.0, n.1, u.0, u.1, b.0, b.1, e.0, e.1) })
    }
    /// Batches of at most `n` sentences and 16 KiB tokenised afterwards run in one kernel launch (`k_small_batch`),
    /// with the same tokens and text: the per-sentence `Worker` loop pays one launch per call.  0 = off (the default).
    pub fn small_batch(&self, n: u32) -> Result<()> {
        check(unsafe { vbt_tokenizer_set_option(self.handle(), b"small_batch\0".as_ptr() as *const c_char, n as i64) })
    }
    /// Marginal probabilities at temperature `theta` > 0 (0 = off; see `vbt_tokenizer_set_marginals`): batches
    /// tokenised afterwards carry `BatchResult::marginals`.  Set it before an output format that prints `%pP`.
    pub fn marginals(&self, theta: f64) -> Result<()> {
        check(unsafe { vbt_tokenizer_set_marginals(self.handle(), theta) })
    }
    /// Lattice output (option "lattice"): batches tokenised afterwards carry `BatchResult::lattice`; `text` also
    /// renders the nodes in place of the tokens in the output text (MeCab -a).  Set it before a format that prints `%pb`.
    pub fn lattice(&self, on: bool, text: bool) -> Result<()> {
        let v = if !on { 0 } else if text { 2 } else { 1 };
        check(unsafe { vbt_tokenizer_set_option(self.handle(), b"lattice\0".as_ptr() as *const c_char, v) })
    }
    /// Near-best lattice (option "lattice_margin"): `Some(d)` (0..=2^62) keeps only the nodes of paths whose cost is
    /// within `d` of the best one, plus the best path, and adds `BatchResult::lattice_margins`; `None` keeps every node.
    pub fn lattice_margin(&self, d: Option<i64>) -> Result<()> {
        let opt = b"lattice_margin\0".as_ptr() as *const c_char;
        check(unsafe { vbt_tokenizer_set_option(self.handle(), opt, d.unwrap_or(-1)) })
    }
    /// Segmentation uncertainty (option "uncertainty"; needs `marginals`): batches tokenised afterwards carry
    /// `BatchResult::uncertainty`; `boundary_probs` also carries each character position's boundary probability.
    pub fn uncertainty(&self, on: bool, boundary_probs: bool) -> Result<()> {
        let v = if !on { 0 } else if boundary_probs { 2 } else { 1 };
        check(unsafe { vbt_tokenizer_set_option(self.handle(), b"uncertainty\0".as_ptr() as *const c_char, v) })
    }
    /// Posterior decoding (see `vbt_tokenizer_set_posterior`; needs `marginals`): batches tokenised afterwards carry
    /// `BatchResult::posterior`, each sentence's path of the largest total gain at weight `gamma` >= 0; `None` switches
    /// it off.  `text`: the output text renders the posterior path in place of the best path (option "posterior_text").
    pub fn posterior(&self, gamma: Option<f64>, text: bool) -> Result<()> {
        let opt = b"posterior_text\0".as_ptr() as *const c_char;
        if !text {
            check(unsafe { vbt_tokenizer_set_option(self.handle(), opt, 0) })?;
        }
        check(unsafe { vbt_tokenizer_set_posterior(self.handle(), gamma.is_some() as i32, gamma.unwrap_or(0.0)) })?;
        if text {
            check(unsafe { vbt_tokenizer_set_option(self.handle(), opt, 1) })?;
        }
        Ok(())
    }
    /// Segmentation sampling (see `vbt_tokenizer_set_sampling`): `n` (1..1024, 0 = off) paths per sentence drawn from
    /// P(path) at temperature `theta`, keyed by `seed`; batches tokenised afterwards carry `BatchResult::samples`.
    /// `text`: the output text renders each sentence's `n` samples in place of its best path (option "sample_text").
    pub fn sampling(&self, n: u32, theta: f64, seed: u64, text: bool) -> Result<()> {
        let opt = b"sample_text\0".as_ptr() as *const c_char;
        if !text {
            check(unsafe { vbt_tokenizer_set_option(self.handle(), opt, 0) })?;
        }
        check(unsafe { vbt_tokenizer_set_sampling(self.handle(), n, theta, seed) })?;
        if text {
            check(unsafe { vbt_tokenizer_set_option(self.handle(), opt, 1) })?;
        }
        self.samples.set(n);
        Ok(())
    }
    /// The draws of the next calls' sentence `s` use the sentence index `i + s` (option "sample_base"; `i + n_sent`
    /// at most 2^32), so that a corpus tokenised over several calls draws what one call would.
    pub fn sample_base(&self, i: u64) -> Result<()> {
        check(unsafe { vbt_tokenizer_set_option(self.handle(), b"sample_base\0".as_ptr() as *const c_char, i as i64) })
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
        Ok(BatchResult { r, n_samples: self.samples.get() })
    }
    /// Required tokens (vbt_tokenize_batch_spans): `spans[i]` are line i's spans, byte ranges that must each be one
    /// token, with a feature pattern (csv fields, `*` for any) or `None` for any feature.  No explicit boundaries.
    pub fn tokenize_batch_spans(&self, lines: &[String], spans: &[Vec<(u32, u32, Option<String>)>]) -> Result<BatchResult> {
        let mut utf8 = Vec::new();
        let mut off = vec![0u64];
        for l in lines { utf8.extend_from_slice(l.as_bytes()); off.push(utf8.len() as u64); }
        let (mut span_off, mut recs) = (vec![0u64], Vec::new());
        let (mut pat, mut pat_off, mut index) = (Vec::new(), vec![0u64], std::collections::HashMap::new());
        for i in 0..lines.len() {
            for (a, b, p) in spans.get(i).map(|v| v.as_slice()).unwrap_or(&[]) {
                let k = match p {
                    None => SPAN_ANY,
                    Some(p) => *index.entry(p.clone()).or_insert_with(|| {
                        pat.extend_from_slice(p.as_bytes());
                        pat_off.push(pat.len() as u64);
                        (pat_off.len() - 2) as u32
                    }),
                };
                recs.push(Span { start_byte: *a, end_byte: *b, pattern: k });
            }
            span_off.push(recs.len() as u64);
        }
        let mut r = std::ptr::null_mut();
        check(unsafe { vbt_tokenize_batch_spans(self.handle(), utf8.as_ptr() as *const c_char, off.as_ptr(),
                                                lines.len() as u64, std::ptr::null(), std::ptr::null(), span_off.as_ptr(),
                                                recs.as_ptr(), pat.as_ptr() as *const c_char, pat_off.as_ptr(),
                                                (pat_off.len() - 1) as u64, &mut r) })?;
        Ok(BatchResult { r, n_samples: self.samples.get() })
    }
}

/// vbt_span: a required token of vbt_tokenize_batch_spans.
#[repr(C)]
pub struct Span { pub start_byte: u32, pub end_byte: u32, pub pattern: u32 }
/// VBT_SPAN_ANY: a required token of any feature.
pub const SPAN_ANY: u32 = 0xFFFF_FFFF;

pub struct BatchResult { r: *mut vbt_result, n_samples: u32 }
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
    /// (per-token marginal, per-sentence best-path probability); an error for a batch tokenised without marginals.
    pub fn marginals(&self) -> Result<(&[f32], &[f32])> {
        let (mut tp, mut pp) = (std::ptr::null(), std::ptr::null());
        check(unsafe { vbt_result_marginals(self.r, &mut tp, &mut pp) })?;
        let (mut o, mut t, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut o, &mut t, &mut ns, &mut nt);
            let s = |p: *const f32, n: u64| if n == 0 { &[][..] } else { std::slice::from_raw_parts(p, n as usize) };
            Ok((s(tp, nt), s(pp, ns)))
        }
    }
    /// (node offsets, nodes, links, node marginals or None without marginals); an error for a batch tokenised
    /// without the lattice.
    pub fn lattice(&self) -> Result<(&[u64], &[vbt_token], &[vbt_lattice_link], Option<&[f32]>)> {
        let (mut o, mut nd, mut l, mut p, mut nn) = (std::ptr::null(), std::ptr::null(), std::ptr::null(), std::ptr::null(), 0u64);
        check(unsafe { vbt_result_lattice(self.r, &mut o, &mut nd, &mut l, &mut p, &mut nn) })?;
        let (mut to, mut t, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut to, &mut t, &mut ns, &mut nt);
            let n = nn as usize;
            let nodes: &[vbt_token] = if n == 0 { &[] } else { std::slice::from_raw_parts(nd, n) };
            let links: &[vbt_lattice_link] = if n == 0 { &[] } else { std::slice::from_raw_parts(l, n) };
            let probs = if p.is_null() { None } else if n == 0 { Some(&[][..]) } else { Some(std::slice::from_raw_parts(p, n)) };
            Ok((std::slice::from_raw_parts(o, ns as usize + 1), nodes, links, probs))
        }
    }
    /// The exact cost margin of every node of `lattice()`; an error for a batch tokenised without the lattice or without
    /// `Tokenizer::lattice_margin`.
    pub fn lattice_margins(&self) -> Result<&[i64]> {
        let mut m = std::ptr::null();
        check(unsafe { vbt_result_lattice_margins(self.r, &mut m) })?;
        let n = self.lattice()?.1.len();
        Ok(if n == 0 { &[] } else { unsafe { std::slice::from_raw_parts(m, n) } })
    }
    /// (entropy, log_path_prob, Some((boundary offsets, boundary probabilities)) or None without boundary
    /// probabilities): sentence i's positions 0..n are `probs[offsets[i]..offsets[i + 1]]`; an error for a batch
    /// tokenised without `Tokenizer::uncertainty`.
    pub fn uncertainty(&self) -> Result<(&[f64], &[f64], Option<(&[u64], &[f32])>)> {
        let (mut e, mut l, mut o, mut b) = (std::ptr::null(), std::ptr::null(), std::ptr::null(), std::ptr::null());
        check(unsafe { vbt_result_uncertainty(self.r, &mut e, &mut l, &mut o, &mut b) })?;
        let (mut to, mut t, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut to, &mut t, &mut ns, &mut nt);
            let f = |p: *const f64| if ns == 0 { &[][..] } else { std::slice::from_raw_parts(p, ns as usize) };
            let bnd = if o.is_null() {
                None
            } else {
                let off = std::slice::from_raw_parts(o, ns as usize + 1);
                let n = off[ns as usize] as usize;
                Some((off, if n == 0 { &[][..] } else { std::slice::from_raw_parts(b, n) }))
            };
            Ok((f(e), f(l), bnd))
        }
    }
    /// (posterior offsets, posterior tokens, their marginals, gains): sentence i's posterior-decoded path is
    /// `tokens[offsets[i]..offsets[i + 1]]` and its total gain `gains[i]`; an error for a batch tokenised without
    /// `Tokenizer::posterior`.
    pub fn posterior(&self) -> Result<(&[u64], &[vbt_token], &[f32], &[f64])> {
        let (mut o, mut t, mut p, mut g, mut n) =
            (std::ptr::null(), std::ptr::null(), std::ptr::null(), std::ptr::null(), 0u64);
        check(unsafe { vbt_result_posterior(self.r, &mut o, &mut t, &mut p, &mut g, &mut n) })?;
        let (mut to, mut tt, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut to, &mut tt, &mut ns, &mut nt);
            let n = n as usize;
            Ok((std::slice::from_raw_parts(o, ns as usize + 1),
                if n == 0 { &[][..] } else { std::slice::from_raw_parts(t, n) },
                if n == 0 { &[][..] } else { std::slice::from_raw_parts(p, n) },
                if ns == 0 { &[][..] } else { std::slice::from_raw_parts(g, ns as usize) }))
        }
    }
    /// (sample offsets, sampled tokens): sample j of sentence i is `samples[offsets[i * n + j]..offsets[i * n + j + 1]]`;
    /// an error for a batch tokenised without sampling.
    pub fn samples(&self) -> Result<(&[u64], &[vbt_token])> {
        let (mut o, mut st, mut nst) = (std::ptr::null(), std::ptr::null(), 0u64);
        check(unsafe { vbt_result_samples(self.r, &mut o, &mut st, &mut nst) })?;
        let (mut to, mut t, mut ns, mut nt) = (std::ptr::null(), std::ptr::null(), 0u64, 0u64);
        unsafe {
            vbt_result_view(self.r, &mut to, &mut t, &mut ns, &mut nt);
            let recs: &[vbt_token] = if nst == 0 { &[] } else { std::slice::from_raw_parts(st, nst as usize) };
            Ok((std::slice::from_raw_parts(o, ns as usize * self.n_samples as usize + 1), recs))
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
        let b = BatchResult { r, n_samples: 0 };
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
