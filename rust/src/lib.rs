//! Drop-in replacement for whisper-burn's hot-path modules over `include/whisper_b200.h` (libwhisper_b200.so).
//!
//! Meant to be compiled INSIDE the whisper-burn crate in place of `src/audio.rs`, `src/model/*`, `src/beam.rs` and
//! `src/transcribe.rs` (reference `src/lib.rs:1-6` exports `audio, helper, model, token, transcribe, beam`); `src/token.rs`
//! (Gpt2Tokenizer, Language, SpecialToken) and the binaries stay the reference's own code -- `mod token` below is that file,
//! unchanged.  What changes for a caller of the reference:
//!   * `Whisper<B>` is no longer generic over a burn `Backend`; it owns a `wb_model*` and a cached decoding session.
//!   * tensors crossing the API are plain host `Vec<f32>` + shape (the reference's `Tensor<B, D>` are device handles of the
//!     backend this crate replaces).
//! Contract violations that `assert!`/panic in the reference (audio.rs:292, mod.rs:134-139, 231-241) come back as
//! WB_ERR_INVALID_ARG and are turned into `panic!` here; CUDA/OOM failures become `Err`.
//! NOT compiled in this repository's build container (no cargo/rustc there); kept in lock-step with the header by review.
#![allow(non_camel_case_types)]

use std::ffi::{c_char, c_int, c_void, CStr, CString};
use std::sync::Mutex;

pub mod token;   // the reference's own src/token.rs, unchanged

pub mod ffi {
    use super::*;
    #[repr(C)]
    #[derive(Clone, Copy, Debug)]
    pub struct wb_dims {
        pub n_mels: i32, pub n_audio_ctx: i32, pub n_audio_state: i32, pub n_audio_head: i32, pub n_audio_layer: i32,
        pub n_vocab: i32, pub n_text_ctx: i32, pub n_text_state: i32, pub n_text_head: i32, pub n_text_layer: i32,
    }
    pub const WB_SEARCH_BEAM: c_int = 0;          // search rules of a session (wb_session_set_search)
    pub const WB_SEARCH_GREEDY_LOOP: c_int = 1;
    #[repr(C)]
    #[derive(Clone, Copy, Debug)]
    pub struct wb_special_ids { pub sot: i64, pub lang: i64, pub transcribe: i64, pub notimestamps: i64, pub eot: i64 }

    extern "C" {
        pub fn wb_last_error() -> *const c_char;
        pub fn wb_max_waveform_samples(n_frame_max: i64) -> i64;
        pub fn wb_prep_audio(device: c_int, wave: *const f32, n_batch: i64, n_samples: i64, mel_out: *mut f32, n_frames_out: *mut i64) -> c_int;
        pub fn wb_model_create(dims: *const wb_dims, device: c_int, out: *mut *mut c_void) -> c_int;
        pub fn wb_model_set_tensor(m: *mut c_void, path: *const c_char, data: *const f32, shape: *const i64, ndim: c_int) -> c_int;
        pub fn wb_npy_tree_probe(dir: *const c_char, dims_out: *mut wb_dims) -> c_int;
        pub fn wb_model_load_npy_tree(dir: *const c_char, device: c_int, ln_eps_outside: c_int, out: *mut *mut c_void) -> c_int;
        pub fn wb_load_wav(path: *const c_char, strict_16k_mono: c_int, out: *mut f32, capacity: i64, n_samples_out: *mut i64, sample_rate_out: *mut i64, channels_out: *mut c_int) -> c_int;
        pub fn wb_model_set_layernorm_eps_mode(m: *mut c_void, outside: c_int) -> c_int;
        pub fn wb_model_finalize(m: *mut c_void) -> c_int;
        pub fn wb_model_destroy(m: *mut c_void);
        pub fn wb_forward_encoder(m: *mut c_void, mel: *const f32, n_batch: i64, n_mels: i64, n_ctx: i64, out: *mut f32) -> c_int;
        pub fn wb_forward_decoder(m: *mut c_void, tokens: *const i64, n_batch: i64, seq_len: i64, enc: *const f32, n_enc_ctx: i64, logits_out: *mut f32) -> c_int;
        pub fn wb_session_create(m: *mut c_void, max_windows: i64, max_beams: i64, max_text_len: i64, kv_dtype: c_int, out: *mut *mut c_void) -> c_int;
        pub fn wb_session_destroy(s: *mut c_void);
        pub fn wb_session_set_search(s: *mut c_void, rule: c_int) -> c_int;
        pub fn wb_session_encode_mels(s: *mut c_void, mel: *const f32, n_windows: i64, n_mels: i64, n_ctx: i64) -> c_int;
        pub fn wb_session_begin(s: *mut c_void, prompt: *const i64, prompt_len: i64) -> c_int;
        pub fn wb_session_step(s: *mut c_void, n_rows: i64, window_of_row: *const i32, parent_row: *const i32, token: *const i64, apply_special_mask: c_int,
                               is_special: *const u8, k: c_int, topk_ids_out: *mut i64, topk_logprob_out: *mut f32) -> c_int;
        pub fn wb_first_repetition_end(tokens: *const i64, n: i64, period: i64) -> i64;
        pub fn wb_repetition_period(tokens: *const i64, n: i64, min_repetitions: i64) -> i64;
        pub fn wb_find_repeated_tokens_index(tokens: *const i64, n: i64, window_size: i64, min_repeat_count: i64, first_repeat_index: *mut i64, end: *mut i64) -> c_int;
        pub fn wb_waveform_to_tokens(s: *mut c_void, waveform: *const f32, n_samples: i64, sample_rate: i64, beam_size: c_int, max_depth: c_int,
                                     ids: *const wb_special_ids, is_special: *const u8, tokens_out: *mut i64, capacity: i64, n_tokens_out: *mut i64) -> c_int;
        pub fn wb_session_last_logprobs(s: *mut c_void, index: i64, out: *mut f32, capacity: i64, n_out: *mut i64) -> c_int;
        pub fn wb_session_encode_waveforms(s: *mut c_void, waves: *const *const f32, lens: *const i64, n_windows: i64) -> c_int;
        pub fn wb_session_score_tokens(s: *mut c_void, n_seqs: i64, window_of_seq: *const i32, tokens: *const i64, lens: *const i64,
                                       apply_special_mask: c_int, is_special: *const u8, lp_out: *mut f32, argmax_out: *mut i64) -> c_int;
        pub fn wb_session_set_prev_prompt(s: *mut c_void, startofprev: i64) -> c_int;
        pub fn wb_transcribe_windows_prev(s: *mut c_void, waves: *const *const f32, lens: *const i64, n_windows: i64, prev_tokens: *const i64,
                                          prev_lens: *const i64, startofprev: i64, beam_size: c_int, max_depth: c_int, ids: *const wb_special_ids,
                                          is_special: *const u8, tokens_out: *mut i64, capacity: i64, lens_out: *mut i64) -> c_int;
        pub fn wb_session_last_nbest(s: *mut c_void, index: i64, max_hyps: i64, capacity: i64, ids_out: *mut i64, lp_out: *mut f32,
                                     lens_out: *mut i64, scores_out: *mut f64, finished_out: *mut i32, n_hyps_out: *mut i64) -> c_int;
        pub fn wb_resampled_length(n_frames: i64, sample_rate: i64) -> i64;
        pub fn wb_resample(device: c_int, input: *const f32, n_frames: i64, channels: i64, sample_rate: i64, out: *mut f32, capacity: i64,
                           n_out: *mut i64) -> c_int;
        pub fn wb_waveforms_to_tokens_resampled(s: *mut c_void, waveforms: *const *const f32, n_frames: *const i64, channels: *const i64,
                                                sample_rates: *const i64, n_waveforms: i64, beam_size: c_int, max_depth: c_int,
                                                ids: *const wb_special_ids, is_special: *const u8, tokens_out: *mut i64, capacity: i64,
                                                n_tokens_out: *mut i64) -> c_int;
        pub fn wb_session_align_tokens(s: *mut c_void, n_seqs: i64, window_of_seq: *const i32, tokens: *const i64, lens: *const i64,
                                       first: *const i64, n_heads: i64, heads: *const i32, start_out: *mut i32, end_out: *mut i32,
                                       matrix_out: *mut f32, matrix_capacity: i64) -> c_int;
    }
}

pub type Error = Box<dyn std::error::Error + Send + Sync>;   // token::Result's error type (src/token.rs:6)

fn check(status: c_int) -> Result<(), Error> {
    if status == 0 { return Ok(()); }
    let msg = unsafe { CStr::from_ptr(ffi::wb_last_error()) }.to_string_lossy().into_owned();
    if status == 1 { panic!("{}", msg); }                       // WB_ERR_INVALID_ARG == reference assert!/panic
    Err(format!("whisper_b200 status {}: {}", status, msg).into())
}

pub mod audio {
    use super::*;
    /// src/audio.rs:12-17
    pub fn max_waveform_samples(n_frame_max: usize) -> usize { unsafe { ffi::wb_max_waveform_samples(n_frame_max as i64) as usize } }
    /// src/audio.rs:34-56: waveform [n_batch, n_samples] -> (mel [n_batch, 80, n_frames], n_frames).  The library's frontend tables
    /// are the 16 kHz ones the reference always uses (transcribe.rs:134 passes the file's rate, the binary asserts 16 kHz).
    pub fn prep_audio(waveform: &[f32], n_batch: usize, sample_rate: f64) -> Result<(Vec<f32>, usize), Error> {
        assert!(sample_rate == 16000.0, "prep_audio: only 16 kHz input is supported (src/bin/transcribe/main.rs:38)");
        let n = waveform.len() / n_batch;
        let mut out = vec![0f32; n_batch * 80 * (n / 160)];
        let mut nf = 0i64;
        check(unsafe { ffi::wb_prep_audio(0, waveform.as_ptr(), n_batch as i64, n as i64, out.as_mut_ptr(), &mut nf) })?;
        Ok((out, nf as usize))
    }
    /// Downmix + resampling to the 16 kHz mono everything else takes (wb_resample; the reference's README runs
    /// `sox audio.wav -r 16000 -c 1` instead): `waveform` is frames x `channels` interleaved samples at `sample_rate`.
    /// Unsupported rates (gcd with 16000 leaving up or down above 1024) are an `Err`.
    pub fn resample(waveform: &[f32], channels: usize, sample_rate: usize) -> Result<Vec<f32>, Error> {
        let n_frames = (waveform.len() / channels.max(1)) as i64;
        let n = unsafe { ffi::wb_resampled_length(n_frames, sample_rate as i64) };
        if n < 0 { return Err(format!("resample: unsupported sample rate {}", sample_rate).into()); }
        let mut out = vec![0f32; n as usize];
        let mut n_out = 0i64;
        check(unsafe { ffi::wb_resample(0, waveform.as_ptr(), n_frames, channels as i64, sample_rate as i64, out.as_mut_ptr(), n, &mut n_out) })?;
        Ok(out)
    }
    /// load_audio_waveform (src/bin/transcribe/main.rs:31-55) over wb_load_wav: (interleaved samples, channels, sample rate).
    /// `strict` keeps the binary's 16 kHz mono asserts (a panic here too); without it any rate and channel count loads.
    pub fn load_audio_waveform(path: &str, strict: bool) -> Result<(Vec<f32>, usize, usize), Error> {
        let c = CString::new(path)?;
        let (mut n, mut sr, mut ch) = (0i64, 0i64, 0 as c_int);
        check(unsafe { ffi::wb_load_wav(c.as_ptr(), strict as c_int, std::ptr::null_mut(), 0, &mut n, &mut sr, &mut ch) })?;
        let mut out = vec![0f32; n as usize];
        check(unsafe { ffi::wb_load_wav(c.as_ptr(), strict as c_int, out.as_mut_ptr(), n, &mut n, &mut sr, &mut ch) })?;
        Ok((out, ch as usize, sr as usize))
    }
}

pub mod model {
    use super::*;
    pub use ffi::wb_dims as WhisperConfig;   // src/model/mod.rs:16-39

    /// Decoding state behind `&Whisper` (the reference's `next` closure is `Fn + Clone` over `&whisper`, transcribe.rs:253):
    /// one wb_session (KV caches, workspaces, CUDA stream), created on first use and reused by every call.
    pub(crate) struct Session { pub(crate) h: *mut c_void, pub(crate) max_windows: usize, pub(crate) max_beams: usize, pub(crate) max_text_len: usize }
    impl Drop for Session { fn drop(&mut self) { unsafe { ffi::wb_session_destroy(self.h) } } }

    /// src/model/mod.rs:41-71
    pub struct Whisper { pub(crate) h: *mut c_void, pub config: WhisperConfig, pub(crate) session: Mutex<Option<Session>> }
    unsafe impl Send for Whisper {}
    unsafe impl Sync for Whisper {}          // the model is immutable after finalize; the session sits behind the mutex
    impl Drop for Whisper {
        fn drop(&mut self) {
            *self.session.lock().unwrap() = None;   // sessions die before their model
            unsafe { ffi::wb_model_destroy(self.h) }
        }
    }

    impl Whisper {
        /// Builds the model from the reference's npy tree (src/model/load.rs:19-310): `tensors` yields
        /// (path without ".npy", shape, values) for every file of the tree.
        pub fn from_tensors<'a, I: IntoIterator<Item = (&'a str, &'a [i64], &'a [f32])>>(config: WhisperConfig, tensors: I) -> Result<Self, Error> {
            let mut h = std::ptr::null_mut();
            check(unsafe { ffi::wb_model_create(&config, 0, &mut h) })?;
            let w = Whisper { h, config, session: Mutex::new(None) };
            for (path, shape, data) in tensors {
                let c = CString::new(path)?;
                check(unsafe { ffi::wb_model_set_tensor(w.h, c.as_ptr(), data.as_ptr(), shape.as_ptr(), shape.len() as c_int) })?;
            }
            check(unsafe { ffi::wb_model_finalize(w.h) })?;
            Ok(w)
        }
        /// model::load::load_whisper (src/model/load.rs:295-310): the directory python/dump.py writes.
        pub fn load_npy_tree(dir: &str) -> Result<Self, Error> {
            let c = CString::new(dir)?;
            let mut config: WhisperConfig = unsafe { std::mem::zeroed() };
            check(unsafe { ffi::wb_npy_tree_probe(c.as_ptr(), &mut config) })?;
            let mut h = std::ptr::null_mut();
            check(unsafe { ffi::wb_model_load_npy_tree(c.as_ptr(), 0, 1, &mut h) })?;
            Ok(Whisper { h, config, session: Mutex::new(None) })
        }
        /// The cached session, grown when a call needs more windows / beams / positions than the current one holds.
        pub(crate) fn with_session<R>(&self, max_windows: usize, max_beams: usize, max_text_len: usize,
                                      f: impl FnOnce(*mut c_void) -> Result<R, Error>) -> Result<R, Error> {
            let mut guard = self.session.lock().unwrap();
            let fits = guard.as_ref().map_or(false, |s| s.max_windows >= max_windows && s.max_beams >= max_beams && s.max_text_len >= max_text_len);
            if !fits {
                *guard = None;
                let mut s = std::ptr::null_mut();
                check(unsafe { ffi::wb_session_create(self.h, max_windows as i64, max_beams as i64, max_text_len as i64, 0, &mut s) })?;
                *guard = Some(Session { h: s, max_windows, max_beams, max_text_len });
            }
            f(guard.as_ref().unwrap().h)
        }
        /// mod.rs:52-54: mel [n_batch, 80, n_ctx] -> [n_batch, (n_ctx-1)/2+1, d]
        pub fn forward_encoder(&self, mel: &[f32], n_batch: usize, n_ctx: usize) -> Result<Vec<f32>, Error> {
            let t = (n_ctx - 1) / 2 + 1;
            let mut out = vec![0f32; n_batch * t * self.config.n_audio_state as usize];
            check(unsafe { ffi::wb_forward_encoder(self.h, mel.as_ptr(), n_batch as i64, 80, n_ctx as i64, out.as_mut_ptr()) })?;
            Ok(out)
        }
        /// mod.rs:56-62 (stateless): tokens [n_batch, seq_len], encoder_output [n_batch, n_enc_ctx, d] -> logits [n_batch, seq_len, n_vocab]
        pub fn forward_decoder(&self, tokens: &[i64], n_batch: usize, encoder_output: &[f32], n_enc_ctx: usize) -> Result<Vec<f32>, Error> {
            let seq_len = tokens.len() / n_batch;
            let mut out = vec![0f32; n_batch * seq_len * self.config.n_vocab as usize];
            check(unsafe { ffi::wb_forward_decoder(self.h, tokens.as_ptr(), n_batch as i64, seq_len as i64, encoder_output.as_ptr(), n_enc_ctx as i64, out.as_mut_ptr()) })?;
            Ok(out)
        }
        pub fn encoder_ctx_size(&self) -> usize { self.config.n_audio_ctx as usize }   // mod.rs:64-66
        pub fn decoder_ctx_size(&self) -> usize { self.config.n_text_ctx as usize }    // mod.rs:68-70
    }
}

/// Same public items as the reference's src/beam.rs (BeamNode, beam_search, beam_search_step), generic over the token type
/// and the two closures, with its tie-breaks: `get_top_elements` keeps the EARLIER of two equal scores, `max_by` the LAST
/// maximum.  The library runs the identical search in C++ (whisper-burn_b200/host/beam.hpp) for wb_transcribe_windows; this
/// module is for callers that drive the search themselves over `transcribe::DecoderSteps`.
pub mod beam {
    #[derive(Clone)]
    pub struct BeamNode<T: Clone> { pub seq: Vec<T>, pub log_prob: f64 }   // beam.rs:3-7

    /// beam.rs:9-37
    pub fn beam_search<T, F, G>(initial_beams: Vec<BeamNode<T>>, next: F, is_finished: G, beam_size: usize, max_depth: usize) -> Vec<T>
    where T: Clone, F: Fn(&[BeamNode<T>]) -> Vec<Vec<(T, f64)>> + Clone, G: Fn(&[T]) -> bool + Clone {
        let beams = beam_search_final(initial_beams, next, is_finished, beam_size, max_depth);
        last_max(&beams).map(|b| b.seq.clone()).unwrap_or_default()
    }

    /// beam_search's n-best list: the carried beams when the search stops (`beams` at beam.rs:33), ranked by applying
    /// beam.rs:33-36's max_by again to what remains after each pick (descending log_prob, exact ties with the LATER carried beam
    /// first).  Element 0 is what beam_search returns; at most 2 * beam_size beams.
    pub fn beam_search_nbest<T, F, G>(initial_beams: Vec<BeamNode<T>>, next: F, is_finished: G, beam_size: usize, max_depth: usize)
            -> Vec<BeamNode<T>>
    where T: Clone, F: Fn(&[BeamNode<T>]) -> Vec<Vec<(T, f64)>> + Clone, G: Fn(&[T]) -> bool + Clone {
        let mut rest = beam_search_final(initial_beams, next, is_finished, beam_size, max_depth);
        let mut ranked = Vec::with_capacity(rest.len());
        while !rest.is_empty() {
            let mut best = 0;
            for i in 1..rest.len() { if !(rest[i].log_prob < rest[best].log_prob) { best = i; } }
            ranked.push(rest.remove(best));
        }
        ranked
    }

    /// beam.rs:9-32: the carried beams when the search stops, in carried order
    fn beam_search_final<T, F, G>(initial_beams: Vec<BeamNode<T>>, next: F, is_finished: G, beam_size: usize, max_depth: usize)
            -> Vec<BeamNode<T>>
    where T: Clone, F: Fn(&[BeamNode<T>]) -> Vec<Vec<(T, f64)>> + Clone, G: Fn(&[T]) -> bool + Clone {
        let mut beams = initial_beams;
        for _ in 0..max_depth {
            if let Some(best) = last_max(&beams) {
                if is_finished(&best.seq) { break; }
            }
            beams = beam_search_step(beams, next.clone(), is_finished.clone(), beam_size);
        }
        beams
    }

    /// beam.rs:39-79: `next` sees every beam (finished ones included, their continuations are dropped); up to 2 * beam_size
    /// beams are carried: the best live continuations, then the best finished beams.
    pub fn beam_search_step<T, F, G>(beams: Vec<BeamNode<T>>, next: F, is_finished: G, beam_size: usize) -> Vec<BeamNode<T>>
    where T: Clone, F: Fn(&[BeamNode<T>]) -> Vec<Vec<(T, f64)>>, G: Fn(&[T]) -> bool {
        let continuations = next(&beams);
        let (mut finished, mut grown) = (Vec::new(), Vec::new());
        for (beam, conts) in beams.into_iter().zip(continuations) {
            if is_finished(&beam.seq) { finished.push(beam); continue; }
            for (tok, log_prob) in get_top_elements(&conts, |c| c.1, beam_size) {
                let mut seq = beam.seq.clone();
                seq.push(tok);
                grown.push(BeamNode { seq, log_prob });
            }
        }
        let mut out = get_top_elements(&grown, |b| b.log_prob, beam_size);
        out.extend(get_top_elements(&finished, |b| b.log_prob, beam_size));
        out
    }

    /// beam.rs:81-110: ascending insertion list of at most `num` elements; an element equal to the current minimum of a full
    /// list is inserted in front and evicted at once, so the earlier element survives a tie.
    pub fn get_top_elements<E: Clone>(elems: &[E], score: impl Fn(&E) -> f64, num: usize) -> Vec<E> {
        let mut kept: Vec<(E, f64)> = Vec::with_capacity(num + 1);
        for e in elems {
            let s = score(e);
            if kept.len() == num && (num == 0 || s < kept[0].1) { continue; }
            let at = kept.iter().position(|(_, ks)| *ks >= s).unwrap_or(kept.len());
            kept.insert(at, (e.clone(), s));
            if kept.len() > num { kept.remove(0); }
        }
        kept.into_iter().map(|(e, _)| e).collect()
    }

    fn last_max<T: Clone>(beams: &[BeamNode<T>]) -> Option<&BeamNode<T>> {   // Iterator::max_by(partial_cmp): last maximum
        let mut best: Option<&BeamNode<T>> = None;
        for b in beams { if best.map_or(true, |m| !(b.log_prob < m.log_prob)) { best = Some(b); } }
        best
    }
}

pub mod transcribe {
    use super::*;
    use crate::token::{self, Gpt2Tokenizer, Language, SpecialToken};

    const BEAM_SIZE: usize = 5;     // transcribe.rs:232
    const MAX_DEPTH: usize = 100;   // transcribe.rs:233

    /// What `mels_to_text` looks up in the tokenizer (src/transcribe.rs:179-185) + `is_special` for every id (:243-251).
    pub struct SpecialTokens { pub ids: ffi::wb_special_ids, pub is_special: Vec<u8> }
    impl SpecialTokens {
        pub fn from_tokenizer(bpe: &Gpt2Tokenizer, lang: Language) -> Self {
            let id = |t: SpecialToken| bpe.special_token(t).unwrap() as i64;
            let ids = ffi::wb_special_ids { sot: id(SpecialToken::StartofTranscript), lang: id(SpecialToken::Language(lang)),
                                            transcribe: id(SpecialToken::Transcribe), notimestamps: id(SpecialToken::NoTimeStamps),
                                            eot: id(SpecialToken::EndofText) };
            SpecialTokens { ids, is_special: (0..bpe.vocab_size()).map(|t| bpe.is_special(t) as u8).collect() }
        }
    }

    /// src/transcribe.rs:23-29, same signature minus `<B>`: windows of `max_waveform_samples(n_ctx_max - 10)` samples with 3 s
    /// overlap, prep_audio + encoder + beam search (width 5, depth 100) per window -- all windows batched inside the library --
    /// overlap merge (transcribe.rs:56-63), then the reference's own detokenisation (transcribe.rs:67).
    pub fn waveform_to_text(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>, sample_rate: usize)
            -> token::Result<(String, Vec<usize>)> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(sample_rate * 3).max(1);                             // transcribe.rs:120-123
        let n_windows = waveform.len().saturating_sub(1) / shift + 1;
        let cap = n_windows * (4 + MAX_DEPTH + 1) + 16;
        let mut out = vec![0i64; cap];
        let mut n = 0i64;
        whisper.with_session(n_windows.min(64), BEAM_SIZE, 4 + MAX_DEPTH + 1, |s| {
            check(unsafe { ffi::wb_waveform_to_tokens(s, waveform.as_ptr(), waveform.len() as i64, sample_rate as i64, BEAM_SIZE as c_int,
                                                      MAX_DEPTH as c_int, &sp.ids, sp.is_special.as_ptr(), out.as_mut_ptr(), cap as i64, &mut n) })
        })?;
        let tokens: Vec<usize> = out[..n as usize].iter().map(|&t| t as usize).collect();
        Ok((bpe.decode(&tokens[..], true)?, tokens))
    }

    /// src/transcribe.rs:142-146: a token with the log-prob the search scored it with (0.0 for the prompt, :205-208).
    #[derive(Clone, Copy, Debug, PartialEq)]
    pub struct BeamSearchToken { pub token: usize, pub log_prob: f64 }

    /// waveform_to_text's windowing, beam width and depth, returning the merged tokens with the `BeamSearchToken.log_prob`
    /// each was chosen with (wb_session_last_logprobs: f32 values, which the reference's f64 holds exactly) instead of text.
    pub fn waveform_to_tokens_with_log_probs(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>,
                                             sample_rate: usize) -> token::Result<Vec<BeamSearchToken>> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(sample_rate * 3).max(1);                             // transcribe.rs:120-123
        let n_windows = waveform.len().saturating_sub(1) / shift + 1;
        let cap = n_windows * (4 + MAX_DEPTH + 1) + 16;
        let (mut out, mut lps) = (vec![0i64; cap], vec![0f32; cap]);
        let (mut n, mut n_lp) = (0i64, 0i64);
        whisper.with_session(n_windows.min(64), BEAM_SIZE, 4 + MAX_DEPTH + 1, |s| {
            check(unsafe { ffi::wb_waveform_to_tokens(s, waveform.as_ptr(), waveform.len() as i64, sample_rate as i64, BEAM_SIZE as c_int,
                                                      MAX_DEPTH as c_int, &sp.ids, sp.is_special.as_ptr(), out.as_mut_ptr(), cap as i64, &mut n) })?;
            check(unsafe { ffi::wb_session_last_logprobs(s, 0, lps.as_mut_ptr(), cap as i64, &mut n_lp) })
        })?;
        assert_eq!(n, n_lp, "one log-prob per token");
        Ok((0..n as usize).map(|i| BeamSearchToken { token: out[i] as usize, log_prob: lps[i] as f64 }).collect())
    }

    /// waveform_to_text with the previous-text prompt the reference builds and then shadows (transcribe.rs:43-54, 195-201): window
    /// i is decoded from [<|startofprev|>] + the last (at most) 5 non-special ids merged so far + [sot, lang, transcribe,
    /// notimestamps] (window 0 from the 4 ids alone).  The windows of the waveform are decoded in order, one launch each.
    pub fn waveform_to_text_with_prev_prompt(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>,
                                             sample_rate: usize) -> token::Result<(String, Vec<usize>)> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let startofprev = bpe.special_token(SpecialToken::StartofPrev).unwrap() as i64;              // transcribe.rs:181
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(sample_rate * 3).max(1);                             // transcribe.rs:120-123
        let n_windows = waveform.len().saturating_sub(1) / shift + 1;
        let cap = n_windows * (10 + MAX_DEPTH + 1) + 16;
        let mut out = vec![0i64; cap];
        let mut n = 0i64;
        whisper.with_session(1, BEAM_SIZE, 10 + MAX_DEPTH + 1, |s| {
            check(unsafe { ffi::wb_session_set_prev_prompt(s, startofprev) })?;
            let r = check(unsafe { ffi::wb_waveform_to_tokens(s, waveform.as_ptr(), waveform.len() as i64, sample_rate as i64, BEAM_SIZE as c_int,
                                                              MAX_DEPTH as c_int, &sp.ids, sp.is_special.as_ptr(), out.as_mut_ptr(), cap as i64, &mut n) });
            check(unsafe { ffi::wb_session_set_prev_prompt(s, -1) })?;   // the cached session's other callers use the 4-id prompt
            r
        })?;
        let tokens: Vec<usize> = out[..n as usize].iter().map(|&t| t as usize).collect();
        Ok((bpe.decode(&tokens[..], true)?, tokens))
    }

    /// waveform_to_text for audio at any supported rate and channel count (`waveform`: frames x `channels` interleaved samples
    /// at `sample_rate`): the library converts it to 16 kHz mono on the GPU (wb_waveforms_to_tokens_resampled, the conversion
    /// of audio::resample), then windows, decodes and merges it as waveform_to_text does the converted audio.
    pub fn waveform_to_text_resampled(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>, channels: usize,
                                      sample_rate: usize) -> token::Result<(String, Vec<usize>)> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let n_frames = (waveform.len() / channels.max(1)) as i64;
        let n16 = unsafe { ffi::wb_resampled_length(n_frames, sample_rate as i64) }.max(0) as usize;   // 16 kHz samples
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(16000 * 3).max(1);                                   // transcribe.rs:120-123
        let n_windows = n16.saturating_sub(1) / shift + 1;
        let cap = n_windows * (4 + MAX_DEPTH + 1) + 16;
        let mut out = vec![0i64; cap];
        let mut n = 0i64;
        let (wave, ch, sr) = (waveform.as_ptr(), channels as i64, sample_rate as i64);
        whisper.with_session(n_windows.min(64), BEAM_SIZE, 4 + MAX_DEPTH + 1, |s| {
            check(unsafe { ffi::wb_waveforms_to_tokens_resampled(s, &wave, &n_frames, &ch, &sr, 1, BEAM_SIZE as c_int, MAX_DEPTH as c_int,
                                                                 &sp.ids, sp.is_special.as_ptr(), out.as_mut_ptr(), cap as i64, &mut n) })
        })?;
        let tokens: Vec<usize> = out[..n as usize].iter().map(|&t| t as usize).collect();
        Ok((bpe.decode(&tokens[..], true)?, tokens))
    }

    /// When each token of given sequences was spoken in one audio window: openai-whisper's find_alignment (cross-attention of
    /// the decoder layers n_text_layer / 2 .., normalised, median-filtered, averaged, then dynamic time warping), all on the GPU
    /// (wb_session_align_tokens).  The window is encoded in the cached session; sequence i's tokens from first[i] on are
    /// aligned (4 for a transcribed row: after sot, language, transcribe, notimestamps).  Per aligned token its (start, end)
    /// in seconds from the window's start.
    pub fn align_tokens(whisper: &model::Whisper, waveform_window: &[f32], sequences: &[Vec<usize>], first: &[usize])
            -> Result<Vec<Vec<(f64, f64)>>, Error> {
        let lens: Vec<i64> = sequences.iter().map(|q| q.len() as i64).collect();
        let tokens: Vec<i64> = sequences.iter().flatten().map(|&t| t as i64).collect();
        let firsts: Vec<i64> = first.iter().map(|&f| f as i64).collect();
        if firsts.len() != sequences.len() || sequences.iter().zip(first).any(|(q, &f)| f < 1 || f >= q.len()) {
            return Err("align_tokens: one first index per sequence, in [1, len - 1]".into());
        }
        let windows = vec![0i32; sequences.len()];
        let n_ids: usize = sequences.iter().zip(first).map(|(q, &f)| q.len() - f).sum();
        let (mut start, mut end) = (vec![0i32; n_ids.max(1)], vec![0i32; n_ids.max(1)]);
        whisper.with_session(1, 1, 2, |s| {
            let (wave, n) = (waveform_window.as_ptr(), waveform_window.len() as i64);
            check(unsafe { ffi::wb_session_encode_waveforms(s, &wave, &n, 1) })?;
            check(unsafe { ffi::wb_session_align_tokens(s, sequences.len() as i64, windows.as_ptr(), tokens.as_ptr(), lens.as_ptr(),
                                                        firsts.as_ptr(), 0, std::ptr::null(), start.as_mut_ptr(), end.as_mut_ptr(),
                                                        std::ptr::null_mut(), 0) })
        })?;
        let mut off = 0;
        Ok(sequences.iter().zip(first).map(|(q, &f)| {
            let r = (off..off + q.len() - f).map(|k| (start[k] as f64 * 0.02, end[k] as f64 * 0.02)).collect();
            off += q.len() - f;
            r
        }).collect())
    }

    /// What the transcribe binary does with a WAV file of any rate and channel count (src/bin/transcribe/main.rs:31-55 without
    /// its 16 kHz mono asserts): load it as it is (wb_load_wav with strict_16k_mono = 0), then waveform_to_text_resampled.
    pub fn wav_file_to_text(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, path: &str) -> token::Result<(String, Vec<usize>)> {
        let (waveform, channels, sample_rate) = audio::load_audio_waveform(path, false)?;
        waveform_to_text_resampled(whisper, bpe, lang, waveform, channels, sample_rate)
    }

    /// One hypothesis of a window's n-best list: its tokens (prompt included, 0.0 log-probs there), the cumulative log-prob the
    /// search carried it with (the f64 sum of the tokens' log-probs), and whether it ends in EOT.
    #[derive(Clone, Debug, PartialEq)]
    pub struct Hypothesis { pub tokens: Vec<BeamSearchToken>, pub log_prob: f64, pub finished: bool }

    /// waveform_to_text's windowing, beam width and depth, returning per window (in waveform order) the n-best list the beam
    /// search ranks and drops at beam.rs:33-36 (wb_session_last_nbest): at most 2 * 5 hypotheses, best first, the first being
    /// the window's transcribed row before the overlap merge.
    pub fn waveform_to_tokens_nbest(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>,
                                    sample_rate: usize) -> token::Result<Vec<Vec<Hypothesis>>> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(sample_rate * 3).max(1);                             // transcribe.rs:120-123
        let n_windows = waveform.len().saturating_sub(1) / shift + 1;
        let cap = n_windows * (4 + MAX_DEPTH + 1) + 16;
        let (max_hyps, row_cap) = (2 * BEAM_SIZE, 4 + MAX_DEPTH + 1);
        let mut out = vec![0i64; cap];
        let mut n = 0i64;
        whisper.with_session(n_windows.min(64), BEAM_SIZE, 4 + MAX_DEPTH + 1, |s| {
            check(unsafe { ffi::wb_waveform_to_tokens(s, waveform.as_ptr(), waveform.len() as i64, sample_rate as i64, BEAM_SIZE as c_int,
                                                      MAX_DEPTH as c_int, &sp.ids, sp.is_special.as_ptr(), out.as_mut_ptr(), cap as i64, &mut n) })?;
            let mut windows = Vec::with_capacity(n_windows);
            for w in 0..n_windows {
                let (mut ids, mut lps) = (vec![0i64; max_hyps * row_cap], vec![0f32; max_hyps * row_cap]);
                let (mut lens, mut scores, mut fin) = (vec![0i64; max_hyps], vec![0f64; max_hyps], vec![0i32; max_hyps]);
                let mut n_hyps = 0i64;
                check(unsafe { ffi::wb_session_last_nbest(s, w as i64, max_hyps as i64, row_cap as i64, ids.as_mut_ptr(), lps.as_mut_ptr(),
                                                          lens.as_mut_ptr(), scores.as_mut_ptr(), fin.as_mut_ptr(), &mut n_hyps) })?;
                windows.push((0..n_hyps as usize).map(|r| Hypothesis {
                    tokens: (0..lens[r] as usize).map(|j| BeamSearchToken { token: ids[r * row_cap + j] as usize,
                                                                           log_prob: lps[r * row_cap + j] as f64 }).collect(),
                    log_prob: scores[r], finished: fin[r] != 0 }).collect());
            }
            Ok(windows)
        })
    }

    /// How well given token sequences fit one audio window: `forward_decoder` (mod.rs:131-157) and `log_softmax`
    /// (transcribe.rs:276) at every position, without the special-token mask.  The window (at most
    /// max_waveform_samples(n_audio_ctx - 10) samples) is encoded in the cached session, then every sequence is scored in one
    /// pass on the GPU (wb_session_score_tokens): entry j of a sequence's result is the log-prob of its token j given tokens
    /// 0 .. j-1, entry 0 is 0.0.
    pub fn score_tokens(whisper: &model::Whisper, waveform_window: &[f32], sequences: &[Vec<usize>]) -> Result<Vec<Vec<f64>>, Error> {
        let lens: Vec<i64> = sequences.iter().map(|q| q.len() as i64).collect();
        let tokens: Vec<i64> = sequences.iter().flatten().map(|&t| t as i64).collect();
        let windows = vec![0i32; sequences.len()];
        let mut lp = vec![0f32; tokens.len().max(1)];
        whisper.with_session(1, 1, 2, |s| {
            let (wave, n) = (waveform_window.as_ptr(), waveform_window.len() as i64);
            check(unsafe { ffi::wb_session_encode_waveforms(s, &wave, &n, 1) })?;
            check(unsafe { ffi::wb_session_score_tokens(s, sequences.len() as i64, windows.as_ptr(), tokens.as_ptr(), lens.as_ptr(), 0,
                                                        std::ptr::null(), lp.as_mut_ptr(), std::ptr::null_mut()) })
        })?;
        let mut off = 0;
        Ok(sequences.iter().map(|q| { let r = lp[off..off + q.len()].iter().map(|&x| x as f64).collect(); off += q.len(); r }).collect())
    }

    /// The greedy loop the reference leaves commented out in `mels_to_text` (src/transcribe.rs:314-380), with waveform_to_text's
    /// signature and windowing: per window the arg-max of the raw logits (no special-token mask) until the EOT probability stop,
    /// the repetition cut of find_repeated_tokens_index(tokens, 5, 4) or n_text_ctx tokens, all on the GPU in one decoder launch
    /// per batch of windows (WB_SEARCH_GREEDY_LOOP with max_depth = n_text_ctx - 4: the reference's loop exactly).
    pub fn waveform_to_text_greedy_loop(whisper: &model::Whisper, bpe: &Gpt2Tokenizer, lang: Language, waveform: Vec<f32>, sample_rate: usize)
            -> token::Result<(String, Vec<usize>)> {
        let sp = SpecialTokens::from_tokenizer(bpe, lang);
        let window = audio::max_waveform_samples(whisper.encoder_ctx_size() - 10);            // transcribe.rs:32-34
        let shift = window.saturating_sub(sample_rate * 3).max(1);                             // transcribe.rs:120-123
        let n_windows = waveform.len().saturating_sub(1) / shift + 1;
        let n_ctx = whisper.decoder_ctx_size();
        let cap = n_windows * (n_ctx + 1) + 16;
        let mut out = vec![0i64; cap];
        let mut n = 0i64;
        whisper.with_session(n_windows.min(64), 1, n_ctx, |s| {
            check(unsafe { ffi::wb_session_set_search(s, ffi::WB_SEARCH_GREEDY_LOOP) })?;
            let r = check(unsafe { ffi::wb_waveform_to_tokens(s, waveform.as_ptr(), waveform.len() as i64, sample_rate as i64, 1,
                                                              (n_ctx - 4) as c_int, &sp.ids, std::ptr::null(), out.as_mut_ptr(), cap as i64, &mut n) });
            check(unsafe { ffi::wb_session_set_search(s, ffi::WB_SEARCH_BEAM) })?;   // the cached session's other callers search by beam
            r
        })?;
        let tokens: Vec<usize> = out[..n as usize].iter().map(|&t| t as usize).collect();
        Ok((bpe.decode(&tokens[..], true)?, tokens))
    }

    /// transcribe.rs:385-393 (same signature; private and only reachable from the reference's commented-out greedy loop there).
    pub fn first_repetition_end(tokens: &[usize], period: usize) -> usize {
        let t: Vec<i64> = tokens.iter().map(|&x| x as i64).collect();
        let r = unsafe { ffi::wb_first_repetition_end(t.as_ptr(), t.len() as i64, period as i64) };
        assert!(r >= 0, "attempt to subtract with overflow");   // the reference's `tokens.len() - period`
        r as usize
    }
    /// transcribe.rs:395-419.
    pub fn repetition_period(tokens: &[usize], min_repetitions: usize) -> Option<usize> {
        let t: Vec<i64> = tokens.iter().map(|&x| x as i64).collect();
        match unsafe { ffi::wb_repetition_period(t.as_ptr(), t.len() as i64, min_repetitions as i64) } { r if r > 0 => Some(r as usize), _ => None }
    }
    /// transcribe.rs:421-447.
    pub fn find_repeated_tokens_index(tokens: &[usize], window_size: usize, min_repeat_count: usize) -> Option<(usize, usize)> {
        let t: Vec<i64> = tokens.iter().map(|&x| x as i64).collect();
        let (mut a, mut b) = (0i64, 0i64);
        match unsafe { ffi::wb_find_repeated_tokens_index(t.as_ptr(), t.len() as i64, window_size as i64, min_repeat_count as i64, &mut a, &mut b) } {
            1 => Some((a as usize, b as usize)),
            0 => None,
            _ => panic!("called `Option::unwrap()` on a `None` value"),   // the reference's second `repeats.next().unwrap()`
        }
    }

    /// The `beamsearch_next` closure of transcribe.rs:253-307 as an object: KV-cached decoder steps for the beams of ONE window
    /// (wb_session_step).  `next` returns, per live beam, its `k` best (token, log-prob) continuations of log_softmax over the
    /// vocabulary -- what `beam::beam_search_step` keeps of the reference's V-sized lists -- instead of V floats per beam.
    pub struct DecoderSteps<'a> { whisper: &'a model::Whisper, sp: &'a SpecialTokens, first: bool }
    impl<'a> DecoderSteps<'a> {
        /// mel [1, 80, n_ctx] (already padded as transcribe.rs:161-177 does) -> encoder + cross K/V, prompt fed
        pub fn begin(whisper: &'a model::Whisper, sp: &'a SpecialTokens, mel: &[f32], n_ctx: usize, prompt: &[i64], max_beams: usize) -> Result<Self, Error> {
            whisper.with_session(1, max_beams, whisper.decoder_ctx_size().min(4 + MAX_DEPTH + 1), |s| {
                check(unsafe { ffi::wb_session_encode_mels(s, mel.as_ptr(), 1, 80, n_ctx as i64) })?;
                check(unsafe { ffi::wb_session_begin(s, prompt.as_ptr(), prompt.len() as i64) })
            })?;
            Ok(DecoderSteps { whisper, sp, first: true })
        }
        /// parent_row[r] = cache row (index into the previous call's rows) that beam r extends with token[r];
        /// the special-token mask applies while the longest sequence has <= 5 tokens (transcribe.rs:271-275).
        pub fn next(&mut self, parent_row: &[i32], token: &[i64], max_seq_len: usize, k: usize) -> Result<Vec<Vec<(usize, f64)>>, Error> {
            let n = token.len();
            let (mut ids, mut lps) = (vec![0i64; n * k], vec![0f32; n * k]);
            let windows = vec![0i32; n];
            let bitmap = if self.first { self.sp.is_special.as_ptr() } else { std::ptr::null() };
            self.first = false;
            self.whisper.with_session(1, 1, 2, |s| {
                check(unsafe { ffi::wb_session_step(s, n as i64, windows.as_ptr(), parent_row.as_ptr(), token.as_ptr(), (max_seq_len <= 5) as c_int,
                                                    bitmap, k as c_int, ids.as_mut_ptr(), lps.as_mut_ptr()) })
            })?;
            Ok((0..n).map(|r| (0..k).filter(|&i| ids[r * k + i] >= 0).map(|i| (ids[r * k + i] as usize, lps[r * k + i] as f64)).collect()).collect())
        }
    }
}
