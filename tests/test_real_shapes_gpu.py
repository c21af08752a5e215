"""GPU parity tests at the REAL shapes of BASELINE.json configs 3-5 (small.en 12 layers x 24 rows x V = 51 864, medium
d = 1024, large-v2 d = 1280 with beams), against committed oracle fixtures (tests/golden/tokens_real.json, written by
tests/golden/make_golden_real.py from the CPU oracle; the oracle itself is too slow to re-run these shapes inside the suite).

Token ids must be identical.  The synthetic deep models decode to one or two distinct tokens per window (what differs between
windows is WHERE the switch happens), so the tests also compare the continuous quantities the search consumes: the 5 best ids
and their log-probs at every step, through wb_session_step (the beamsearch_next closure, transcribe.rs:253-307), with an absolute
tolerance of 2e-4 on log-probs of magnitude ~10 (fp32 rounding through 12-32 layers; ids of candidates whose oracle log-probs lie
closer than the tolerance may swap)."""
import numpy as np
import pytest

import harness as h
import wb200  # noqa: F401
from harness import is_special_of, kv_code
from oracle import synth
from whisper_burn_b200 import model, transcribe

pytestmark = pytest.mark.gpu


def check_topk_steps(sess, sp, windows, recs, depth):
    """Greedy re-run through wb_session_step with k = 5: at every step the 5 best (id, log-prob) of every row against the oracle."""
    n = len(windows)
    sess.encode_waveforms(windows)
    prompt = sp.prompt()
    sess.begin(prompt)
    last = [prompt[-1]] * n
    rows = list(range(n))
    worst = 0.0
    for step in range(depth):
        ids, lps = sess.step(rows, rows, last, step + 4 <= 5, is_special_of(sp) if step == 0 else None, 5)
        for r in range(n):
            want_ids, want_lp = recs[r]["top5"][step]
            err = np.abs(lps[r] - np.asarray(want_lp, np.float32)).max()
            worst = max(worst, float(err))
            assert err < h.REAL_LP_TOL, f"row {r} step {step}: log-probs {lps[r]} vs oracle {want_lp}"
            for j in range(5):   # ids identical unless the oracle's own values are within the tolerance of a neighbour
                if int(ids[r, j]) != want_ids[j]:
                    near = [abs(want_lp[j] - want_lp[i]) < h.REAL_LP_TOL for i in range(5) if i != j]
                    assert any(near), f"row {r} step {step}: ids {ids[r]} vs oracle {want_ids}"
            last[r] = recs[r]["tokens"][4 + step]      # follow the oracle's greedy path (== ids[r, 0] when margins allow)
            assert int(ids[r, 0]) == last[r]
    return worst


@pytest.fixture(scope="module")
def small_en():
    return h.named_model("small.en")


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_small_en_8_chunks_greedy_golden(small_en, kv):
    """BASELINE config 3: small.en, 8 x 30 s chunks = 24 reference windows decoded in ONE batch, greedy to depth 100
    (TextDecoder::forward mod.rs:131-157 through the search closure transcribe.rs:253-309)."""
    dims, sp, wh, *_ = small_en
    g = h.golden("tokens_real")["small.en"]
    waves, recs = h.real_windows("small.en", kv)
    want = [r["tokens"] for r in recs]
    sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv))
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 5
    bad = [i for i in range(24) if got[i] != want[i]]
    assert not bad, f"windows {bad} differ (oracle min margin {g['min_margin_' + kv]})"


def test_small_en_step_logprobs_vs_oracle(small_en):
    dims, sp, wh, *_ = small_en
    waves, recs = h.real_windows("small.en", "f32", range(8))
    sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=105)
    worst = check_topk_steps(sess, sp, waves, recs, 100)
    assert sess.last_decoder() == 5
    print("small.en 24 rows x 100 steps: worst |log-prob - oracle| =", worst)


def test_medium_greedy_and_logprobs_golden():
    """BASELINE config 4 shape (d = 1024, 24 layers): chunk 0 = 3 windows, greedy depth 30."""
    g = h.golden("tokens_real")["medium"]
    dims, w_np, _ = synth.make_weights("medium", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    chunk = synth.chunk_waveform(0)
    waves = [chunk[s:e] for s, e in g["bounds"]]
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=35)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=30)
    assert sess.last_decoder() == 5
    assert got == [r["tokens"] for r in g["f32"]], f"oracle min margin {g['min_margin_f32']}"
    worst = check_topk_steps(sess, sp, waves, g["f32"], 30)
    print("medium 3 rows x 30 steps: worst |log-prob - oracle| =", worst)


@pytest.fixture(scope="module")
def large_v2():
    dims, w_np, _ = synth.make_weights("large-v2", seed=0)
    return dims, synth.special_tokens(dims), model.Whisper(dims, w_np)


@pytest.mark.parametrize("kv", ["f16", "f32"])
def test_large_v2_beam5_golden(large_v2, kv):
    """BASELINE config 5 shape (d = 1280, 32 layers, beam width 5, fp16 K/V cache): the short window of chunk 0, depth 20;
    host beam search (beam.rs:9-79) over wb_session_step."""
    g = h.golden("tokens_real")["large-v2"]
    dims, sp, wh = large_v2
    s, e = g["window"]
    wave = synth.chunk_waveform(0)[s:e]
    sess = transcribe.Session(wh, max_windows=1, max_beams=5, max_text_len=25, kv_dtype=kv_code(kv))
    got = sess.transcribe_windows([wave], sp, is_special_of(sp), beam_size=5, max_depth=20)[0]
    assert sess.last_decoder() == 5
    assert got == g[kv]["tokens"], f"oracle min margin {g[kv]['min_margin']}"


# ---------------------------------------------------------------- tiny.en, the cluster decoder's configurations (decoder6.cu)
@pytest.fixture(scope="module")
def tiny_en():
    return h.named_model("tiny.en")


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_cluster_decoder_one_chunk(tiny_en, kv, monkeypatch):
    """BASELINE config 2 through decoder6.cu (one CTA per head, 6-CTA clusters) with a single n-tile in the vocabulary
    projection."""
    dims, sp, wh, *_ = tiny_en
    monkeypatch.setenv("WB200_DECODER", "6")     # 3 rows are decoder4.cu's range by default
    waves, recs = h.real_windows("tiny.en", kv, [0])
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv))
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 6
    h.check_ids_where_separated(got, recs)


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_cluster_decoder_8_chunks(tiny_en, kv):
    """tiny.en, 8 x 30 s chunks = 24 rows in one launch: one cluster per row (rows beyond the co-resident clusters are looped),
    three n-tiles in the vocabulary projection."""
    dims, sp, wh, *_ = tiny_en
    waves, recs = h.real_windows("tiny.en", kv, range(8))
    sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv))
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 6
    h.check_ids_where_separated(got, recs)
    # batching invariance: 9 windows (two n-tiles, the second partially filled) give the same ids as inside the batch of 24
    sess9 = transcribe.Session(wh, max_windows=9, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv))
    got9 = sess9.transcribe_windows(waves[5:14], sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess9.last_decoder() == 6
    h.check_ids_where_separated(got9, recs[5:14])
