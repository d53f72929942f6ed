"""Phrase boosting per row on the GPU (rs_set_boost_roots, boosting.combine_tables): every row of a mixed batch, and every
stream of a mixed set of live streams, decodes exactly as it does alone with its own list set globally -- in every kBoost
instance of the offline and resumed decode, at the tiny size and at the bench's production geometry -- and the C / Python
surfaces (argument checks, phrases=, open(boosting=...), the global setting restored after a call)."""
import random

import numpy as np
import pytest
import torch

from ngram_oracle import write_arpa
from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables, combine_tables
from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

LM_ALPHA = 0.1


def _enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()


def _random_list(V, n, seed, max_len=3, score=2.0):
    rng = np.random.default_rng(seed)
    return PhraseBoostingConfig([[int(x) for x in rng.integers(0, V, int(rng.integers(1, max_len + 1)))] for _ in range(n)], score)


def _set(eng, tables):
    eng.set_phrase_boosting(None if tables is None else tables.bonus, None if tables is None else tables.next)


def _rows_equal(got, ref, b, r, tag):
    """row b of the batch outputs ``got`` against row r of ``ref``, byte for byte over the row's stored tokens"""
    n = int(ref[2][r])
    assert int(got[2][b]) == n, f"{tag}: n_tok {int(got[2][b])} vs {n}"
    for i in (0, 1) + ((3,) if len(ref) > 3 else ()):
        assert torch.equal(got[i][b, :n], ref[i][r, :n]), f"{tag}: output {i}"


def _mixed_vs_solo(eng, V, enc, lens, lists, alpha, tag, base=None, tok=None):
    """Decode the batch on the combined table with per-row roots, then every row alone with its list (or ``base`` for a None
    row) set globally.  Returns how many rows the boosting changed against the unboosted decode."""
    tables, roots = combine_tables(lists, V, tok, base=base)
    U = None
    _set(eng, tables)
    eng.set_boost_roots(roots)
    try:
        mixed = [a.cpu() for a in eng.greedy(enc, lens, U, alpha=alpha)]
    finally:
        _set(eng, None)
    plain = [a.cpu() for a in eng.greedy(enc, lens, U, alpha=alpha)]
    changed = 0
    for b, cfg in enumerate(lists):
        own = cfg if cfg is not None else base
        _set(eng, None if own is None else build_tables(own, V, tok))
        try:
            solo = [a.cpu() for a in eng.greedy(enc[b:b + 1].contiguous(), lens[b:b + 1], U, alpha=alpha)]
        finally:
            _set(eng, None)
        _rows_equal(mixed, solo, b, 0, f"{tag} row {b}")
        n = int(solo[2][0])
        changed += int(int(plain[2][b]) != n or not torch.equal(plain[0][b, :n], solo[0][0, :n]))
    return changed


@pytest.fixture(scope="module")
def tiny_lm_tables(tmp_path_factory, tiny_cfg):
    path = str(tmp_path_factory.mktemp("lm") / "tiny3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    return build_lm_tables(NgramLMConfig(path, LM_ALPHA), tiny_cfg.vocab_size)


@pytest.mark.parametrize("conf", [False, True])
@pytest.mark.parametrize("lm", [False, True])
def test_mixed_batch_equals_solo_tiny(tiny_cfg, tiny_engine, tiny_lm_tables, conf, lm):
    eng, V = tiny_engine, tiny_cfg.vocab_size
    enc, lens = _enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9, 28], seed=31)
    a = _random_list(V, 12, seed=1)
    lists = [a, None, _random_list(V, 8, seed=2, score=3.0), a, _random_list(V, 20, seed=3, score=1.0), None,
             _random_list(V, 4, seed=4, score=5.0), PhraseBoostingConfig([list(p) for p in a.phrases], a.score),
             _random_list(V, 12, seed=5), _random_list(V, 30, seed=6)]
    eng.set_ngram_lm(tiny_lm_tables if lm else None)
    try:
        changed = _mixed_vs_solo(eng, V, enc, lens, lists, 0.33 if conf else None, f"conf={conf} lm={lm}")
        # with a global list in region 0: the None rows decode with it
        changed_base = _mixed_vs_solo(eng, V, enc, lens, lists, 0.33 if conf else None, f"conf={conf} lm={lm} base",
                                      base=_random_list(V, 6, seed=7))
    finally:
        eng.set_ngram_lm(None)
    assert changed >= 3 and changed_base >= 3, (changed, changed_base)


def test_none_rows_without_global_list_equal_unboosted(tiny_cfg, tiny_engine):
    eng = tiny_engine
    enc, lens = _enc(tiny_cfg, [30, 12, 25], seed=32)
    plain = [a.cpu() for a in eng.greedy(enc, lens, alpha=0.5)]
    tables, roots = combine_tables([None, None, None], tiny_cfg.vocab_size)
    _set(eng, tables)
    eng.set_boost_roots(roots)
    try:
        got = [a.cpu() for a in eng.greedy(enc, lens, alpha=0.5)]
    finally:
        _set(eng, None)
    assert all(torch.equal(x, y) for x, y in zip(got, plain))


def _phrases_from_pieces(pieces, n, seed):
    """n text phrases of 1-4 pieces each, drawn from the piece table's kana / ideographs as scripts/bench_boosting.py draws them"""
    rng = np.random.default_rng(seed)
    return ["".join(pieces[int(i)] for i in rng.integers(7, len(pieces), int(rng.integers(1, 5)))) for _ in range(n)]


def test_production_geometry_mixed_equals_solo():
    """The bench's 32 x 30 s clips at the production size, 32 different lists of 20-100 phrases drawn from the piece table
    (text through the tokenizer), lambda = 2 as in the boosting benchmark."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    tok = PieceTableTokenizer(synthetic_pieces(cfg.vocab_size))
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(32)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    enc, enc_len = eng.encode(*eng.log_mel(x, torch.full((32,), len(waves[0]), dtype=torch.int32).cuda()))
    rng = np.random.default_rng(9)
    lists = [PhraseBoostingConfig(_phrases_from_pieces(tok.pieces, int(rng.integers(20, 101)), 100 + i), 2.0) for i in range(32)]
    for alpha in (None, 0.33):
        changed = _mixed_vs_solo(eng, cfg.vocab_size, enc, enc_len, lists, alpha, f"production alpha={alpha}", tok=tok)
        print(f"production, alpha {alpha}: boosting changed the transcript of {changed} of 32 clips")
        assert changed >= 8


def test_bad_roots_rejected_before_any_launch(tiny_cfg, tiny_engine):
    eng = tiny_engine
    enc, lens = _enc(tiny_cfg, [12, 7, 9], seed=33)
    lib, h = eng.lib, eng.h
    roots = lambda *v: np.asarray(v, np.int32)
    set_roots = lambda r: lib.rs_set_boost_roots(h, r.ctypes.data, r.size)
    before = eng.launch_count
    assert set_roots(roots(0, 0)) == -1 and b"no phrase-boosting table" in lib.rs_last_error(h)    # no table set
    tables, _ = combine_tables([_random_list(tiny_cfg.vocab_size, 5, seed=8)], tiny_cfg.vocab_size)
    _set(eng, tables)
    try:
        for bad in (roots(0, tables.n_states), roots(-1, 0), roots(0, 1 << 20)):
            assert set_roots(bad) == -1 and b"outside" in lib.rs_last_error(h)
        assert lib.rs_set_boost_roots(h, None, 2) == -1 and lib.rs_set_boost_roots(h, roots(0).ctypes.data, -1) == -1
        assert set_roots(roots(0, 1)) == 0
        with pytest.raises(RuntimeError, match="boosting roots"):                                # B = 3 > n = 2
            eng.greedy(enc, lens)
        with pytest.raises(RuntimeError, match="boosting roots"):
            eng.transcribe_host(torch.zeros(3, 16000), torch.full((3,), 16000, dtype=torch.int32))
        with pytest.raises(RuntimeError, match="boosting roots"):
            eng.transcribe_device(torch.zeros(3, 16000, device="cuda"), torch.full((3,), 16000, dtype=torch.int32, device="cuda"))
        i32 = lambda *v: torch.tensor(v, dtype=torch.int32)
        states = torch.zeros(3, eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
        out = (torch.zeros(3, 50, dtype=torch.int32), torch.zeros(3, 50, dtype=torch.int32), torch.zeros(3, dtype=torch.int32))
        with pytest.raises(RuntimeError, match="boosting roots"):
            eng.stream_step(torch.zeros(3, 16000), i32(16000, 16000, 16000), i32(0, 0, 0), i32(1, 1, 1), i32(0, 1, 2), states, 50, out)
        with pytest.raises(RuntimeError, match="boosting roots"):
            eng.greedy_resume(enc, i32(0, 0, 0), i32(1, 1, 1), i32(0, 1, 2), states)
        assert eng.launch_count == before and int(states.sum()) == 0
        # n = 0 clears, and so does setting a table
        eng.set_boost_roots(None)
        eng.greedy(enc, lens)
        eng.set_boost_roots([0, 0])
        _set(eng, tables)
        eng.greedy(enc, lens)
    finally:
        _set(eng, None)


# ---- the Python API
def _audios(n, seed):
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    return [AudioData(synth_clip(seed + i, 0.8 + 0.45 * i).astype(np.float32), 16000) for i in range(n)]


def _hyp(r):
    return r.hypothesis.y_sequence.tolist(), r.hypothesis.timestamp, r.hypothesis.token_confidence


@pytest.mark.parametrize("conf", [False, True])
def test_transcribe_batch_phrases_equals_solo(tiny_cfg, conf):
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    V = tiny_cfg.vocab_size
    model = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, confidence=ConfidenceConfig() if conf else None,
                           boosting=_random_list(V, 5, seed=20))
    audios = _audios(7, seed=60)
    a = _random_list(V, 10, seed=21, score=3.0)
    lists = [a, None, PhraseBoostingConfig(["あ", "い"], 2.0), a, _random_list(V, 6, seed=22, score=4.0), None, _random_list(V, 9, seed=23)]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    before = [_hyp(r) for r in asr.transcribe_batch(model, audios, cfg)]
    got = [_hyp(r) for r in asr.transcribe_batch(model, audios, cfg, phrases=lists)]
    dev = model._phrase_cache[1]
    again = [_hyp(r) for r in asr.transcribe_batch(model, audios, cfg, phrases=lists)]
    assert again == got and model._phrase_cache[1] is dev                      # cached: not uploaded again
    after = [_hyp(r) for r in asr.transcribe_batch(model, audios, cfg)]
    assert after == before                                                     # the global setting is back
    # audio that is resampled on the GPU (iter_token_batches_raw) takes the same lists
    raw = [AudioData(np.repeat(x.waveform, 3)[::2].copy(), 24000) for x in audios]
    got_raw = [_hyp(r) for r in asr.transcribe_batch(model, raw, cfg, phrases=lists)]
    glob = model.boosting
    solo, solo_raw = [], []
    for au, rw, lst in zip(audios, raw, lists):
        model.set_phrase_boosting(lst if lst is not None else glob)
        solo.append(_hyp(asr.transcribe_batch(model, [au], cfg)[0]))
        solo_raw.append(_hyp(asr.transcribe_batch(model, [rw], cfg)[0]))
    model.set_phrase_boosting(glob)
    assert got == solo and got_raw == solo_raw
    assert sum(g != b for g, b in zip(got, before)) >= 2


def test_phrases_rejected_with_alsd_and_bad_lengths(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    audios = _audios(2, seed=70)
    alsd = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, decoding="alsd")
    with pytest.raises(ValueError, match="ALSD"):
        asr.transcribe_batch(alsd, audios, phrases=[None, None])
    greedy = asr.load_model(synthetic=True, config=tiny_cfg, seed=0)
    with pytest.raises(ValueError, match="2 inputs"):
        asr.transcribe_batch(greedy, audios, phrases=[None])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu_phrases(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    V = tiny_cfg.vocab_size
    one = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2)
    two = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, devices=[0, 1])
    audios = _audios(6, seed=80)
    lists = [_random_list(V, 8, seed=30 + i % 3, score=3.0) if i != 2 else None for i in range(6)]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    assert ([_hyp(r) for r in asr.transcribe_batch(one, audios, cfg, phrases=lists)] ==
            [_hyp(r) for r in asr.transcribe_batch(two, audios, cfg, phrases=lists)])


# ---- streams
def _schedule(n_streams, seed):
    """Per stream: (open tick, pieces of irregular size)."""
    from reazonspeech_b200.synth import synth_clip
    rng = random.Random(seed)
    out = []
    for i in range(n_streams):
        w = synth_clip(200 + i, rng.uniform(1.0, 6.0)).astype(np.float32)
        sizes, pos = [], 0
        while pos < len(w):
            k = rng.choice([5920, 5920, 3000, 12000, 777])
            sizes.append(w[pos:pos + k]); pos += k
        out.append((rng.randint(0, 6), sizes))
    return out


def _run_streams(model, sched, lists, which, max_batch, change_at=None, change_to=None):
    """Streams ``which`` of ``sched`` on one transcriber, stream i opened with ``lists[i]`` (None when ``lists`` is None); at
    tick ``change_at`` the model's global list becomes ``change_to``.  -> {i: (token ids, timestamps, token confidence)}"""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    model.max_batch = max_batch
    st = StreamingTranscriber(model, max_streams=len(which))
    sid, nxt, done, tick = {}, {i: 0 for i in which}, {}, 0
    while len(done) < len(which):
        if tick == change_at:
            model.set_phrase_boosting(change_to)
        for i in which:
            t_open, pieces = sched[i]
            if tick == t_open:
                sid[i] = st.open(boosting=None if lists is None else lists[i])
            if i in sid and nxt[i] < len(pieces):
                st.feed(sid[i], pieces[nxt[i]]); nxt[i] += 1
                if nxt[i] == len(pieces):
                    st.close(sid[i])
        st.step()
        for i in [i for i, s in sid.items() if st.done(s)]:
            done[i] = _hyp(st.result(sid.pop(i)))
        tick += 1
        assert tick < 10000
    return done


@pytest.mark.parametrize("conf", [False, True])
def test_streams_equal_solo_runs(tiny_cfg, conf):
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.nemo.asr import load_model
    V = tiny_cfg.vocab_size
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg, confidence=ConfidenceConfig() if conf else None)
    sched = _schedule(7, seed=3)
    a = _random_list(V, 10, seed=40, score=3.0)
    lists = [a, None, _random_list(V, 6, seed=41, score=4.0), _random_list(V, 15, seed=42), a, None, _random_list(V, 8, seed=43, score=5.0)]
    batched = _run_streams(model, sched, lists, list(range(7)), max_batch=3)
    plain = _run_streams(model, sched, None, list(range(7)), max_batch=3)
    changed = 0
    for i in range(7):
        model.set_phrase_boosting(lists[i])
        alone = _run_streams(model, sched, None, [i], max_batch=1)[i]
        model.set_phrase_boosting(None)
        assert batched[i] == alone, f"stream {i}"
        changed += int(alone != plain[i])
    assert changed >= 3
    # the global list changes mid-stream: streams with their own list are moved, not restarted
    moved = _run_streams(model, sched, lists, list(range(7)), max_batch=3, change_at=4, change_to=_random_list(V, 30, seed=44))
    model.set_phrase_boosting(None)
    for i in range(7):
        if lists[i] is not None:
            assert moved[i] == batched[i], f"stream {i} after the global change"


@pytest.mark.parametrize("conf", [False, True])
def test_out_of_range_states_fall_back_to_the_row_root(tiny_cfg, tiny_engine, conf):
    """A transition or a stream record's state outside the table sends a row to ITS root: every row of a mixed batch whose
    region has half its transitions pointing outside the table, and whose records are reset to -1 and to n_states half-way,
    equals the row alone with its own table edited the same way (where the fallback is state 0)."""
    eng, V = tiny_engine, tiny_cfg.vocab_size
    enc, lens = _enc(tiny_cfg, [37, 30, 44, 21], seed=34)
    lists = [_random_list(V, 12, seed=60 + i, score=3.0) for i in range(4)]
    tables, roots = combine_tables(lists, V)
    cut = list(range(0, V, 2))                                         # even tokens leave the table
    solo_tables = []
    for cfg_, r in zip(lists, roots):
        t = build_tables(cfg_, V)
        t.next[:, cut] = -1
        tables.next[r:r + t.n_states, cut] = -1
        solo_tables.append(t)
    alpha = 0.5 if conf else None
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    mid = [int(n) // 2 for n in lens.tolist()]

    def halves(tab, root_list, rows):
        _set(eng, tab)
        if root_list is not None:
            eng.set_boost_roots(root_list)
        try:
            states = torch.zeros(len(rows), eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
            e, sl = enc[rows].contiguous(), i32(list(range(len(rows))))
            first = [a.cpu() for a in eng.greedy_resume(e, i32([0] * len(rows)), i32([mid[b] for b in rows]), sl, states, alpha=alpha)]
            out_of_range = [-1 if i % 2 == 0 else tab.n_states for i in range(len(rows))]
            states.view(torch.int32)[:, 1] = torch.tensor(out_of_range, dtype=torch.int32, device="cuda")
            second = [a.cpu() for a in eng.greedy_resume(e, i32([mid[b] for b in rows]), lens[rows].cpu(), sl, states, alpha=alpha)]
            whole = [a.cpu() for a in eng.greedy(e, lens[rows], alpha=alpha)]
            return first, second, whole
        finally:
            _set(eng, None)

    mixed = halves(tables, roots, [0, 1, 2, 3])
    for b in range(4):
        solo = halves(solo_tables[b], None, [b])
        for part, name in zip(range(3), ("first half", "second half after a reset", "offline")):
            _rows_equal(mixed[part], solo[part], b, 0, f"conf={conf} row {b} {name}")
    assert sum(int(n) for n in mixed[2][2]) > 20
