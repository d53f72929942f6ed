"""Streaming on the GPU (reazonspeech_b200/streaming.py): the resumed decode kernel against one-call decodes, bit for bit, in every
instance (confidence x boosting x LM) and at the production decoder size; the whole path at unlimited context against
transcribe(); finite contexts batched against one stream at a time and against the oracle; table changes mid-stream."""
import random

import numpy as np
import pytest
import torch

from ngram_oracle import write_arpa
from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables
from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables
from reazonspeech_b200.streaming import PAD_SAMPLES, StreamingConfig
from streaming_oracle import follow_resume

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

NEAR_TIE = 1e-3
LM_ALPHA = 0.1


def _enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()


def _set_tables(eng, boost, lm):
    eng.set_phrase_boosting(None if boost is None else boost.bonus, None if boost is None else boost.next)
    eng.set_ngram_lm(lm)


def _cuts(rng, tokens, frames, T):
    """1-6 ranges covering [0, T): random cuts, one right after a frame that emitted several tokens, an empty range and a
    one-frame range."""
    multi = [f for f in set(frames) if frames.count(f) > 1]
    cuts = {rng.randint(0, T) for _ in range(rng.randint(0, 3))}
    if multi:
        cuts.add(rng.choice(multi) + 1)
    if T > 2 and rng.random() < 0.5:
        t = rng.randint(1, T - 1)
        cuts |= {t, t + 1}
    cuts = sorted(cuts - {0, T})[:4]
    edges = [0] + cuts + [T]
    if rng.random() < 0.5:
        k = rng.randint(0, len(edges) - 1)
        edges.insert(k, edges[k])                                      # an empty range
    return list(zip(edges, edges[1:]))


def _resume_equals_one_call(eng, cfg, enc, lens, alpha, seed, tag):
    B, T = enc.shape[0], enc.shape[1]
    U = T * cfg.max_symbols
    ref = [a.cpu() for a in eng.greedy(enc, lens, U, alpha=alpha)]
    rng = random.Random(seed)
    ranges = [_cuts(rng, ref[0][b, :int(ref[2][b])].tolist(), ref[1][b, :int(ref[2][b])].tolist(), int(lens[b])) for b in range(B)]
    start = [0 if b % 3 else rng.randint(0, 2) for b in range(B)]     # some rows join later: fresh and resumed rows in one batch
    n_rec = B + 3
    slot_of = rng.sample(range(n_rec), B)                              # permuted slots; three records never used
    states = torch.zeros(n_rec, eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
    spare = [s for s in range(n_rec) if s not in slot_of]
    states[spare] = torch.randint(0, 256, (len(spare), eng.stream_state_bytes), dtype=torch.uint8, device="cuda")
    spare_before = states[spare].clone()
    got = [([], [], []) for _ in range(B)]
    n_calls = max(s + len(r) for s, r in zip(start, ranges))
    for k in range(n_calls):
        rows = [b for b in range(B) if start[b] <= k]
        if not rows:
            continue
        rng.shuffle(rows)
        seg = lambda b: ranges[b][k - start[b]] if k - start[b] < len(ranges[b]) else (int(lens[b]), int(lens[b]))
        db = torch.tensor([seg(b)[0] for b in rows], dtype=torch.int32)
        de = torch.tensor([seg(b)[1] for b in rows], dtype=torch.int32)
        sl = torch.tensor([slot_of[b] for b in rows], dtype=torch.int32)
        out = [a.cpu() for a in eng.greedy_resume(enc[rows].contiguous(), db, de, sl, states, U, alpha=alpha)]
        for r, b in enumerate(rows):
            n = int(out[2][r])
            got[b][0].extend(out[0][r, :n].tolist()); got[b][1].extend(out[1][r, :n].tolist())
            if alpha is not None:
                got[b][2].append(out[3][r, :n])
    for b in range(B):
        n = int(ref[2][b])
        assert got[b][0] == ref[0][b, :n].tolist() and got[b][1] == ref[1][b, :n].tolist(), f"{tag} b={b} ranges={ranges[b]}"
        if alpha is not None:
            assert torch.equal(torch.cat(got[b][2]) if got[b][2] else torch.zeros(0, 4), ref[3][b, :n]), f"{tag} b={b}: stats"
    assert torch.equal(states[spare], spare_before), f"{tag}: records outside the batch changed"
    return sum(int(n) for n in ref[2])


@pytest.fixture(scope="module")
def tiny_lm_tables(tmp_path_factory, tiny_cfg):
    path = str(tmp_path_factory.mktemp("lm") / "tiny3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    return build_lm_tables(NgramLMConfig(path, LM_ALPHA), tiny_cfg.vocab_size)


@pytest.mark.parametrize("conf", [False, True])
@pytest.mark.parametrize("boost", [False, True])
@pytest.mark.parametrize("lm", [False, True])
def test_resume_is_exact_tiny(tiny_cfg, tiny_engine, tiny_lm_tables, conf, boost, lm):
    eng = tiny_engine
    enc, lens = _enc(tiny_cfg, [37, 64, 1, 48, 0, 60, 23, 55], seed=11)
    tables = None
    if boost:                                                          # phrases the plain decode spells: they match across splits
        _set_tables(eng, None, None)
        tk, _, nt = [a.cpu() for a in eng.greedy(enc, lens)]
        phrases = [tk[b, i:i + 3].tolist() for b in range(tk.shape[0]) for i in range(0, max(int(nt[b]) - 3, 0), 5)]
        tables = build_tables(PhraseBoostingConfig(phrases[:40], 3.0), tiny_cfg.vocab_size)
    _set_tables(eng, tables, tiny_lm_tables if lm else None)
    try:
        n = _resume_equals_one_call(eng, tiny_cfg, enc, lens, 0.5 if conf else None, seed=1 + 2 * boost + 4 * lm,
                                    tag=f"conf={conf} boost={boost} lm={lm}")
        assert n > 20
    finally:
        _set_tables(eng, None, None)


@pytest.fixture(scope="module")
def full_model():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from reazonspeech_b200.nemo.asr import load_model
    return load_model("cuda:0", synthetic=True, max_batch=8)


def test_resume_is_exact_production(full_model):
    eng, cfg = full_model.engine, full_model.cfg
    assert cfg.joint_hidden == 640 and cfg.pred_hidden == 640
    enc, lens = _enc(cfg, [120, 200, 3, 157, 188, 90], seed=5)
    for conf in (None, 0.5):
        n = _resume_equals_one_call(eng, cfg, enc, lens, conf, seed=7, tag=f"production conf={conf}")
        assert n > 20


def test_resume_rejects_bad_step_arguments(tiny_cfg, tiny_engine):
    eng = tiny_engine
    states = torch.zeros(4, eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
    wav = torch.zeros(2, 32000)
    lens = torch.tensor([32000, 20000], dtype=torch.int32)
    out = (torch.zeros(2, 100, dtype=torch.int32), torch.zeros(2, 100, dtype=torch.int32), torch.zeros(2, dtype=torch.int32))
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32)
    for db, de, sl in ((i32(0, 0), i32(5, 5), i32(1, 1)),               # repeated slot
                       (i32(3, 0), i32(2, 5), i32(0, 1)),               # dec_begin > dec_end
                       (i32(0, 0), i32(5, 200), i32(0, 1)),             # beyond rs_enc_valid(len)
                       (i32(-1, 0), i32(5, 5), i32(0, 1))):
        with pytest.raises(RuntimeError):
            eng.stream_step(wav, lens, db, de, sl, states, 100, out)
    assert int(states.sum()) == 0


# ---- the whole path
def _stream_all(model, waves, config):
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    st = StreamingTranscriber(model, config, max_streams=len(waves))
    ids = [st.open() for _ in waves]
    for sid, w in zip(ids, waves):
        st.feed(sid, w)
        st.close(sid)
    finals = {sid: [] for sid in ids}
    while not all(st.done(s) for s in ids):
        for sid, subs in st.step().items():
            finals[sid] += subs
    return [st.result(s) for s in ids], [finals[s] for s in ids]


def _anchor(model, waves):
    from reazonspeech_b200.nemo.asr import audio_from_numpy, transcribe_batch
    longest = max(len(w) for w in waves) / 16000 + 1.0
    cfg = StreamingConfig(1.6, 0.08 * int(longest / 0.08 + 1), 0.08 * int(longest / 0.08 + 1))
    results, finals = _stream_all(model, waves, cfg)
    refs = transcribe_batch(model, [audio_from_numpy(w, 16000) for w in waves])
    for i, (got, ref, fin) in enumerate(zip(results, refs, finals)):
        assert got.text == ref.text and got.subwords == ref.subwords and got.segments == ref.segments, f"clip {i}"
        assert fin == ref.subwords, f"clip {i}: per-step subwords"
    return sum(len(r.subwords) for r in refs)


def test_unlimited_context_equals_transcribe_tiny(tiny_cfg):
    from reazonspeech_b200.nemo.asr import load_model
    from reazonspeech_b200.synth import synth_clip
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg, max_batch=3)
    waves = [synth_clip(40 + i, s).astype(np.float32) for i, s in enumerate((2.0, 3.3, 0.7, 5.1))]
    assert _anchor(model, waves) > 10


def test_unlimited_context_equals_transcribe_production(full_model):
    from reazonspeech_b200.synth import synth_clip
    waves = [synth_clip(i, 30.0).astype(np.float32) for i in range(4)]
    assert _anchor(full_model, waves) > 40


# ---- finite contexts
def _schedule(n_streams, seed):
    """Per stream: (open tick, close tick, pieces of about 0.37 s); ticks are step() calls."""
    from reazonspeech_b200.synth import synth_clip
    rng = random.Random(seed)
    out = []
    for i in range(n_streams):
        w = synth_clip(100 + i, rng.uniform(1.0, 6.0)).astype(np.float32)
        sizes, pos = [], 0
        while pos < len(w):
            k = rng.choice([5920, 5920, 3000, 12000])
            sizes.append(w[pos:pos + k]); pos += k
        out.append((rng.randint(0, 4), sizes))
    return out


def _run_schedule(model, config, sched, which, max_batch):
    """Run the streams ``which`` of ``sched`` on one transcriber: at tick k every open stream gets its next piece (closing after
    the last), then step().  -> per stream (result, per-step subwords, rows of its steps)."""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    model.max_batch = max_batch
    st = StreamingTranscriber(model, config, max_streams=len(which))
    sid, nxt, finals, rows, done = {}, {i: 0 for i in which}, {i: [] for i in which}, {i: [] for i in which}, {}
    tick = 0
    while len(done) < len(which):
        for i in which:
            t_open, pieces = sched[i]
            if tick == t_open:
                sid[i] = st.open()
            if i in sid and nxt[i] < len(pieces):
                st.feed(sid[i], pieces[nxt[i]]); nxt[i] += 1
                if nxt[i] == len(pieces):
                    st.close(sid[i])
        plan = dict(st.plan())
        for i, s in sid.items():
            if s in plan:
                rows[i].append(plan[s])
        for s, subs in st.step().items():
            finals[next(i for i, x in sid.items() if x == s)].append(subs)
        for i in [i for i, s in sid.items() if st.done(s)]:
            done[i] = st.result(sid.pop(i))
        tick += 1
        assert tick < 10000
    return {i: (done[i], finals[i], rows[i]) for i in which}


def test_finite_context_batched_equals_one_at_a_time_and_oracle(tiny_cfg, tiny_sd):
    from oracle import nemo_restated as O
    from reazonspeech_b200.nemo.asr import load_model
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg)
    config = StreamingConfig()
    sched = _schedule(7, seed=2)
    batched = _run_schedule(model, config, sched, list(range(7)), max_batch=3)
    n_tok = n_dec = 0
    for i in range(7):
        alone = _run_schedule(model, config, sched, [i], max_batch=1)[i]
        got = batched[i]
        assert got[0].text == alone[0].text and got[0].subwords == alone[0].subwords and got[0].segments == alone[0].segments, f"stream {i}"
        assert got[1] == alone[1] and got[2] == alone[2], f"stream {i}: steps"
        assert len(got[2]) > 1
        # every step's buffer through the GPU encoder, the kernel's decisions walked through the oracle's carried-state decoder
        eng = model.engine
        padded = np.concatenate([np.zeros(PAD_SAMPLES, np.float32)] + list(sched[i][1]) + [np.zeros(PAD_SAMPLES, np.float32)])
        state = None
        for row in got[2]:
            x = torch.from_numpy(padded[row.a:row.b].copy())[None].cuda()
            with torch.no_grad():
                enc, enc_len = eng.encode(*eng.log_mel(x, torch.tensor([x.shape[1]], dtype=torch.int32, device="cuda")))
                ep = O.joint_enc_proj(enc[0].cpu(), tiny_sd)
            lo, hi = row.dec_begin + row.offset, row.dec_end + row.offset
            toks = [t for t, f in zip(_tokens(got), _frames(got)) if lo <= f < hi]
            frs = [f - row.offset for f in _frames(got) if lo <= f < hi]
            gaps, state = follow_resume(ep, tiny_sd, tiny_cfg, row.dec_begin, row.dec_end, toks, frs, state)
            assert all(g[3] < NEAR_TIE for g in gaps), f"stream {i} rows {row}: {gaps[:3]}"
            n_dec += row.dec_end - row.dec_begin
        n_tok += len(_tokens(got))
    assert n_tok > 20 and n_dec > 100


def _tokens(got):
    return got[0].hypothesis.y_sequence.tolist()[1:]


def _frames(got):
    return [ts - i - 1 for i, ts in enumerate(got[0].hypothesis.timestamp)]


# ---- table changes with streams open
def test_table_change_restarts_from_root(tiny_cfg, tiny_engine, tiny_lm_tables):
    eng = tiny_engine
    enc, lens = _enc(tiny_cfg, [60, 52, 64], seed=21)
    _set_tables(eng, None, None)
    tk, _, nt = [a.cpu() for a in eng.greedy(enc, lens)]
    phr = [tk[b, i:i + 2].tolist() for b in range(3) for i in range(0, max(int(nt[b]) - 2, 0), 3)]
    tab_a = build_tables(PhraseBoostingConfig(phr[0::2], 3.0), tiny_cfg.vocab_size)
    tab_b = build_tables(PhraseBoostingConfig(phr[1::2], 3.0), tiny_cfg.vocab_size)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    mid = [int(n) // 2 for n in lens.tolist()]
    try:
        for word, first, then, root in ((1, (tab_a, None), (tab_b, None), 0), (2, (None, tiny_lm_tables), (tab_b, tiny_lm_tables), tiny_lm_tables.start_state)):
            states = torch.zeros(3, eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
            _set_tables(eng, *first)
            eng.greedy_resume(enc, i32([0, 0, 0]), i32(mid), i32([0, 1, 2]), states)
            changed, ref = states.clone(), states.clone()
            changed.view(torch.int32)[:, word] = -1                    # what a table change writes into open records
            ref.view(torch.int32)[:, word] = root
            _set_tables(eng, *then)
            a = [x.cpu() for x in eng.greedy_resume(enc, i32(mid), lens.cpu(), i32([0, 1, 2]), changed)]
            b = [x.cpu() for x in eng.greedy_resume(enc, i32(mid), lens.cpu(), i32([0, 1, 2]), ref)]
            assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(changed, ref), f"word {word}"
    finally:
        _set_tables(eng, None, None)
    # the model writes -1 into the open streams' records when its tables change
    from reazonspeech_b200.nemo.asr import StreamingTranscriber, load_model
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg)
    st = StreamingTranscriber(model, max_streams=3)
    s0, s1 = st.open(), st.open()
    model.set_phrase_boosting(PhraseBoostingConfig(phr[:4], 2.0))
    words = st.states.view(torch.int32)
    assert words[s0, 1] == -1 and words[s1, 1] == -1 and words[2, 1] == 0
