"""Phrase boosting per row on the CPU: the combined table of several lists (boosting.combine_tables), its region sharing and
state cap, the boosted oracle run per row on the combined table against each row alone, and the stream-record remap."""
import numpy as np
import pytest
import torch

from boosting_oracle import greedy_boosted
from reazonspeech_b200.boosting import MAX_STATES, PhraseBoostingConfig, build_tables, combine_tables, config_key


def _random_list(V, n, seed, max_len=4, score=2.0):
    rng = np.random.default_rng(seed)
    return PhraseBoostingConfig([[int(x) for x in rng.integers(0, V, int(rng.integers(1, max_len + 1)))] for _ in range(n)], score)


def _regions(tables, roots):
    """root -> (start, size) from the distinct roots and the table's state count"""
    starts = sorted(set(roots) | {0}) + [tables.n_states]
    return {r: (r, starts[starts.index(r) + 1] - r) for r in set(roots) | {0}}


@pytest.mark.parametrize("seed", range(5))
@pytest.mark.parametrize("with_base", [False, True])
def test_regions_equal_their_own_tables(seed, with_base):
    V = 129
    rng = np.random.default_rng(seed)
    lists = [_random_list(V, int(rng.integers(1, 30)), seed=100 * seed + i, score=float(rng.uniform(0.5, 4))) for i in range(6)]
    base = _random_list(V, 10, seed=999) if with_base else None
    tables, roots = combine_tables(lists, V, base=base)
    assert tables.pitch == build_tables(lists[0], V).pitch
    regions = _regions(tables, roots)
    ref0 = build_tables(base if base is not None else PhraseBoostingConfig(), V)
    assert regions[0] == (0, ref0.n_states)
    assert np.array_equal(tables.bonus[:ref0.n_states], ref0.bonus) and np.array_equal(tables.next[:ref0.n_states], ref0.next)
    for cfg, r in zip(lists, roots):
        ref = build_tables(cfg, V)
        start, size = regions[r]
        assert size == ref.n_states and start == r
        assert np.array_equal(tables.bonus[start:start + size], ref.bonus)
        assert np.array_equal(tables.next[start:start + size, :V], ref.next[:, :V] + start)
        assert np.array_equal(tables.f[start:start + size], ref.f) and np.array_equal(tables.g[start:start + size], ref.g)
        assert (tables.next[start:start + size, :V] >= start).all() and (tables.next[start:start + size, :V] < start + size).all()
    assert tables.n_states == ref0.n_states + sum(build_tables(c, V).n_states for c in lists)


def test_duplicates_share_a_region_and_none_is_root_0():
    V = 64
    a, b = _random_list(V, 8, seed=1), _random_list(V, 5, seed=2)
    a_again = PhraseBoostingConfig([list(p) for p in a.phrases], a.score)
    tables, roots = combine_tables([a, None, b, a_again, None, b], V)
    assert roots[1] == roots[4] == 0
    assert roots[0] == roots[3] == 1 and roots[2] == roots[5] == 1 + build_tables(a, V).n_states
    assert tables.n_states == 1 + build_tables(a, V).n_states + build_tables(b, V).n_states
    assert not tables.bonus[0].any() and not tables.next[0].any()          # no global list: the empty automaton
    # the same phrases at another score are a different list
    assert config_key(a) != config_key(PhraseBoostingConfig(a.phrases, a.score * 2))
    only_none, roots = combine_tables([None, None], V)
    assert only_none.n_states == 1 and roots == [0, 0]


def test_state_cap():
    """The cap counts every region, region 0 included: exactly MAX_STATES states build, one more raises."""
    V = 32
    singles = lambda toks: PhraseBoostingConfig([[t] for t in toks], 1.0)
    # 20 one-token phrases and one unique three-token phrase: 24 states per list
    lists = [PhraseBoostingConfig([[t] for t in range(20)] + [[31, i % 31, i // 31]], 1.0) for i in range((MAX_STATES - 1) // 24)]
    assert {build_tables(c, V).n_states for c in lists} == {24}
    room = MAX_STATES - 1 - 24 * len(lists)
    assert room >= 2
    tables, _ = combine_tables(lists + [singles(range(room - 1))] + lists[:3], V)
    assert tables.n_states == MAX_STATES
    with pytest.raises(ValueError, match=f"the {len(lists) + 1} distinct phrase lists need {MAX_STATES + 1} automaton states"):
        combine_tables(lists + [singles(range(room))], V)


def _tiny_enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    return enc, lens


def test_oracle_with_roots_equals_each_row_alone(tiny_cfg, tiny_sd):
    """The boosted oracle walked from each row's root on the combined table gives every row exactly its solo decode."""
    V = tiny_cfg.vocab_size
    enc, lens = _tiny_enc(tiny_cfg, [23, 9, 30, 17], seed=5)
    lists = [_random_list(V, 12, seed=11), None, _random_list(V, 6, seed=12, score=3.0), _random_list(V, 12, seed=11)]
    base = _random_list(V, 4, seed=13)
    tables, roots = combine_tables(lists, V, base=base)
    n_changed = 0
    for b, (cfg, r) in enumerate(zip(lists, roots)):
        alone = build_tables(cfg if cfg is not None else base, V)
        solo = greedy_boosted(enc[b, :lens[b]], tiny_sd, tiny_cfg, alone.bonus, alone.next)
        rowed = greedy_boosted(enc[b, :lens[b]], tiny_sd, tiny_cfg, *_start_at(tables, r))
        assert (rowed.tokens, rowed.frames, rowed.decisions) == (solo.tokens, solo.frames, solo.decisions), f"row {b}"
        n_changed += solo.changed
    assert n_changed > 0


def _start_at(tables, root):
    """The combined table with states 0 and ``root`` swapped, so that the oracle, which starts every row at state 0, starts at
    ``root``: a relabelling of the states that leaves every transition and bonus as it was."""
    p = np.arange(tables.n_states)
    p[[0, root]] = p[[root, 0]]
    nxt = p[tables.next[p]]
    return tables.bonus[p], nxt


def test_stream_record_remap_is_exact():
    from reazonspeech_b200.nemo.asr.streaming import remap_boost_states
    # per record: its list's old region [old_start, old_start + old_size) and new start; (100, 0): a list new to the layout
    old_start = torch.tensor([0, 0, 40, 40, 40, 7, 7, 100, 0], dtype=torch.int32)
    old_size = torch.tensor([7, 7, 60, 60, 60, 33, 33, 0, 0], dtype=torch.int32)
    new_start = torch.tensor([0, 0, 5, 5, 5, 90, 90, 12, 0], dtype=torch.int32)
    state = torch.tensor([3, -1, 40, 99, 100, 39, 6, 100, 5], dtype=torch.int32)
    got = remap_boost_states(state, old_start, old_size, new_start)
    assert got.tolist() == [3, 0, 5, 64, 5, 122, 90, 12, 0]
    assert got.dtype == torch.int32


class _RootsStub:
    """A stand-in engine for the streaming host layer: records the table and roots of every step, and leaves each decoded
    row's boost_state one state past its root (a partial match) -- the record word the next layout change must move."""

    def __init__(self, cfg):
        self.cfg, self.device, self.stream_state_bytes = cfg, torch.device("cpu"), 64
        self._boost, self.roots, self.steps = None, None, []

    def set_phrase_boosting(self, bonus, next_state=None):
        self._boost = None if bonus is None else (torch.as_tensor(bonus), torch.as_tensor(next_state))
        self.roots = None

    def set_boost_roots(self, roots):
        self.roots = list(roots)

    def stream_step(self, wav, lens, dec_begin, dec_end, slot, states, U, out, alpha=None):
        words = states.view(torch.int32)
        self.steps.append((None if self._boost is None else int(self._boost[0].shape[0]), self.roots, slot.tolist(),
                           words[slot.long(), 1].tolist()))
        for r, s in enumerate(slot.tolist()):
            words[s, 0] = 1
            if self.roots is not None:
                words[s, 1] = self.roots[r] + 1
        out[2][:wav.shape[0]] = 0
        return out


def test_stream_lists_follow_their_region(tiny_cfg):
    """Streams with their own lists share one table; when a list leaves, the others' records move to their new region with
    their partial match, and streams on the global list keep state 0's region."""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    V = tiny_cfg.vocab_size
    eng = _RootsStub(tiny_cfg)
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(V)), max_batch=4)
    st = StreamingTranscriber(model, max_streams=4)
    a, b = _random_list(V, 6, seed=50), _random_list(V, 9, seed=51)
    na, nb = build_tables(a, V).n_states, build_tables(b, V).n_states
    s0, s1, s2 = st.open(boosting=a), st.open(), st.open(boosting=b)
    for s in (s0, s1, s2):
        st.feed(s, np.zeros(40000, np.float32))
    st.step()
    n_states, roots, slots, _ = eng.steps[-1]
    assert n_states == 1 + na + nb and roots == [1, 0, 1 + na] and slots == [s0, s1, s2]
    assert eng._boost is None                                          # the global setting is back after the step
    st.close(s0)
    while not st.done(s0):
        st.step()
    n_before = len(eng.steps)
    st.feed(s1, np.zeros(100000, np.float32)); st.feed(s2, np.zeros(100000, np.float32))
    st.step()                                                          # a's region is gone: b moves down to 1
    assert len(eng.steps) == n_before + 1
    n_states, roots, slots, words = eng.steps[-1]
    assert n_states == 1 + nb and roots == [0, 1] and slots == [s1, s2]
    # s2's partial match (its old root + 1) moved with it; s1's word 1 lay outside the 1-state empty region 0: its root
    assert words == [0, 2]


def test_stream_lists_rejected_at_open_leave_the_others_stepping(tiny_cfg):
    """A list with a bad token id or text that tokenises to nothing, and a list that would take the open streams' lists past
    MAX_STATES, raise in open() and take no slot; a global list that would not fit is refused by set_phrase_boosting with
    nothing changed.  The streams already open keep stepping to the end."""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    V = tiny_cfg.vocab_size
    eng = _RootsStub(tiny_cfg)
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(V)), max_batch=4)
    st = StreamingTranscriber(model, max_streams=3)
    big = PhraseBoostingConfig([[i % V, i // V] for i in range(MAX_STATES - 600)], 1.0)       # most of the cap
    good = st.open(boosting=big)
    n_big = build_tables(big, V).n_states
    for bad, why in ((PhraseBoostingConfig([[V + 5]], 1.0), "outside"), (PhraseBoostingConfig([""], 1.0), "tokenises to nothing"),
                     (PhraseBoostingConfig([[a, b] for a in range(V) for b in range(5)], 1.0), "more than 8192")):
        with pytest.raises(ValueError, match=why):
            st.open(boosting=bad)
    assert st.open_streams == [good]
    glob = PhraseBoostingConfig([[a, b] for a in range(V) for b in range(6)], 1.0)             # more than the room left
    assert 1 + n_big <= MAX_STATES < build_tables(glob, V).n_states + n_big
    with pytest.raises(ValueError, match="global list is unchanged"):
        model.set_phrase_boosting(glob)
    assert model.boosting is None and eng._boost is None
    other = st.open()
    for s in (good, other):
        st.feed(s, np.zeros(40000, np.float32))
        st.close(s)
    for _ in range(50):
        st.step()
        if st.done(good) and st.done(other):
            break
    assert st.done(good) and st.done(other) and eng.steps
    assert eng.steps[0][0] == 1 + n_big and eng.steps[0][1] == [1, 0]
