"""Phrase boosting without a GPU: the automaton tables against brute-force string matching, their shapes and validation,
``text_to_ids``, the boosted oracle with an empty table, the CLI options and load_model's argument checks."""
import math

import numpy as np
import pytest
import torch

from boosting_oracle import brute_force_bonus, greedy_boosted
from reazonspeech_b200.boosting import MAX_STATES, PhraseBoostingConfig, build_tables, load_phrases
from reazonspeech_b200.tokenizer import WORD_BOUNDARY, PieceTableTokenizer, synthetic_pieces


def _walk(tables, stream):
    total, state = 0.0, 0
    for k in stream:
        total += float(tables.bonus[state, k])
        state = int(tables.next[state, k])
    return total, state


@pytest.mark.parametrize("seed", range(6))
def test_tables_match_brute_force(seed):
    """Random small phrase sets over a small alphabet (prefix / suffix phrases, duplicates, single tokens all occur) and
    random token streams: the bonus summed along the stream equals lambda * (completed |p| + f(n_t))."""
    rng = np.random.default_rng(seed)
    V = 6 + seed
    for trial in range(150):
        n_phr = int(rng.integers(0, 7))
        phrases = [list(rng.integers(0, 4, int(rng.integers(1, 5)))) for _ in range(n_phr)]
        if phrases and trial % 3 == 0:
            p = phrases[0]
            phrases += [p[: max(1, len(p) - 1)], p[1:] or p, list(p), [p[-1]]]     # prefix, suffix, duplicate, single token
        score = 2.0 if trial % 2 == 0 else float(rng.uniform(0.1, 5.0))
        tables = build_tables(PhraseBoostingConfig([[int(x) for x in p] for p in phrases], score), V)
        for _ in range(8):
            stream = [int(x) for x in rng.integers(0, 5, int(rng.integers(0, 25)))]
            got, state = _walk(tables, stream)
            ref = brute_force_bonus(phrases, stream, score)
            assert math.isclose(got, ref, rel_tol=1e-5, abs_tol=1e-4), (phrases, stream, got, ref)
            if score == 2.0:
                assert got == ref                                      # exact: integer multiples of a power of two


def test_known_automaton():
    """Phrases [1 2 3] and [2 3 4], lambda 1: stream 1 2 3 4 completes both (3 + 3); 1 2 5 gives the partial match back."""
    t = build_tables(PhraseBoostingConfig([[1, 2, 3], [2, 3, 4]], 1.0), 8)
    assert _walk(t, [1, 2, 3, 4])[0] == 6.0
    assert _walk(t, [1, 2])[0] == 2.0 and _walk(t, [1, 2, 5])[0] == 0.0
    st = _walk(t, [1, 2])[1]
    assert t.bonus[st, 5] == -2.0 and t.bonus[st, 3] == 1.0


def test_shapes_pitch_and_empty_list():
    for V in (5, 8, 127, 3000):
        t = build_tables(PhraseBoostingConfig([[0, 1], [V - 1]], 1.5), V)
        assert t.pitch == (V + 3) // 4 * 4 and t.pitch % 4 == 0 and t.pitch >= V
        assert t.bonus.dtype == np.float32 and t.next.dtype == np.int32 and t.bonus.shape == t.next.shape == (4, t.pitch)
        assert np.all(t.bonus[:, V:] == 0) and np.all(t.next[:, V:] == 0)
        assert t.next.min() >= 0 and t.next.max() < t.n_states
    e = build_tables(PhraseBoostingConfig([], 3.0), 3000)
    assert e.n_states == 1 and e.pitch == 3000 and np.all(e.bonus == 0) and np.all(e.next == 0)


def test_validation_errors():
    with pytest.raises(ValueError, match="score"):
        build_tables(PhraseBoostingConfig([[1]], 0.0), 10)
    for bad in (-1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="score"):
            PhraseBoostingConfig([[1]], bad).validate()
    with pytest.raises(ValueError, match="tokenises to nothing"):
        build_tables(PhraseBoostingConfig([[]], 1.0), 10)
    tok = PieceTableTokenizer(synthetic_pieces(100))
    with pytest.raises(ValueError, match="tokenises to nothing"):
        build_tables(PhraseBoostingConfig([""], 1.0), 100, tok)
    for ids in ([10], [-1], [3, 11]):
        with pytest.raises(ValueError, match="outside"):
            build_tables(PhraseBoostingConfig([ids], 1.0), 10)
    with pytest.raises(ValueError, match="no tokenizer"):
        build_tables(PhraseBoostingConfig(["あ"], 1.0), 100)
    # 2048 four-token phrases without a shared prefix: 1 + 8192 states, one past the cap
    many = [[a, 1, 2, 3] for a in range(2048)]
    with pytest.raises(ValueError, match=f"more than {MAX_STATES}.*MB"):
        build_tables(PhraseBoostingConfig(many, 1.0), 3000)
    assert build_tables(PhraseBoostingConfig(many[:-1] + [[2047, 1, 2]], 1.0), 3000).n_states == MAX_STATES


def test_text_to_ids_piece_table():
    tok = PieceTableTokenizer(synthetic_pieces(3000))
    ids = tok.text_to_ids("あい")
    assert tok.ids_to_pieces(ids) == ["あ", "い"]                        # the leading lone boundary piece is dropped
    assert tok.ids_to_pieces(tok.text_to_ids("あ い")) == ["あ", WORD_BOUNDARY, "い"]
    assert tok.ids_to_text(tok.text_to_ids("一丁、七")) == "一丁、七"
    with pytest.raises(ValueError, match="no piece covers"):
        tok.text_to_ids("abc")
    longest = PieceTableTokenizer(["⁇", WORD_BOUNDARY, "あ", "あい", WORD_BOUNDARY + "う"])
    assert longest.text_to_ids("あいあ") == [3, 2] and longest.text_to_ids("う") == [4]   # a boundary fused into a piece stays


def test_load_phrases(tmp_path):
    p = tmp_path / "phrases.txt"
    p.write_text("東京\n\n  大阪 \n\n", encoding="utf-8")
    assert load_phrases(str(p)) == ["東京", "大阪"]


def test_oracle_empty_table_equals_rnnt_greedy(tiny_cfg, tiny_sd):
    from oracle import nemo_restated as O
    e = build_tables(PhraseBoostingConfig([], 2.0), tiny_cfg.vocab_size)
    g = torch.Generator().manual_seed(7)
    for T in (1, 9, 30):
        enc = torch.randn(T, tiny_cfg.d_model, generator=g)
        ref = O.rnnt_greedy(enc, tiny_sd, tiny_cfg, emulate=True)
        got = greedy_boosted(enc, tiny_sd, tiny_cfg, e.bonus, e.next)
        assert got.tokens == ref.tokens and got.frames == ref.frames and got.decisions == ref.decisions
        assert got.margins == ref.margins and got.changed == 0


def test_oracle_boosting_changes_decisions(tiny_cfg, tiny_sd):
    """A single-token phrase with a large bonus: the oracle emits it max_symbols times on every frame."""
    k = 5
    t = build_tables(PhraseBoostingConfig([[k]], 1e4), tiny_cfg.vocab_size)
    enc = torch.randn(6, tiny_cfg.d_model, generator=torch.Generator().manual_seed(8))
    got = greedy_boosted(enc, tiny_sd, tiny_cfg, t.bonus, t.next)
    assert got.tokens == [k] * 6 * tiny_cfg.max_symbols


def test_cli_options_parse():
    from reazonspeech_b200.nemo.asr.cli import parse
    o = parse(["--phrases=p.txt", "--phrase-score=3.5", "a.wav"])
    assert o.phrases == "p.txt" and o.phrase_score == 3.5 and o.audio == ["a.wav"]
    o = parse(["a.wav"])
    assert o.phrases is None and o.phrase_score is None


def test_load_model_rejects_boosting_with_alsd():
    from reazonspeech_b200.nemo import asr
    with pytest.raises(ValueError, match="greedy"):
        asr.load_model(synthetic=True, decoding="alsd", boosting=PhraseBoostingConfig([[1]], 2.0))
    with pytest.raises(ValueError, match="score"):
        asr.load_model(synthetic=True, boosting=PhraseBoostingConfig([[1]], -1.0))
