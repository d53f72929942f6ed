"""n-gram LM fusion on the CPU: the tables and the kernel-emulating ``lookup`` against the brute-force ARPA oracle
(tests/ngram_oracle.py) on a handwritten fixture and on generated 2- to 5-gram LMs, the input validation, the API / CLI
rejections, and the decode kernel's register budget."""
import math
import os
import re
import subprocess

import numpy as np
import pytest

from ngram_oracle import ArpaOracle, write_arpa
from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables, lookup

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "ngram_small.arpa")


def _check_all_pairs(path, V, alpha):
    t = build_lm_tables(NgramLMConfig(path, alpha), V)
    o = ArpaOracle(path, V, alpha)
    assert set(t.contexts) == o.states
    sid = {c: s for s, c in enumerate(t.contexts)}
    S = t.n_states
    states = np.repeat(np.arange(S), V)
    tokens = np.tile(np.arange(V), S)
    score, nxt = lookup(t, states, tokens)
    worst = 0.0
    for s, k, sc, nx in zip(states.tolist(), tokens.tolist(), score.tolist(), nxt.tolist()):
        h = t.contexts[s]
        ref = o.score(h, k)
        worst = max(worst, abs(sc - ref))
        assert abs(sc - ref) <= 1e-5, (h, k, sc, ref)
        assert nx == sid[o.next(h, k)], (h, k, t.contexts[nx], o.next(h, k))
    return t, worst


def test_fixture_against_oracle():
    t, worst = _check_all_pairs(FIXTURE, 8, 0.7)
    assert t.order == 3 and t.start_state == t.contexts.index((8,))
    assert (6,) not in t.contexts and (4, 1) not in t.contexts    # no unigram / the trigram's absent bigram prefix
    s, k = lookup(t, 0, 6)                                        # token 6 has no unigram: <unk>'s probability
    assert abs(s - 0.7 * math.log(10) * -2.0) < 1e-6 and k == 0
    print(f"fixture: {t.n_states} states x 8 tokens, largest |score - oracle| {worst:.2e}")


@pytest.mark.parametrize("order", (2, 3, 4, 5))
def test_generated_against_oracle(tmp_path, order):
    path = str(tmp_path / f"lm{order}.arpa")
    n = write_arpa(path, 127, order, n_sentences=150, seed=order)
    t, worst = _check_all_pairs(path, 127, 0.45)
    assert t.order == order and t.n_arcs > 0
    print(f"{order}-gram: {n} n-grams, {t.n_states} states x 127 tokens, largest |score - oracle| {worst:.2e}")


def test_gap_arcs_follow_the_back_off_rule(tmp_path):
    """Bigrams 'k e' and 'd k' where k (token 7) has no unigram: in state (d, k) the back-off rule reaches the explicit 'k e'
    through the context (k,), which is no state.  The tables carry it as a gap arc on (d, k); scores and transitions match
    the oracle for every pair."""
    src = open(FIXTURE, encoding="utf-8").read()
    src = src.replace("ngram 2=9", "ngram 2=11").replace("\\2-grams:\n", "\\2-grams:\n-0.3\tk e\t-0.1\n-0.4\td k\t-0.2\n")
    p = tmp_path / "gap.arpa"
    p.write_text(src, encoding="utf-8")
    t, _ = _check_all_pairs(str(p), 8, 0.5)
    s = t.contexts.index((0, 7))
    assert int(t.backoff[s]) == 0 and (7,) not in t.contexts and (7, 1) in t.contexts
    arcs = dict(zip(t.arc_tok[t.arc_begin[s]:t.arc_begin[s + 1]].tolist(), t.arc_to[t.arc_begin[s]:t.arc_begin[s + 1]].tolist()))
    assert 1 in arcs and t.contexts[arcs[1]] == (7, 1)
    score, nxt = lookup(t, s, 1)
    assert abs(score - 0.5 * math.log(10) * (-0.2 - 0.3)) < 1e-5 and t.contexts[nxt] == (7, 1)


def _write(tmp_path, text, name="x.arpa"):
    p = tmp_path / name
    p.write_text(text, encoding="utf-8")
    return str(p)


BASE = "\\data\\\nngram 1=3\nngram 2=1\n\n\\1-grams:\n-1.0\td\t-0.2\n-1.0\te\n-2.0\t<unk>\n\n\\2-grams:\n-0.5\td e\n\n\\end\\\n"


def test_rejections(tmp_path):
    ok = _write(tmp_path, BASE)
    build_lm_tables(NgramLMConfig(ok, 0.5), 8)
    cases = {
        "bad count": BASE.replace("ngram 2=1", "ngram 2=2"),
        "missing end": BASE.replace("\\end\\\n", ""),
        "unknown word": BASE.replace("-0.5\td e", "-0.5\td zz"),
        "out of vocabulary": BASE.replace("-0.5\td e", "-0.5\td " + chr(100 + 8)),
        "no unk": BASE.replace("ngram 1=3", "ngram 1=2").replace("-2.0\t<unk>\n", ""),
    }
    for what, text in cases.items():
        with pytest.raises(ValueError) as ei:
            build_lm_tables(NgramLMConfig(_write(tmp_path, text), 0.5), 8)
        if what == "unknown word":
            assert "'zz'" in str(ei.value)
        if what == "out of vocabulary":
            assert repr(chr(108)) in str(ei.value)
    seven = "\\data\\\n" + "".join(f"ngram {n}=1\n" for n in range(1, 8)) + "\n\\1-grams:\n-1.0\t<unk>\n"
    for n in range(2, 8):
        seven += f"\n\\{n}-grams:\n-1.0\t" + " ".join(["d"] * n) + "\n"
    with pytest.raises(ValueError, match="order 7"):
        build_lm_tables(NgramLMConfig(_write(tmp_path, seven + "\n\\end\\\n"), 0.5), 8)
    for alpha in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="alpha"):
            build_lm_tables(NgramLMConfig(ok, alpha), 8)


def test_load_model_rejects_lm_with_alsd(tmp_path):
    from reazonspeech_b200.nemo import asr
    with pytest.raises(ValueError, match="greedy"):
        asr.load_model(synthetic=True, decoding="alsd", lm=NgramLMConfig(_write(tmp_path, BASE), 0.5))


def test_cli_lm_options():
    from reazonspeech_b200.nemo.asr.cli import parse
    opt = parse(["--lm=x.arpa", "--lm-alpha=0.4", "a.wav"])
    assert opt.lm == "x.arpa" and opt.lm_alpha == 0.4 and opt.audio == ["a.wav"]
    with pytest.raises(ValueError, match="--lm-alpha"):
        parse(["--lm=x.arpa", "a.wav"])
    with pytest.raises(ValueError, match="--lm"):
        parse(["--lm-alpha=0.4", "a.wav"])


def test_decode_kernel_registers_and_spills(tmp_path):
    """Every instance of the decode kernel is free of spills, and the instances without the LM keep their register counts."""
    from reazonspeech_b200.build import ARCH, CSRC, FLAGS, _nvcc
    r = subprocess.run([_nvcc(), *ARCH, *FLAGS, "-Xptxas", "-v", "-c", os.path.join(CSRC, "decode_spec.cu"), "-o", str(tmp_path / "d.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = {}
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '_ZN2rs23rnnt_greedy_spec_kernelILi(\d+)ELi\d+ELb(\d)ELb(\d)ELb(\d)E", line)
        if m:
            cur = (int(m.group(1)), m.group(2) == "1", m.group(3) == "1", m.group(4) == "1")
            continue
        if cur is None:
            continue
        if "spill" in line:
            assert "0 bytes spill stores, 0 bytes spill loads" in line and "0 bytes stack frame" in line, (cur, line)
        m = re.search(r"Used (\d+) registers", line)
        if m:
            found[cur] = int(m.group(1))
            cur = None
    assert len(found) == 16, found
    expect = {(640, False, False): 234, (640, True, False): 255, (128, False, False): 146, (128, True, False): 167,
              (640, False, True): 254, (640, True, True): 252, (128, False, True): 154, (128, True, True): 168}
    for (hj, conf, boost), regs in expect.items():
        assert found[(hj, conf, boost, False)] == regs, (hj, conf, boost, found)
    print("decode kernel registers (HJ, conf, boost, lm):", found)
