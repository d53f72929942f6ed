"""Phrase boosting (context biasing) of the greedy decode: the caller lists key phrases, and hypotheses that spell them get a
bonus of ``score`` (lambda, in logit units) per token -- NeMo's "boosting tree" idea (R), stated here as an Aho-Corasick
automaton over the phrase trie and applied inside the decode kernel (csrc/decode_spec.cu, kBoost).

Semantics.  The state after tokens y_1..y_t is n_t, the longest suffix of y_1..y_t that is a prefix of some phrase; delta(n, k)
is the goto / failure transition.  For a trie node n: D(n) = length of the longest prefix of n that is a phrase (0 if none),
f(n) = |n| - D(n) (provisional credit of the unfinished part of the match), O(m) = sum of |p| over the phrases p that are
suffixes of m (the phrases the token leading to m completes), g(m) = O(m) + f(m).  Emitting non-blank token k from state n adds

    beta(n, k) = lambda * (g(delta(n, k)) - f(n))

to token k's logit; blank is never boosted.  Summed along a hypothesis the bonus is lambda * (sum over completed phrase
occurrences of |p| + f(n_t)): a completed occurrence keeps lambda per token, an open partial match holds provisional credit,
and a partial match that breaks gives its credit back (beta can be negative).  The phrase list is a set: a phrase listed twice
counts once.  Every utterance starts at the root in every call; the state advances only on emissions.

Tables: ``bonus`` f32 and ``next`` i32, both [n_states, pitch] over the vocab_size non-blank columns, pitch = vocab_size
rounded up to a multiple of 4 (rows copy in 16-byte pieces); columns >= vocab_size are zero.  beta is computed in fp32 as
float32(lambda) * float32(g - f), the entries the kernel and the tests' oracle both add.  At most MAX_STATES trie nodes."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Hashable, List, Optional, Sequence, Tuple, Union

import numpy as np

MAX_STATES = 8192          # include/rs_engine.h RS_MAX_BOOST_STATES

Phrase = Union[str, Sequence[int]]


@dataclass
class PhraseBoostingConfig:
    """``phrases``: text (tokenised with the model's tokenizer, ``text_to_ids``) or token-id sequences; ``score``: lambda > 0,
    the bonus per phrase token in logit (nat) units."""
    phrases: List[Phrase] = field(default_factory=list)
    score: float = 2.0

    def validate(self) -> "PhraseBoostingConfig":
        if not (isinstance(self.score, (int, float)) and math.isfinite(self.score) and self.score > 0):
            raise ValueError(f"phrase boosting score must be finite and > 0, got {self.score!r}")
        return self


@dataclass
class PhraseBoostingTables:
    bonus: np.ndarray          # float32 [n_states, pitch]
    next: np.ndarray           # int32 [n_states, pitch]
    f: np.ndarray              # int64 [n_states] provisional credit |n| - D(n) of every state
    g: np.ndarray              # int64 [n_states] O(n) + f(n)

    @property
    def n_states(self) -> int:
        return int(self.bonus.shape[0])

    @property
    def pitch(self) -> int:
        return int(self.bonus.shape[1])


def phrase_ids(cfg: PhraseBoostingConfig, vocab_size: int, tokenizer=None) -> List[List[int]]:
    """The phrases as token-id lists, validated: non-empty, ids in [0, vocab_size)."""
    out = []
    for p in cfg.phrases:
        if isinstance(p, str):
            if tokenizer is None:
                raise ValueError(f"phrase {p!r} is text but no tokenizer was given")
            ids = list(tokenizer.text_to_ids(p))
        else:
            ids = [int(i) for i in p]
        if len(ids) == 0:
            raise ValueError(f"phrase {p!r} tokenises to nothing")
        bad = [i for i in ids if not 0 <= i < vocab_size]
        if bad:
            raise ValueError(f"phrase {p!r}: token ids {bad} outside [0, {vocab_size}) (blank is never part of a phrase)")
        out.append(ids)
    return out


def build_tables(cfg: PhraseBoostingConfig, vocab_size: int, tokenizer=None) -> PhraseBoostingTables:
    """Trie + failure links -> the dense tables (module docstring).  Raises ValueError on an invalid config."""
    cfg.validate()
    phrases = phrase_ids(cfg, vocab_size, tokenizer)
    # trie: node 0 is the root
    children: List[dict] = [{}]
    depth, is_end = [0], [False]
    for ids in phrases:
        n = 0
        for k in ids:
            c = children[n].get(k)
            if c is None:
                c = len(children)
                children.append({}); depth.append(depth[n] + 1); is_end.append(False)
                children[n][k] = c
                if len(children) > MAX_STATES:
                    raise ValueError(f"the phrases need more than {MAX_STATES} automaton states (about 2000 four-token phrases; "
                                     f"the tables would take {2 * 4 * MAX_STATES * _pitch(vocab_size) / 1e6:.0f} MB at "
                                     f"vocab_size {vocab_size})")
            n = c
        is_end[n] = True
    S, pitch = len(children), _pitch(vocab_size)
    nxt = np.zeros((S, pitch), np.int32)
    out = np.zeros(S, np.int64)              # O(n)
    fail = np.zeros(S, np.int64)
    last_end = np.zeros(S, np.int64)         # D(n)
    order = [0]
    for k, c in children[0].items():
        nxt[0, k] = c
    i = 0
    while i < len(order):                    # breadth first: fail(n) and its row are done before n's
        n = order[i]; i += 1
        if n != 0:
            nxt[n, :vocab_size] = nxt[fail[n], :vocab_size]
            for k, c in children[n].items():
                nxt[n, k] = c
        for k, c in children[n].items():
            fail[c] = nxt[fail[n], k] if n != 0 else 0
            last_end[c] = depth[c] if is_end[c] else last_end[n]
            out[c] = (depth[c] if is_end[c] else 0) + out[fail[c]]
            order.append(c)
    f = np.asarray(depth, np.int64) - last_end
    g = out + f
    bonus = np.zeros((S, pitch), np.float32)
    bonus[:, :vocab_size] = (g[nxt[:, :vocab_size]] - f[:, None]).astype(np.float32) * np.float32(cfg.score)
    return PhraseBoostingTables(bonus, nxt, f, g)


def config_key(cfg: Optional[PhraseBoostingConfig]) -> Hashable:
    """A hashable identity of a phrase list: configs with equal phrases (in order) and score build equal tables."""
    if cfg is None:
        return None
    return (tuple(p if isinstance(p, str) else tuple(int(i) for i in p) for p in cfg.phrases), float(cfg.score))


def combine_tables(lists: Sequence[Optional[PhraseBoostingConfig]], vocab_size: int, tokenizer=None,
                   base: Optional[PhraseBoostingConfig] = None) -> Tuple[PhraseBoostingTables, List[int]]:
    """Several phrase lists in one table, for decoding each row of a batch against its own list (rs_set_boost_roots) ->
    (tables, one root per entry of ``lists``).

    Region 0 holds ``base`` (the model's global list; with none, the 1-state empty automaton, whose bonus is zero).  Each
    distinct list follows in its own region: ``build_tables(list)`` with ``next`` offset by the region's start in the columns
    below vocab_size.  A row starting at its region's root never leaves that region, so it decodes exactly as it would with
    its list set alone.  Identical lists (``config_key``) share a region; a ``None`` entry means the global list, root 0.

    Memory: 8 * pitch bytes per state on the device (bonus f32 + next i32), about 24 KB at vocab_size 3000; the whole table
    may hold at most MAX_STATES states and raises ValueError beyond (there is no silent splitting)."""
    distinct = {config_key(c): c for c in lists if c is not None}
    regions = [build_tables(base if base is not None else PhraseBoostingConfig(), vocab_size, tokenizer)]
    regions += [build_tables(c, vocab_size, tokenizer) for c in distinct.values()]
    tables, starts = stack_tables(regions, vocab_size, len(distinct))
    start = dict(zip(distinct, starts[1:]))
    return tables, [0 if c is None else start[config_key(c)] for c in lists]


def stack_tables(regions: Sequence[PhraseBoostingTables], vocab_size: int, n_lists: Optional[int] = None
                 ) -> Tuple[PhraseBoostingTables, List[int]]:
    """Tables already built by ``build_tables`` laid one after another, ``next`` of each offset by its start in the columns
    below vocab_size (the inputs are not modified) -> (tables, start of every region).  Raises ValueError beyond MAX_STATES
    (``n_lists``: the number of distinct lists named in the message, default all regions but the first)."""
    sizes = [t.n_states for t in regions]
    if sum(sizes) > MAX_STATES:
        n = len(regions) - 1 if n_lists is None else n_lists
        raise ValueError(f"the {n} distinct phrase lists need {sum(sizes)} automaton states together with the "
                         f"global list's region, more than {MAX_STATES}; pass fewer or shorter lists per call")
    starts = np.cumsum([0] + sizes[:-1]).tolist()
    nxt = np.concatenate([t.next for t in regions])
    for at, size in zip(starts[1:], sizes[1:]):
        nxt[at:at + size, :vocab_size] += at
    tables = PhraseBoostingTables(np.concatenate([t.bonus for t in regions]), nxt, np.concatenate([t.f for t in regions]),
                                  np.concatenate([t.g for t in regions]))
    return tables, starts


def _pitch(vocab_size: int) -> int:
    return (vocab_size + 3) // 4 * 4


def load_phrases(path: str) -> List[str]:
    """A UTF-8 phrase file: one phrase per line, surrounding whitespace stripped, blank lines ignored."""
    with open(path, encoding="utf-8") as fh:
        return [line.strip() for line in fh if line.strip()]
