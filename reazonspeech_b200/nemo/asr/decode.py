"""Hypothesis -> TranscribeResult.  Output-identical to the reference's decode_hypothesis
(pkg/nemo-asr/src/decode.py:28-66) on the same (y_sequence, timestamp) pair; pinned against the
reference module itself by tests/golden/decode_cases.json (tests/test_decode_golden.py).

The reference was written against NeMo's ALSD beam-search hypotheses: y_sequence carries a
leading blank (decode.py:38-40) and timestamp[i] counts decoder steps t+u, so the frame of token
i is timestamp[i] - i - 1 (decode.py:48).  The engine decodes greedily and presents its result
in that same shape (see transcribe.Hypothesis.from_greedy)."""
from __future__ import annotations

from typing import List, Optional, Sequence

from .interface import Segment, Subword, TranscribeResult

PAD_SECONDS = 0.5            # silence transcribe() adds on both sides       (decode.py:4)
SECONDS_PER_STEP = 0.08      # encoder frame period: 8 x 10 ms               (decode.py:5)
SUBWORDS_PER_SEGMENTS = 10   # soft minimum segment length                   (decode.py:6)
PHONEMIC_BREAK = 0.5         # pause that may end a segment                  (decode.py:7)

TOKEN_EOS = frozenset("。?!")
TOKEN_COMMA = frozenset("、,")
TOKEN_PUNC = TOKEN_EOS | TOKEN_COMMA


def token_seconds(step: int, index: int) -> float:
    """Time of token `index` whose ALSD step counter is `step` (decode.py:48)."""
    return max(SECONDS_PER_STEP * (step - index - 1) - PAD_SECONDS, 0)


def find_end_of_segment(subwords: Sequence[Subword], start: int) -> int:
    """Index of the last subword of the segment beginning at `start` (decode.py:13-26).

    A segment closes after a sentence-final mark, or -- once it holds more than
    SUBWORDS_PER_SEGMENTS subwords -- after a comma or ahead of a pause longer than
    PHONEMIC_BREAK; never directly ahead of a punctuation token."""
    last = len(subwords) - 1
    pos = start
    while pos < last:
        here, ahead = subwords[pos], subwords[pos + 1]
        if ahead.token not in TOKEN_PUNC:
            if here.token in TOKEN_EOS:
                return pos
            long_enough = pos - start >= SUBWORDS_PER_SEGMENTS
            if long_enough and (here.token in TOKEN_COMMA or ahead.seconds - here.seconds > PHONEMIC_BREAK):
                return pos
        pos += 1
    return max(last, start)


def build_result(tokenizer, token_ids: Sequence[int], steps: Sequence[int],
                 token_confidence: Optional[Sequence[float]] = None) -> TranscribeResult:
    """``token_confidence`` (one value per token id) is carried onto the subwords that are kept."""
    token_ids = [int(t) for t in token_ids]
    text = tokenizer.ids_to_text(token_ids)
    # ids_to_text([tid]) is a pure function of tid: remembered per tokenizer object (a 30 s clip asks ~100 times, a batched
    # run thousands of times per second -- with several GPUs behind one interpreter this loop is what they wait for)
    try:
        single = tokenizer.__dict__.setdefault("_single_id_text", {})
    except AttributeError:                          # an object without __dict__: no cache
        single = {}
    pieces: List[Subword] = []
    for index, (tid, step) in enumerate(zip(token_ids, steps)):
        piece = single.get(tid)
        if piece is None:
            piece = single[tid] = tokenizer.ids_to_text([tid])
        if piece:                                   # a bare word-boundary mark decodes to "" (decode.py:51-53)
            pieces.append(Subword(max(SECONDS_PER_STEP * (int(step) - index - 1) - PAD_SECONDS, 0), tid, piece,   # token_seconds, inlined
                                  None if token_confidence is None else float(token_confidence[index])))
    segments: List[Segment] = []
    begin = 0
    while begin < len(pieces):
        end = find_end_of_segment(pieces, begin)
        segments.append(Segment(start_seconds=pieces[begin].seconds,
                                end_seconds=pieces[end].seconds + SECONDS_PER_STEP,
                                text="".join(p.token for p in pieces[begin:end + 1])))
        begin = end + 1
    return TranscribeResult(text, pieces, segments)


def decode_hypothesis(model, hyp) -> TranscribeResult:
    """Same signature as the reference: `model` needs .tokenizer.ids_to_text, `hyp` needs
    .y_sequence (tensor-like with .tolist(), leading blank) and .timestamp; its .token_confidence, when present and not
    None, goes onto the subwords."""
    return build_result(model.tokenizer, hyp.y_sequence.tolist()[1:], list(hyp.timestamp), getattr(hyp, "token_confidence", None))
