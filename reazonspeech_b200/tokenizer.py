"""Tokenizers exposing NeMo's ``tokenizer.ids_to_text`` (the only tokenizer call the reference
makes: pkg/nemo-asr/src/decode.py:41,47).

``SentencePieceTokenizer`` wraps a real ``tokenizer.model`` from the .nemo archive.
``PieceTableTokenizer`` is the stand-in used with synthetic weights: a deterministic table of
3000 pieces decoded with SentencePiece's rules (concatenate pieces, U+2581 -> space, drop the
leading space) so a bare U+2581 decodes to the empty string exactly like the real model does
(which is why decode.py:51-53 filters empty tokens)."""
from __future__ import annotations

from typing import Iterable, List, Sequence

WORD_BOUNDARY = "▁"


class PieceTableTokenizer:
    def __init__(self, pieces: Sequence[str]):
        self.pieces = list(pieces)

    @property
    def vocab_size(self) -> int:
        return len(self.pieces)

    def ids_to_text(self, ids: Iterable[int]) -> str:
        text = "".join(self.pieces[int(i)] for i in ids).replace(WORD_BOUNDARY, " ")
        return text[1:] if text.startswith(" ") else text

    def ids_to_pieces(self, ids: Iterable[int]) -> List[str]:
        return [self.pieces[int(i)] for i in ids]


def synthetic_pieces(vocab_size: int) -> List[str]:
    """Deterministic Japanese-looking piece table: <unk>, the word-boundary mark, punctuation,
    kana, then CJK ideographs from U+4E00."""
    pieces = ["⁇", WORD_BOUNDARY, "。", "、", "?", "!", ","]
    pieces += [chr(c) for c in range(0x3041, 0x3094)]       # hiragana
    pieces += [chr(c) for c in range(0x30A1, 0x30F7)]       # katakana
    c = 0x4E00
    while len(pieces) < vocab_size:
        pieces.append(chr(c))
        c += 1
    return pieces[:vocab_size]


class SentencePieceTokenizer:
    def __init__(self, model_bytes: bytes):
        import sentencepiece as spm
        self.sp = spm.SentencePieceProcessor(model_proto=model_bytes)

    @property
    def vocab_size(self) -> int:
        return self.sp.get_piece_size()

    def ids_to_text(self, ids: Iterable[int]) -> str:
        return self.sp.decode_ids([int(i) for i in ids])

    def ids_to_pieces(self, ids: Iterable[int]) -> List[str]:
        return [self.sp.id_to_piece(int(i)) for i in ids]
