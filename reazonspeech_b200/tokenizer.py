"""Tokenizers exposing NeMo's ``tokenizer.ids_to_text`` (the only tokenizer call the reference
makes: pkg/nemo-asr/src/decode.py:41,47).

``SentencePieceTokenizer`` wraps a real ``tokenizer.model`` from the .nemo archive.
``PieceTableTokenizer`` is the stand-in used with synthetic weights: a deterministic table of
3000 pieces decoded with SentencePiece's rules (concatenate pieces, U+2581 -> space, drop the
leading space) so a bare U+2581 decodes to the empty string exactly like the real model does
(which is why decode.py:51-53 filters empty tokens).

``text_to_ids`` (phrase boosting's tokenisation, boosting.py) segments a phrase ON ITS OWN, with the word-boundary piece that
SentencePiece puts in front of a text dropped when it stands alone: a phrase inside a Japanese sentence carries no word
boundary.  Known limitation: a phrase's segmentation alone may differ from its segmentation inside the sentences the model
transcribes, and then boosting the phrase's ids favours a spelling the model would not produce; pass token-id sequences
where that matters.

``sentence_to_ids`` (forced alignment's tokenisation, alignment.py) encodes a whole sentence the way the model's training
targets were encoded: SentencePiece's ``encode`` unchanged, the leading word-boundary piece kept."""
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

    def sentence_to_ids(self, text: str) -> List[int]:
        """Longest match over the pieces with SentencePiece's space handling (a leading boundary, spaces -> U+2581), the
        boundary piece kept.  A character no piece covers raises ValueError."""
        if not hasattr(self, "_index"):
            self._index = {}
            for i, piece in enumerate(self.pieces):
                self._index.setdefault(piece, i)
            self._longest = max((len(piece) for piece in self.pieces), default=1)
        s = WORD_BOUNDARY + text.replace(" ", WORD_BOUNDARY)
        ids, i = [], 0
        while i < len(s):
            for n in range(min(self._longest, len(s) - i), 0, -1):
                k = self._index.get(s[i:i + n])
                if k is not None:
                    ids.append(k); i += n
                    break
            else:
                raise ValueError(f"{text!r}: no piece covers {s[i]!r}")
        return ids

    def text_to_ids(self, text: str) -> List[int]:
        """Longest match over the pieces (SentencePiece's space handling: a leading boundary, spaces -> U+2581), a leading lone
        U+2581 piece dropped.  A character no piece covers raises ValueError."""
        ids = self.sentence_to_ids(text)
        return _drop_lone_boundary(ids, self.pieces[ids[0]] if ids else "")


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

    def sentence_to_ids(self, text: str) -> List[int]:
        """SentencePiece's ``encode`` unchanged (the leading U+2581 piece kept).  Text no piece covers raises ValueError."""
        ids = [int(i) for i in self.sp.encode(text)]
        if self.sp.unk_id() in ids:
            raise ValueError(f"{text!r}: not covered by the piece table (encodes to <unk>)")
        return ids

    def text_to_ids(self, text: str) -> List[int]:
        """SentencePiece's ``encode``, a leading lone U+2581 piece dropped."""
        ids = [int(i) for i in self.sp.encode(text)]
        return _drop_lone_boundary(ids, self.sp.id_to_piece(ids[0]) if ids else "")


def _drop_lone_boundary(ids: List[int], first_piece: str) -> List[int]:
    return ids[1:] if first_piece == WORD_BOUNDARY else ids
