"""Command line of the drop-in package: ``python -m reazonspeech_b200.nemo.asr.cli [options] AUDIO [AUDIO ...]``.

Same contract as the reference's ``reazonspeech-nemo-asr`` entry point (pkg/nemo-asr/src/cli.py:36-74):

  -h / --help          usage on stderr, nothing else happens
  -o FILE / --output=  where the transcript goes (default: stdout)
  --to=FMT             vtt | srt | ass | json | tsv; anything else, or no option, gives the bracketed plain-text
                       lines.  Like the reference, the format is NOT inferred from FILE's extension
                       (see writer.get_writer)
  no AUDIO argument    "no audio file specified" + usage on stderr, exit status 1
  unknown option       getopt.GetoptError propagates, as in the reference

First extension: several AUDIO arguments are transcribed as one batch on the GPU (the reference reads exactly one);
their segments are written one file after the other through the same writer, every file's times shifted by the total
duration of the files before it, i.e. the transcript of the files played back to back (subtitle formats need monotonic times).
Second extension, phrase boosting (reazonspeech_b200/boosting.py): the greedy decode favours hypotheses that spell key phrases
  --phrases=FILE       UTF-8 text, one phrase per line (blank lines ignored)
  --phrase-score=L     bonus per phrase token in logit units, L > 0 (default 2.0; alone, without --phrases, it boosts nothing)
With neither option the output is unchanged.
Third extension, n-gram LM shallow fusion (reazonspeech_b200/ngram_lm.py): the greedy decode adds alpha * ln(10) * log10 P(k | h)
of an ARPA LM over BPE token ids (words chr(token id + 100)) to every non-blank logit
  --lm=FILE            the ARPA file
  --lm-alpha=A         the LM weight, A > 0; required with --lm (there is no default)
With neither option the output is unchanged.
Fourth extension, forced alignment of known transcripts (reazonspeech_b200/alignment.py): instead of transcribing, each AUDIO is
aligned to its given transcript and the segments are written through the same writer with the same time offsets
  --text=FILE          UTF-8 text, one transcript line per AUDIO argument, in order (a count mismatch is an error)
  --band=SECONDS       long-form alignment (reazonspeech_b200/longform.py) of the one AUDIO argument: FILE is its whole
                       transcript (the non-blank lines are joined), aligned in a band of SECONDS around the recording's greedy
                       transcript (4 is the library's default; not calibrated).  Needs --text and exactly one AUDIO argument
Without the option the output is unchanged.
Fifth extension, streaming (reazonspeech_b200/streaming.py): the one AUDIO argument is decoded chunk by chunk as a live stream
  --stream             AUDIO is a file, or - for raw 16-bit little-endian 16 kHz mono PCM on stdin; every chunk's final
                       text goes to stderr as "[start seconds] text" as soon as it is decoded, and at the end the usual
                       output (--to, -o) is written from the whole stream
  --chunk=S --left=S --right=S   chunk and context seconds (multiples of 0.08; default 1.6, 1.2, 1.2)
Without the option the output is unchanged.
Sixth extension, caption alignment (reazonspeech_b200/captions.py): the captions of the one AUDIO argument are located in
its audio, each inside the window [start - before, end + after), and written as segments through the same writer
  --captions=FILE      UTF-8 lines start<TAB>end<TAB>text in seconds, the format --to=tsv writes (its header line is skipped)
  --before=S --after=S the window's margins in seconds (default 25 and 0: live captions trail the speech by about 25 s)
Captions that cannot be located (an empty window, or no token) are skipped.  Without the option the output is unchanged.
Seventh extension, beam search: the decoding strategy of the transcription
  --decoding=D         greedy (default) | alsd (NeMo's ALSD beam search) | maes (NeMo's modified adaptive expansion search
                       with its default parameters, or the checkpoint's maes_* settings); --lm / --lm-alpha fuse the LM into
                       maes as into greedy; alsd takes no LM, no phrases; neither beam search streams
  --beam=N             beam size of alsd / maes (default 4; maes: 1..8)
Without the options the output is unchanged.
Eighth extension, keyword spotting (reazonspeech_b200/keywords.py): instead of transcribing, every occurrence of each keyword is
searched in each AUDIO on the RNN-T lattice, and the hits are written as segments (text = the keyword, sorted by start)
through the same writer with the same time offsets
  --keywords=FILE      UTF-8 text, one keyword per line (blank lines ignored)
  --keyword-threshold=X  the least mean per-frame log-probability of a hit (default -1.0; not calibrated, see keywords.py)
  --max-hits=N         at most N hits per keyword per AUDIO, 1..256 (default 64)
It goes with none of --text, --captions, --stream, --decoding, --beam, --phrases, --phrase-score and --lm.  Without it the
output is unchanged.
Audio decoding: soundfile when installed, scipy for WAV, librosa for compressed containers, see audio.audio_from_path.
"""
import dataclasses
import getopt
import sys
import warnings
from dataclasses import dataclass, field
from typing import List, Optional

SHORT_OPTS = "ho:"
LONG_OPTS = ("help", "output=", "to=", "phrases=", "phrase-score=", "lm=", "lm-alpha=", "text=", "stream", "chunk=", "left=", "right=",
             "captions=", "before=", "after=", "decoding=", "beam=", "keywords=", "keyword-threshold=", "max-hits=", "band=")


@dataclass
class Options:
    help: bool = False
    output: Optional[str] = None
    fmt: Optional[str] = None
    audio: List[str] = field(default_factory=list)
    phrases: Optional[str] = None
    phrase_score: Optional[float] = None
    lm: Optional[str] = None
    lm_alpha: Optional[float] = None
    text: Optional[str] = None
    stream: bool = False
    chunk: float = 1.6
    left: float = 1.2
    right: float = 1.2
    captions: Optional[str] = None
    before: float = 25.0
    after: float = 0.0
    decoding: str = "greedy"
    beam: Optional[int] = None
    keywords: Optional[str] = None
    keyword_threshold: Optional[float] = None
    max_hits: Optional[int] = None
    band: Optional[float] = None


def parse(argv) -> Options:
    parsed, rest = getopt.getopt(list(argv), SHORT_OPTS, LONG_OPTS)
    opt = Options(audio=rest)
    for flag, value in parsed:
        if flag in ("-h", "--help"):
            opt.help = True
            break                                            # the reference returns at the first -h it meets
        if flag in ("-o", "--output"):
            opt.output = value
        if flag == "--to":
            opt.fmt = value
        if flag == "--phrases":
            opt.phrases = value
        if flag == "--phrase-score":
            opt.phrase_score = float(value)
        if flag == "--lm":
            opt.lm = value
        if flag == "--lm-alpha":
            opt.lm_alpha = float(value)
        if flag == "--text":
            opt.text = value
        if flag == "--stream":
            opt.stream = True
        if flag in ("--chunk", "--left", "--right", "--before", "--after"):
            setattr(opt, flag[2:], float(value))
        if flag == "--captions":
            opt.captions = value
        if flag == "--decoding":
            opt.decoding = value
        if flag == "--beam":
            opt.beam = int(value)
        if flag == "--keywords":
            opt.keywords = value
        if flag == "--keyword-threshold":
            opt.keyword_threshold = float(value)
        if flag == "--max-hits":
            opt.max_hits = int(value)
        if flag == "--band":
            opt.band = float(value)
    if (opt.lm is None) != (opt.lm_alpha is None):
        raise ValueError("--lm and --lm-alpha go together: the LM weight has no default (try values around 0.3-0.5 and tune "
                         "on held-out audio)" if opt.lm is not None else "--lm-alpha needs an LM: --lm=FILE")
    if opt.decoding not in ("greedy", "alsd", "maes"):
        raise ValueError(f"--decoding must be greedy, alsd or maes, got {opt.decoding!r}")
    if opt.beam is not None and (opt.decoding == "greedy" or opt.beam < 1):
        raise ValueError("--beam=N (N >= 1) sets the beam of --decoding=alsd or maes")
    if opt.decoding != "greedy":
        if opt.lm is not None and opt.decoding == "alsd":
            raise ValueError("--lm is fused into --decoding=greedy or maes, not alsd")
        if opt.phrases is not None or opt.phrase_score is not None:
            raise ValueError("--phrases boosts the greedy decode only")
        if opt.stream:
            raise ValueError("--stream decodes greedily")
    if opt.stream and len(opt.audio) > 1:
        raise ValueError("--stream decodes one AUDIO argument (a file, or - for PCM on stdin)")
    if opt.captions is not None:
        if len(opt.audio) > 1:
            raise ValueError("--captions locates the captions of one AUDIO argument")
        if opt.stream or opt.text is not None:
            raise ValueError("--captions goes with neither --stream nor --text")
        if opt.before < 0 or opt.after < 0:
            raise ValueError(f"--before and --after are margins in seconds >= 0, got {opt.before} and {opt.after}")
    if opt.band is not None:
        if opt.text is None:
            raise ValueError("--band=SECONDS aligns the whole transcript given by --text=FILE")
        if len(opt.audio) > 1:
            raise ValueError("--band aligns the transcript of one AUDIO argument")
        from ...longform import band_frames
        band_frames(opt.band)
    if opt.keywords is None:
        if opt.keyword_threshold is not None or opt.max_hits is not None:
            raise ValueError("--keyword-threshold and --max-hits set the search of --keywords=FILE")
    else:
        clash = [f for f, _ in parsed if f in ("--text", "--captions", "--stream", "--decoding", "--beam", "--phrases", "--phrase-score", "--lm")]
        if clash:
            raise ValueError(f"--keywords searches the audio on the lattice: it goes with none of {', '.join(sorted(set(clash)))}")
        from ...keywords import MAX_HITS, THRESHOLD, check_search
        check_search(THRESHOLD if opt.keyword_threshold is None else opt.keyword_threshold, MAX_HITS if opt.max_hits is None else opt.max_hits)
    return opt


def usage() -> None:
    print(__doc__, file=sys.stderr)


def load_transcripts(path: str, n_audio: int) -> List[str]:
    """--text: one UTF-8 transcript line per AUDIO argument; ValueError when the counts differ."""
    with open(path, encoding="utf-8") as f:
        lines = f.read().splitlines()
    if len(lines) != n_audio:
        raise ValueError(f"--text={path}: {len(lines)} transcript lines for {n_audio} AUDIO arguments")
    return lines


def load_long_transcript(path: str) -> str:
    """--text with --band: the whole transcript of one recording, its non-blank lines joined."""
    with open(path, encoding="utf-8") as f:
        return "".join(line.strip() for line in f.read().splitlines() if line.strip())


def run(opt: Options) -> None:
    from .audio import audio_from_path
    from .transcribe import align_batch, align_long, load_model, transcribe, transcribe_batch
    from .writer import get_writer

    texts = None
    if opt.text is not None:
        texts = [load_long_transcript(opt.text)] if opt.band is not None else load_transcripts(opt.text, len(opt.audio))
    captions = None
    if opt.captions is not None:
        from ...captions import read_captions_tsv
        captions = read_captions_tsv(opt.captions)
    sink = sys.stdout if opt.output is None else open(opt.output, "w")
    warnings.simplefilter("ignore")
    clips = [audio_from_path(path) for path in opt.audio] if not (opt.stream and opt.audio == ["-"]) else []
    boosting = None
    if opt.phrases is not None or opt.phrase_score is not None:
        from ...boosting import PhraseBoostingConfig, load_phrases
        boosting = PhraseBoostingConfig(load_phrases(opt.phrases) if opt.phrases is not None else [])
        if opt.phrase_score is not None:
            boosting.score = opt.phrase_score
    extra = {}
    if boosting is not None:
        extra["boosting"] = boosting
    if opt.lm is not None:
        from ...ngram_lm import NgramLMConfig
        extra["lm"] = NgramLMConfig(opt.lm, opt.lm_alpha)
    if opt.decoding != "greedy":
        extra["decoding"] = opt.decoding
        if opt.beam is not None:
            extra["beam_size"] = opt.beam
    model = load_model(**extra)
    if opt.keywords is not None:
        results = keyword_segments(model, clips, load_keywords(opt.keywords), opt)
    elif captions is not None:
        results = [caption_segments(model, clips[0], captions, opt)]
    elif opt.stream:
        results = [stream(model, opt, clips[0] if clips else None)]
    elif opt.band is not None:
        results = [align_long(model, clips[0], texts[0], band_seconds=opt.band)]
    elif texts is not None:
        results = align_batch(model, clips, texts)
    else:
        results = transcribe_batch(model, clips) if len(clips) > 1 else [transcribe(model, clips[0])]
    with sink:
        out = get_writer(sink, opt.fmt)
        out.write_header()
        offset = 0.0
        for k, result in enumerate(results):
            for segment in result.segments:
                out.write(segment if offset == 0.0 else
                          dataclasses.replace(segment, start_seconds=segment.start_seconds + offset, end_seconds=segment.end_seconds + offset))
            offset += clips[k].seconds if k < len(clips) else 0.0


def caption_segments(model, clip, captions, opt: Options):
    """--captions: the located captions as one result whose segments are (start, end, caption text), in caption order."""
    from .interface import Segment, TranscribeResult
    from .transcribe import align_captions
    found = [a for a in align_captions(model, clip, captions, before=opt.before, after=opt.after) if a is not None]
    return TranscribeResult("".join(a.text for a in found), [w for a in found for w in a.subwords],
                            [Segment(a.start_seconds, a.end_seconds, a.text) for a in found])


def load_keywords(path: str) -> List[str]:
    """--keywords: one UTF-8 keyword per line, blank lines skipped."""
    with open(path, encoding="utf-8") as f:
        return [line.strip() for line in f.read().splitlines() if line.strip()]


def keyword_segments(model, clips, keywords: List[str], opt: Options):
    """--keywords: for each clip one result whose segments are (start, end, keyword) of every hit, sorted by start."""
    from .interface import Segment, TranscribeResult
    from .transcribe import find_keywords_batch
    from ...keywords import MAX_HITS, THRESHOLD
    found = find_keywords_batch(model, clips, keywords, threshold=THRESHOLD if opt.keyword_threshold is None else opt.keyword_threshold,
                                max_hits=MAX_HITS if opt.max_hits is None else opt.max_hits)
    results = []
    for lists in found:
        hits = sorted((h for row in lists for h in row), key=lambda h: (h.start_seconds, h.end_seconds))
        results.append(TranscribeResult("".join(h.keyword for h in hits), [w for h in hits for w in h.subwords],
                                        [Segment(h.start_seconds, h.end_seconds, h.keyword) for h in hits]))
    return results


def stream(model, opt: Options, clip=None):
    """--stream: ``clip`` (a decoded file), or 16-bit PCM from stdin when None, fed to a StreamingTranscriber in 0.16 s pieces;
    each step's final text goes to stderr with its start time -> the stream's TranscribeResult."""
    import numpy as np
    from .audio import norm_audio
    from .streaming import StreamingTranscriber
    from ...streaming import StreamingConfig
    st = StreamingTranscriber(model, StreamingConfig(opt.chunk, opt.left, opt.right), max_streams=1)
    sid = st.open()
    piece = 2560

    def show(new):
        for subs in new.values():
            if subs:
                print(f"[{subs[0].seconds:.2f}] {''.join(s.token for s in subs)}", file=sys.stderr, flush=True)

    if clip is not None:
        wave = np.asarray(norm_audio(clip).waveform)
        wave = wave if wave.dtype == np.int16 else wave.astype(np.float32)
        for lo in range(0, len(wave), piece):
            st.feed(sid, wave[lo:lo + piece])
            show(st.step())
    else:
        raw = sys.stdin.buffer
        while True:
            data = raw.read(2 * piece)
            if not data:
                break
            st.feed(sid, np.frombuffer(data[: len(data) // 2 * 2], dtype="<i2").astype(np.int16))
            show(st.step())
    st.close(sid)
    while not st.done(sid):
        show(st.step())
    return st.result(sid)


def main(argv=None):
    opt = parse(sys.argv[1:] if argv is None else argv)
    if opt.help:
        usage()
        return None
    if not opt.audio:
        print("no audio file specified", file=sys.stderr)
        usage()
        return 1
    run(opt)
    return None


if __name__ == "__main__":
    sys.exit(main())
