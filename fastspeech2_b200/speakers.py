"""Speaker names and ids of a multi-speaker corpus (DESIGN.md section 25).

    python -m fastspeech2_b200.speakers tag IN OUT [--map speakers.json]

`tag` appends the speaker name as a sixth `|` field to every line of the filelist IN and writes OUT, plus the map
{name: id} (default: speakers.json beside OUT).  The speaker name is the wav name up to its first `_`, which fits VCTK's
`p225_003.wav` and LibriTTS's `19_198_000000_000000.wav`.  A line that already carries a sixth field keeps it.  The
reference's `TTSDataset` reads fields 0-4 by index and ignores the rest, so the tagged filelist still trains a
single-speaker model on the reference's loader.  Ids are the sorted names numbered 0 .. n-1, so the same set of speakers
always gives the same map; `hp.model.n_speakers` is its length.
"""
from __future__ import annotations

import argparse
import json
import os
from typing import Dict, Iterable, List, Optional

from .aligner import Line, parse_line, read_filelist


def speaker_from_wav(name: str) -> str:
    """The speaker of a wav name: the text before the first `_` (the whole stem when there is none)."""
    stem = os.path.basename(name).split(".")[0]
    spk = stem.split("_", 1)[0]
    if not spk:
        raise ValueError(f"{name!r}: no speaker name before the first '_'")
    return spk


def speaker_of(line: Line) -> str:
    """A line's speaker: its sixth field, else derived from its wav name."""
    return line.speaker if line.speaker is not None else speaker_from_wav(line.wav)


def build_map(lines: Iterable[Line]) -> Dict[str, int]:
    """{speaker name: id}, names sorted, ids 0 .. n-1."""
    return {name: i for i, name in enumerate(sorted({speaker_of(ln) for ln in lines}))}


def save_map(path: str, mapping: Dict[str, int]) -> None:
    with open(path, "w", encoding="utf-8") as fh:
        json.dump(dict(sorted(mapping.items(), key=lambda kv: kv[1])), fh, indent=1)
        fh.write("\n")


def load_map(path: str) -> Dict[str, int]:
    """A map written by `save_map`; its ids must be exactly 0 .. n-1."""
    with open(path, encoding="utf-8") as fh:
        mapping = json.load(fh)
    if not isinstance(mapping, dict) or sorted(mapping.values()) != list(range(len(mapping))) or \
            not all(isinstance(v, int) and not isinstance(v, bool) for v in mapping.values()):
        raise ValueError(f"{path}: not a speaker map (ids must be the ints 0 .. n-1)")
    return {str(k): int(v) for k, v in mapping.items()}


def tag_line(raw: str, where: str = "line") -> str:
    """One raw filelist line with its speaker field (unchanged when it has one)."""
    ln = parse_line(raw, where)
    body = raw.rstrip("\r\n")
    return body if ln.speaker is not None else body + "|" + speaker_from_wav(ln.wav)


def tag(src: str, dst: str, map_path: Optional[str] = None) -> Dict[str, int]:
    """Write the six-field filelist of `src` to `dst` and the speaker map to `map_path`; returns the map."""
    with open(src, encoding="utf-8") as fh:
        raw = [(i, ln) for i, ln in enumerate(fh) if ln.strip()]
    tagged: List[str] = [tag_line(ln, f"{src}:{i + 1}") for i, ln in raw]
    mapping = build_map(parse_line(ln) for ln in tagged)
    with open(dst, "w", encoding="utf-8") as fh:
        fh.write("".join(ln + "\n" for ln in tagged))
    save_map(map_path or os.path.join(os.path.dirname(os.path.abspath(dst)), "speakers.json"), mapping)
    return mapping


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(prog="python -m fastspeech2_b200.speakers", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    t = sub.add_parser("tag", help="append the speaker field to every line and write the speaker map")
    t.add_argument("src", help="filelist in the reference's five-field format")
    t.add_argument("dst", help="filelist to write")
    t.add_argument("--map", default=None, help="speaker map to write (default: speakers.json beside dst)")
    args = ap.parse_args(argv)
    mapping = tag(args.src, args.dst, args.map)
    print(json.dumps({"speakers": len(mapping), "filelist": args.dst}))


if __name__ == "__main__":
    main()
