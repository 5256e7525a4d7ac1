"""Speaker names and ids of a multi-speaker corpus (DESIGN.md section 25).

    python -m fastspeech2_b200.speakers tag IN OUT [--map speakers.json]
    python -m fastspeech2_b200.speakers average --filelist F --spemb-dir D -o OUT
    python -m fastspeech2_b200.speakers embed --checkpoint embedding_model.ckpt -d WAV_DIR -o SPEMB_DIR [--budget SAMPLES]
                                              [--math-mode M]

`tag` appends the speaker name as a sixth `|` field to every line of the filelist IN and writes OUT, plus the map
{name: id} (default: speakers.json beside OUT).  The speaker name is the wav name up to its first `_`, which fits VCTK's
`p225_003.wav` and LibriTTS's `19_198_000000_000000.wav`.  A line that already carries a sixth field keeps it.  The
reference's `TTSDataset` reads fields 0-4 by index and ignores the rest, so the tagged filelist still trains a
single-speaker model on the reference's loader.  Ids are the sorted names numbered 0 .. n-1, so the same set of speakers
always gives the same map; `hp.model.n_speakers` is its length.

`average` (DESIGN.md section 27) writes one `{speaker}.npy` per speaker of the filelist F to OUT: the mean of that
speaker's L2-normalised utterance embeddings `{D}/{id}.npy` (id = the wav name up to its first dot), float32 [D].  This is
ESPnet2's usual way to synthesize a speaker from several recordings: pass the result as `spemb=`.

`embed` (DESIGN.md section 28) writes one float32 [D] `{id}.npy` per wav of WAV_DIR (id = the wav name up to its first
dot, the rule of `preprocess` and `FilelistDataset(spemb_dir=)`): SpeechBrain's ECAPA-TDNN embedding of the utterance, on
the library's kernels (`fastspeech2_b200.ecapa`), in batches of at most --budget padded samples.  Files at another rate
than 16 kHz are resampled on the GPU with the library's resampler (`preprocess --resample`'s, librosa 0.7's kaiser_best
semantics), not torchaudio's, so their embeddings differ from a SpeechBrain user's in that step.
"""
from __future__ import annotations

import argparse
import json
import os
from typing import Dict, Iterable, List, Optional

import numpy as np

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


def average(filelist: str, spemb_dir: str, out_dir: Optional[str] = None) -> Dict[str, np.ndarray]:
    """{speaker: mean of the speaker's normalised utterance embeddings}, float32 [D], summed in float64 in filelist order;
    each written to `{out_dir}/{speaker}.npy` when out_dir is given."""
    from .data import load_spemb
    sums: Dict[str, np.ndarray] = {}
    counts: Dict[str, int] = {}
    for ln in read_filelist(filelist):
        e = load_spemb(os.path.join(spemb_dir, ln.id + ".npy")).astype(np.float64)
        if not np.isfinite(e).all():
            raise ValueError(f"{ln.wav}: its speaker embedding holds non-finite values")
        e = e / max(float(np.linalg.norm(e)), 1e-12)
        name = speaker_of(ln)
        if name in sums and sums[name].shape != e.shape:
            raise ValueError(f"{ln.wav}: a [{e.shape[0]}] embedding, but speaker {name} has [{sums[name].shape[0]}] ones")
        sums[name] = sums[name] + e if name in sums else e
        counts[name] = counts.get(name, 0) + 1
    out = {name: (sums[name] / counts[name]).astype(np.float32) for name in sorted(sums)}
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        for name, e in out.items():
            np.save(os.path.join(out_dir, name + ".npy"), e)
    return out


def embed(checkpoint, wav_dir: str, out_dir: str, budget: int = 1 << 24, math_mode: str = "3xf16", device="cuda",
          log=print) -> int:
    """Write `{out_dir}/{id}.npy` for every wav of wav_dir; returns how many were written."""
    import glob

    import torch

    from .ecapa import SAMPLE_RATE, ECAPAEncoder
    from .preprocess import batches, gpu_resampler
    enc = ECAPAEncoder.from_checkpoint(checkpoint, math_mode=math_mode)
    resample = gpu_resampler(device)
    paths = sorted(glob.glob(os.path.join(wav_dir, "*.wav")))
    if not paths:
        raise ValueError(f"{wav_dir}: no .wav files")
    os.makedirs(out_dir, exist_ok=True)
    n = 0
    for rate, items in batches(paths, SAMPLE_RATE, budget, resample=True):
        ids = [i for i, _ in items]
        wavs = [w for _, w in items]
        if rate != SAMPLE_RATE:
            wavs = resample(wavs, rate, SAMPLE_RATE)
        for i, w in zip(ids, wavs):
            if len(w) < enc.min_samples:
                raise ValueError(f"{i}: {len(w)} samples at 16 kHz, the encoder needs at least {enc.min_samples}")
        x = np.zeros((len(wavs), max(len(w) for w in wavs)), dtype=np.float32)
        for b, w in enumerate(wavs):
            x[b, : len(w)] = w
        e = enc(torch.from_numpy(x).to(device), torch.tensor([len(w) for w in wavs], device=device)).cpu().numpy()
        for b, i in enumerate(ids):
            np.save(os.path.join(out_dir, i + ".npy"), e[b].astype(np.float32))
        n += len(ids)
        log(f"embed: {n} / {len(paths)}")
    return n


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(prog="python -m fastspeech2_b200.speakers", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    t = sub.add_parser("tag", help="append the speaker field to every line and write the speaker map")
    t.add_argument("src", help="filelist in the reference's five-field format")
    t.add_argument("dst", help="filelist to write")
    t.add_argument("--map", default=None, help="speaker map to write (default: speakers.json beside dst)")
    a = sub.add_parser("average", help="write each speaker's mean normalised embedding as {speaker}.npy")
    a.add_argument("--filelist", required=True, help="filelist whose utterances are averaged (the speaker field or wav name)")
    a.add_argument("--spemb-dir", required=True, help="directory of {id}.npy utterance embeddings")
    a.add_argument("-o", "--out", required=True, help="directory to write {speaker}.npy to")
    e = sub.add_parser("embed", help="write each wav's ECAPA-TDNN speaker embedding as {id}.npy")
    e.add_argument("--checkpoint", required=True, help="SpeechBrain's embedding_model.ckpt (spkrec-ecapa-voxceleb)")
    e.add_argument("-d", "--wav-dir", required=True, help="directory of .wav files (any rate; resampled to 16 kHz on the GPU)")
    e.add_argument("-o", "--out", required=True, help="directory to write {id}.npy to")
    e.add_argument("--budget", type=int, default=1 << 24, help="padded samples per batch (default 2^24)")
    e.add_argument("--math-mode", default="3xf16", help="fp32, tf32, 3xf16 or f16 (default 3xf16)")
    args = ap.parse_args(argv)
    if args.cmd == "embed":
        n = embed(args.checkpoint, args.wav_dir, args.out, args.budget, args.math_mode, log=lambda m: None)
        print(json.dumps({"embedded": n, "out": args.out}))
        return
    if args.cmd == "average":
        means = average(args.filelist, args.spemb_dir, args.out)
        print(json.dumps({"speakers": len(means), "out": args.out}))
        return
    mapping = tag(args.src, args.dst, args.map)
    print(json.dumps({"speakers": len(mapping), "filelist": args.dst}))


if __name__ == "__main__":
    main()
