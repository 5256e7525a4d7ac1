#!/usr/bin/env python
"""Generate tests/golden/align_filelist.npz from the reference's LJSpeech filelist (build container only):

    python tests/golden/make_golden_align.py [path/to/train_filelist.txt]

Stores the first 1,024 lines' phoneme strings, their MFA durations and wav names: data only, no code.  The GPU tests
render a synthetic corpus from them (tests/test_gpu_aligner.py) and never read the reference."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
N_LINES = 1024


def main(argv):
    src = argv[1] if len(argv) > 1 else os.path.join(HERE, "..", "..", "oracle", "_ref", "filelists", "train_filelist.txt")
    with open(src, encoding="utf-8") as f:
        lines = [ln.rstrip("\n").split("|") for ln in f][:N_LINES]
    phonemes = [ln[3].strip() for ln in lines]
    durs = [np.array(ln[2].split(), dtype=np.int64) for ln in lines]
    assert all(len(d) == len(p.split()) for d, p in zip(durs, phonemes))
    np.savez_compressed(os.path.join(HERE, "align_filelist.npz"),
                        phonemes=np.array(phonemes), wavs=np.array([ln[4].strip() for ln in lines]),
                        durations=np.concatenate(durs).astype(np.int16),
                        offsets=np.cumsum([0] + [len(d) for d in durs]).astype(np.int64))


if __name__ == "__main__":
    main(sys.argv)
