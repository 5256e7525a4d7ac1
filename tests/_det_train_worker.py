"""Run by tests/test_gpu_train_deterministic.py in a fresh process: three deterministic train steps of one configuration,
printing the SHA-256 of the resulting state.  `python tests/_det_train_worker.py <precision> <attention> <n_speakers>`"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_gpu_train_deterministic as G  # noqa: E402

if __name__ == "__main__":
    prec, att, n_spk = sys.argv[1], sys.argv[2], int(sys.argv[3])
    print(G.digest(G.three_steps(prec, att, n_spk, det=True)))
