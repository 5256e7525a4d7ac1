"""Training-feature preprocessing on the GPU: what the reference's nvidia_preprocessing.py (and, with --stats,
compute_statistics.py) does, in batches of utterances.

    python -m fastspeech2_b200.preprocess -d WAV_DIR -c config.yaml [--stats] [-o DATA_DIR] [--budget SAMPLES]

Every `*.wav` under WAV_DIR (recursively) is read with the reference's `read_wav_np` rules and written as
  {data_dir}/mels/{id}.npy    float32 [n_mels, T]   log-mel (TacotronSTFT.mel_spectrogram)
  {data_dir}/energy/{id}.npy  float32 [T]           torch.norm(|STFT|, dim=0)
  {data_dir}/pitch/{id}.npy   float64 [plens]       pyworld.dio(...)[:T]
with T = N // hop + 1 and id the file name up to its first dot; data_dir is hp.data.data_dir unless -o is given.  Files
go to the GPU in batches whose padded size B * Nmax stays within --budget samples; the next batch is read while the GPU
works on the current one.  With --stats, e_mean / e_std / f0_mean / f0_std.npy (float32) are computed from the arrays
written, after the reference's in-place `remove_outlier`."""
from __future__ import annotations

import argparse
import glob
import os
import queue
import threading

import numpy as np

from .hparams import load_hp


def read_wav_np(path: str, sample_rate: int) -> np.ndarray:
    """utils/util.py:576-594 for a file at the configured rate: int16 / int32 / uint8 scaled to [-1, 1), the first channel
    of a multi-channel file, float32 (8-bit files are centred in float, where the reference's uint8 arithmetic wraps).
    The reference resamples other rates with librosa; here that is an error."""
    from scipy.io.wavfile import read
    sr, wav = read(path)
    if sr != sample_rate:
        raise ValueError(f"{path}: sample rate {sr} Hz, the config says {sample_rate} Hz (resample the file first)")
    if len(wav.shape) == 2:
        wav = wav[:, 0]
    if wav.dtype == np.int16:
        wav = wav / 32768.0
    elif wav.dtype == np.int32:
        wav = wav / 2147483648.0
    elif wav.dtype == np.uint8:
        wav = (wav.astype(np.float64) - 128) / 128.0     # in float: the reference's uint8 subtraction wraps around
    return wav.astype(np.float32)


def utterance_id(path: str) -> str:
    return os.path.basename(path).split(".")[0]


def batches(paths, sample_rate: int, budget: int):
    """Yield lists of (id, wav) whose padded size len * max(len(wav)) stays within `budget` samples (a longer file goes
    alone)."""
    cur, longest = [], 0
    for p in paths:
        w = read_wav_np(p, sample_rate)
        m = max(longest, len(w))
        if cur and (len(cur) + 1) * m > budget:
            yield cur
            cur, m = [], len(w)
        cur.append((utterance_id(p), w))
        longest = m
    if cur:
        yield cur


def gpu_backend(hp, device="cuda", math_mode="3xf16"):
    """extract(list of float32 wavs) -> list of (mel [n_mels, T], energy [T], pitch [plens]) on the library's kernels."""
    import torch

    from .features import FeatureExtractor
    fx = FeatureExtractor.from_hp(hp, math_mode=math_mode).to(device)

    def extract(wavs):
        n = [len(w) for w in wavs]
        x = np.zeros((len(wavs), max(n)), dtype=np.float32)
        for b, w in enumerate(wavs):
            x[b, : n[b]] = w
        mels, energy, flens, f0, plens = fx(torch.from_numpy(x).to(device), torch.tensor(n, device=device))
        mels, energy, flens, f0, plens = (t.cpu().numpy() for t in (mels, energy, flens, f0, plens))
        return [(mels[b, : flens[b]].T.copy(), energy[b, : flens[b]].copy(), f0[b, : plens[b]].copy()) for b in range(len(wavs))]
    return extract


def remove_outlier(x: np.ndarray) -> np.ndarray:
    """utils/util.py:26-49, in place: values on or outside the 1.5 IQR fences are set to 0, then to the maximum of the
    result; the original zeros are restored last."""
    p25, p75 = np.percentile(x, 25), np.percentile(x, 75)
    lower, upper = p25 - 1.5 * (p75 - p25), p75 + 1.5 * (p75 - p25)
    zero_idxs = np.where(x == 0.0)[0]
    out = [i for i, v in enumerate(x) if v <= lower or v >= upper]
    x[out] = 0.0
    x[out] = np.max(x)
    x[zero_idxs] = 0.0
    return x


def statistics(energies: dict, pitches: dict, log=print) -> dict:
    """compute_statistics.py on {id: energy} and {id: pitch}: remove_outlier on each (in place), then mean and std of the
    non-zero values.  Returns e_mean, e_std, f0_mean, f0_std (float32) and the ids whose pitch is all zero."""
    min_p, max_p, max_e, nz_min_p, nz_min_e = [], [], [], [], []
    e_vecs = []
    for k in energies:
        e = remove_outlier(energies[k])
        e_vecs.append(e)
        if np.any(e > 0):
            nz_min_e.append(e[e > 0].min())
        max_e.append(e.max())
    nz = np.concatenate([v[np.where(v != 0.0)[0]] for v in e_vecs])
    e_mean, e_std = np.mean(nz), np.std(nz)
    log("Non zero Min Energy : {}".format(min(nz_min_e) if nz_min_e else None))
    log("Max Energy : {}".format(max(max_e)))
    log("Energy mean : {}".format(e_mean))
    log("Energy std: {}".format(e_std))
    p_vecs, bad = [], []
    for k in pitches:
        p = remove_outlier(pitches[k])
        p_vecs.append(p)
        try:
            min_p.append(p.min())
            nz_min_p.append(p[p > 0].min())
            max_p.append(p.max())
        except ValueError:
            bad.append(k)
    nz = np.concatenate([v[np.where(v != 0.0)[0]] for v in p_vecs])
    f0_mean, f0_std = np.mean(nz), np.std(nz)
    log("Min Pitch : {}".format(min(min_p)))
    log("Non zero Min Pitch : {}".format(min(nz_min_p) if nz_min_p else None))
    log("Max Pitch : {}".format(max(max_p) if max_p else None))
    log("Pitch mean : {}".format(f0_mean))
    log("Pitch std: {}".format(f0_std))
    log("The len of bad Pitch Vectors is ", len(bad))
    for k in bad:
        log(k)
    return {"e_mean": e_mean.astype(np.float32), "e_std": e_std.astype(np.float32), "f0_mean": f0_mean.astype(np.float32),
            "f0_std": f0_std.astype(np.float32), "bad_pitch": bad}


def run(wav_dir: str, hp, data_dir: str = None, stats: bool = False, budget: int = 1 << 24, extract=None, log=print) -> dict:
    """Preprocess every wav under wav_dir; returns {"ids": [...], and the statistics when `stats`}.  `extract` replaces
    the GPU backend (a function from a list of wavs to a list of (mel, energy, pitch))."""
    if data_dir is None:
        data = hp["data"] if isinstance(hp, dict) else hp.data
        data_dir = data["data_dir"]
    sample_rate = int((hp["audio"] if isinstance(hp, dict) else hp.audio)["sample_rate"])
    paths = sorted(glob.glob(os.path.join(wav_dir, "**", "*.wav"), recursive=True))
    dirs = {k: os.path.join(data_dir, k) for k in ("mels", "energy", "pitch")}
    for d in dirs.values():
        os.makedirs(d, exist_ok=True)
    extract = extract or gpu_backend(hp)
    log("Sample Rate : ", sample_rate)
    # a reader thread keeps one batch ahead of the GPU
    q: queue.Queue = queue.Queue(maxsize=2)

    def reader():
        try:
            for bt in batches(paths, sample_rate, budget):
                q.put(bt)
            q.put(None)
        except BaseException as e:        # re-raised in the consumer
            q.put(e)
    th = threading.Thread(target=reader, daemon=True)
    th.start()
    ids, energies, pitches = [], {}, {}
    while True:
        bt = q.get()
        if bt is None:
            break
        if isinstance(bt, BaseException):
            raise bt
        for (uid, _), (mel, e, p) in zip(bt, extract([w for _, w in bt])):
            np.save(os.path.join(dirs["mels"], uid + ".npy"), mel.astype(np.float32), allow_pickle=False)
            np.save(os.path.join(dirs["energy"], uid + ".npy"), e.astype(np.float32), allow_pickle=False)
            np.save(os.path.join(dirs["pitch"], uid + ".npy"), p.astype(np.float64), allow_pickle=False)
            ids.append(uid)
            if stats:
                energies[uid], pitches[uid] = e.astype(np.float32), p.astype(np.float64)
    th.join()
    log(f"wrote {len(ids)} utterances to {data_dir}")
    out = {"ids": ids}
    if stats and ids:
        st = statistics(energies, pitches, log)
        for k in ("e_mean", "e_std", "f0_mean", "f0_std"):
            np.save(os.path.join(data_dir, k + ".npy"), st[k], allow_pickle=False)
        out.update(st)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("-d", "--data_path", required=True, help="root directory of wav files")
    ap.add_argument("-c", "--config", required=True, help="yaml file for configuration")
    ap.add_argument("-o", "--out", default=None, help="output directory (default: hp.data.data_dir)")
    ap.add_argument("--stats", action="store_true", help="also write e_mean / e_std / f0_mean / f0_std.npy")
    ap.add_argument("--budget", type=int, default=1 << 24, help="samples per GPU batch, padding included")
    args = ap.parse_args(argv)
    run(args.data_path, load_hp(args.config), args.out, args.stats, args.budget)


if __name__ == "__main__":
    main()
