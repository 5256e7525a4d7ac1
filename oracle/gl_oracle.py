"""CPU restatement of the batched vocoder's contract (fastspeech2_b200.vocoder.GriffinLimVocoder, DESIGN.md section 7) on
top of `oracle.stft_oracle.STFT`.  TEST INFRASTRUCTURE ONLY.

  mel inversion   M = max(0, P . exp(mel)), P = pinv(mel filterbank) in float64 rounded to float32; the filterbank is
                  torchaudio's `melscale_fbanks(norm="slaney", mel_scale="slaney")`, an implementation independent of
                  the package's numpy restatement of librosa 0.7 (the tests check the two agree)
  Griffin-Lim     per utterance over its own frames: y = ISTFT(M, angles); n_iters x { Z = STFT(y);
                  Zh = Z - momentum / (1 + momentum) * Z_prev (Z_prev = 0 at first); y = ISTFT(M, atan2(Zh)) }
                  -- with momentum = 0 exactly `stft_oracle.griffin_lim` (atan2 is scale-invariant, so the phase of
                  Zh is the phasor Zh / |Zh| the kernels use, and atan2(0, 0) = 0 gives (1, 0))."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.stft_oracle import STFT


def mel_inverse(sample_rate, n_fft, n_mels, fmin, fmax):
    import torchaudio.functional as TAF
    fb = TAF.melscale_fbanks(n_fft // 2 + 1, float(fmin), float(fmax), n_mels, sample_rate, norm="slaney", mel_scale="slaney").T
    return torch.from_numpy(np.linalg.pinv(fb.double().numpy()).astype(np.float32))          # [cutoff, n_mels]


def mel_to_magnitude(mel, P):
    """mel [frames, n_mels] -> M [cutoff, frames] (float32)."""
    return torch.relu(P @ torch.exp(mel.float()).T)


def spectrum(stft, y):
    """stft_oracle.STFT.transform without the magnitude / phase split: (re, im) [B, cutoff, frames]."""
    B, n = y.shape
    x = F.pad(y.view(B, 1, n).unsqueeze(1), (stft.filter_length // 2, stft.filter_length // 2, 0, 0), mode="reflect").squeeze(1)
    ft = F.conv1d(x, stft.forward_basis, stride=stft.hop_length, padding=0)
    cutoff = stft.filter_length // 2 + 1
    return ft[:, :cutoff, :], ft[:, cutoff:, :]


def griffin_lim(mag, stft, n_iters, angles, momentum=0.0):
    """mag, angles [1, cutoff, frames] -> signal [1, (frames-1)*hop]."""
    k = momentum / (1.0 + momentum)
    y = stft.inverse(mag, angles).squeeze(1)
    prev = None
    for _ in range(n_iters):
        re, im = spectrum(stft, y)
        if momentum and prev is not None:
            hre, him = re - k * prev[0], im - k * prev[1]
        else:
            hre, him = re, im
        prev = (re, im)
        y = stft.inverse(mag, torch.atan2(him, hre)).squeeze(1)
    return y


def vocode(mels, olens, n_iters, angles, momentum=0.0, sample_rate=22050, n_fft=1024, hop=256, win_length=1024, n_mels=80,
           fmin=0.0, fmax=8000.0):
    """mels [B, Lmax, n_mels], olens [B], angles [B, cutoff, Lmax] -> (audio [B, (Lmax-1)*hop], alens [B])."""
    P = mel_inverse(sample_rate, n_fft, n_mels, fmin, fmax)
    stft = STFT(n_fft, hop, win_length)
    B, L, _ = mels.shape
    audio = torch.zeros(B, (L - 1) * hop)
    alens = (torch.as_tensor(olens).long() - 1) * hop
    for b in range(B):
        n = int(olens[b])
        M = mel_to_magnitude(mels[b, :n], P)[None]
        audio[b, : (n - 1) * hop] = griffin_lim(M, stft, n_iters, angles[b: b + 1, :, :n].float(), momentum)[0]
    return audio, alens
