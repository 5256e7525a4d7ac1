"""iSTFTNet windows on the H100 (ISTFTNetVocoder.window / stream / forward(chunk_frames=), fs2_istftnet_window): every
window is bit-identical to the same samples of the whole call in every math mode, including windows that start at an
utterance's first frame (the reflected row) and end at its last (the short envelope), empty windows, and the lockstep
chunks of forward(chunk_frames=k)."""
import pytest
import torch

from fastspeech2_b200.istftnet import HOP, ISTFTNetVocoder
from test_gpu_istftnet import MODES, OLENS, _calibrated_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mels():
    gen = torch.Generator().manual_seed(3)
    return (torch.randn(len(OLENS), max(OLENS), 80, generator=gen) * 2 - 6).cuda()


@pytest.fixture(scope="module")
def vocs(mels):
    sd = {k: v.detach().float().cpu() for k, v in _calibrated_oracle(mels.cpu(), OLENS).state_dict().items()}
    out = {}
    for m in MODES:
        v = ISTFTNetVocoder("v1", math_mode=m)
        v.load_state_dict(sd)
        out[m] = v.cuda().eval()
    return out


# per utterance (olens 37, 1, 160, 5, 64, 17, 161): starts at the first frame, inside, at the last frame, past the end
STARTS = [[0, 0, 0, 0, 0, 0, 0], [3, 0, 17, 4, 33, 16, 150], [36, 1, 129, 2, 63, 9, 157], [30, 0, 155, 0, 60, 13, 140]]


@pytest.mark.parametrize("mode", MODES)
def test_windows_are_bit_identical_to_the_whole_call(vocs, mels, mode):
    v = vocs[mode]
    ol = torch.tensor(OLENS).cuda()
    whole, _ = v(mels, ol)
    for n in (1, 7, 32):
        for starts in STARTS:
            audio, alens = v.window(mels, ol, starts, n)
            for b, (s, L) in enumerate(zip(starts, OLENS)):
                k = max(0, min(s + n, L) - s) * HOP
                assert int(alens[b]) == k
                assert torch.equal(audio[b, :k], whole[b, s * HOP: s * HOP + k]), (mode, n, b, s)
                assert torch.all(audio[b, k:].view(torch.int32) == 0), (mode, n, b, s)


@pytest.mark.parametrize("mode", MODES)
def test_chunked_forward_and_stream_equal_forward(vocs, mels, mode):
    v = vocs[mode]
    ol = torch.tensor(OLENS).cuda()
    whole, alens = v(mels, ol)
    for k in (1, 7, 32):
        got, gl = v(mels, ol, chunk_frames=k)
        assert torch.equal(got, whole) and torch.equal(gl, alens), (mode, k)
        chunks = torch.cat([a for a, _ in v.stream(mels, ol, k)], 1)
        assert torch.equal(chunks, whole), (mode, k)


def test_window_reads_no_mel_frame_outside_its_halo(vocs, mels):
    """NaN in every mel frame outside [c0 - h_0, c1 + h_0) changes no bit of the window."""
    v = vocs["3xf16"]
    h0 = v.window_plan()["halo"][0]
    ol = torch.tensor(OLENS).cuda()
    c0, n = 70, 16
    ref, _ = v.window(mels, ol, c0, n)
    m = mels.clone()
    m[:, : c0 - h0] = float("nan")
    m[:, c0 + n + h0:] = float("nan")
    got, _ = v.window(m, ol, c0, n)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))


def test_bad_starts_raise(vocs, mels):
    with pytest.raises(ValueError, match="starts"):
        vocs["3xf16"].window(mels, torch.tensor(OLENS).cuda(), torch.tensor([0, 0, -1, 0, 0, 0, 0]).cuda(), 8)
