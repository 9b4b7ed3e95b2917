"""GPU: audio front / back ends on the device (SURVEY.md 8f-3) vs the CPU oracle (oracle/ref_audio.py, which restates
librosa.load's resampling via the published torchaudio definition, librosa.util.normalize and torchaudio.save's payload)."""
import numpy as np
import pytest
import torch

from megatts2_b200 import audio
from oracle import ref_audio

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda"


def gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


@pytest.mark.parametrize("orig", [44100, 48000, 22050, 24000, 8000, 16000])
def test_resample_vs_oracle(orig):
    x = torch.rand(3, 9001, generator=gen(orig)) * 2 - 1
    lens = torch.tensor([9001, 4000, 777], dtype=torch.int32)
    y, lo = audio.resample(x.to(DEV), orig, 16000, lens.to(DEV))
    if orig == 16000:
        assert torch.equal(y.cpu(), x) and torch.equal(lo.cpu(), lens)
        return
    for b in range(3):
        ref = ref_audio.resample(x[b, :lens[b]].numpy(), orig, 16000)
        n = int(lo[b])
        assert n == len(ref)
        assert np.abs(y[b, :n].cpu().numpy() - ref).max() < 5e-5          # fp32 FIR of <= 815 taps (fp32 table) vs the fp64 oracle
        assert float(y[b, n:].abs().max()) == 0.0 if n < y.shape[1] else True
    # the un-ragged call equals torchaudio itself (same fp32 table, fp32 accumulation)
    import torchaudio
    ta = torchaudio.functional.resample(x, orig, 16000, resampling_method="sinc_interp_kaiser", **audio.KAISER_BEST)
    y2, _ = audio.resample(x.to(DEV), orig, 16000)
    assert y2.shape == ta.shape and (y2.cpu() - ta).abs().max().item() < 2e-5


def test_peak_normalize_and_prompt_loader():
    x = torch.randn(4, 5000, generator=gen(3)) * torch.tensor([[0.1], [3.0], [1e-3], [0.0]])
    lens = torch.tensor([5000, 2500, 100, 5000], dtype=torch.int32)
    y = audio.peak_normalize(x.clone().to(DEV), lens.to(DEV)).cpu()
    for b in range(4):
        n = int(lens[b])
        ref = ref_audio.peak_normalize(x[b, :n].numpy())
        assert np.array_equal(y[b, :n].numpy(), ref.astype(np.float32)), b      # one IEEE division per sample: bit-exact
        assert torch.equal(y[b, n:], x[b, n:])                                    # samples past the clip are untouched
    clips = [((torch.rand(30000, generator=gen(5)) * 0.2 - 0.1).numpy(), 44100),
             ((torch.rand(8000, generator=gen(6)) * 2 - 1).numpy(), 16000),
             ((torch.rand(12345, generator=gen(7)) - 0.5).numpy(), 44100)]
    wav, wl = audio.load_prompts(clips, torch.device(DEV))
    for i, (c, sr) in enumerate(clips):
        ref = ref_audio.peak_normalize(ref_audio.resample(c, sr, 16000))
        n = int(wl[i])
        assert n == len(ref) and np.abs(wav[i, :n].cpu().numpy() - ref).max() < 5e-5
        assert abs(float(wav[i, :n].abs().max()) - 1.0) < 1e-6


def test_peak_normalize_long_clips():
    """Clips past 131072 samples run on the 64-CTA cap, each CTA striding over the clip: the peak in the last sample, a
    negative peak, and a larger value just past lens[b] that must not count."""
    L = 200003
    x = (torch.rand(3, L, generator=gen(11)) - 0.5).numpy()
    x[0, L - 1] = 0.75
    x[1, 150001] = -1.7
    lens = np.array([L, L, 180000], dtype=np.int32)
    x[2, 179999], x[2, 180000] = 0.625, 5.0
    y = audio.peak_normalize(torch.from_numpy(x).to(DEV), torch.from_numpy(lens).to(DEV)).cpu().numpy()
    for b in range(3):
        n = int(lens[b])
        peak = np.abs(x[b, :n]).max()
        assert peak == np.float32((0.75, 1.7, 0.625)[b]), b
        assert np.array_equal(y[b, :n], x[b, :n] / peak), b                      # one IEEE division per sample
        assert np.array_equal(y[b, n:], x[b, n:]), b


def test_pcm16_exact_edges():
    """round-to-nearest-even of x * 32768, saturated to [-32768, 32767]: every tie (k + 0.5) / 32768, +-1 and just past,
    on a length that is not a multiple of the 256-thread block"""
    from megatts2_b200 import _lib as L
    from megatts2_b200 import ops
    ties = (np.arange(-32768, 32768, dtype=np.float64) + 0.5) / 32768
    one = np.float32(1.0)
    edges = [1.0, -1.0, np.nextafter(one, 2), -np.nextafter(one, 2), np.nextafter(one, 0), -np.nextafter(one, 0), 1.5,
             -2.0, 32767 / 32768, -32767 / 32768, 0.0, -0.0, 0.5 / 32768, -0.5 / 32768, 1.5 / 32768, -1.5 / 32768]
    x = np.concatenate([ties, np.asarray(edges, dtype=np.float64), np.linspace(-1.1, 1.1, 1001)]).astype(np.float32)
    n = x.size
    assert n % 256 != 0
    out = torch.full((n + 7,), 12345, dtype=torch.int16, device=DEV)
    L.check(L.lib().mtts_pcm16_f32(torch.from_numpy(x).to(DEV).data_ptr(), n, out.data_ptr(), ops._stream()))
    out = out.cpu().numpy()
    ref = np.clip(np.rint(x * np.float32(32768)), -32768, 32767).astype(np.int16)                # np.rint: ties to even
    assert np.array_equal(out[:n], ref)
    assert (out[n:] == 12345).all()
    assert out[65536] == 32767 and out[65537] == -32768 and out[65538] == 32767 and out[65539] == -32768
    assert (out[0], out[1], out[32767], out[32768], out[65535]) == (-32768, -32766, 0, 0, 32767)           # ties to even


def test_wav_writer(tmp_path):
    w = (torch.rand(1, 4097, generator=gen(9)) * 2.2 - 1.1).to(DEV)             # includes samples beyond +-1 (saturation)
    pf, pi = str(tmp_path / "f.wav"), str(tmp_path / "i.wav")
    audio.save_wav(pf, w, 16000)
    y, sr = audio.read_wav(pf)
    assert sr == 16000 and np.array_equal(y, w[0].cpu().numpy())
    assert open(pf, "rb").read().endswith(ref_audio.wav_float32_payload(w[0].cpu().numpy()))
    audio.save_wav(pi, w, 16000, length=4000, encoding="PCM_S")
    q, _ = audio.read_wav(pi)
    ref = np.clip(np.rint(w[0, :4000].cpu().numpy() * 32768.0), -32768, 32767) / 32768.0
    assert len(q) == 4000 and np.array_equal(q, ref.astype(np.float32))


def test_prompt_mels_matches_the_reference_loop(weights_cpu):
    """Megatts.prompt_mels = the prompt loop of Megatts.forward (models/megatts2.py:333-346): every clip resampled to
    16 kHz, peak-normalised, mel-extracted and concatenated along time; mels_prompt = the first clip's mel."""
    import helpers
    from oracle import ref_megatts2 as R
    tts = helpers.build_megatts(weights_cpu("g"), weights_cpu("plm"), weights_cpu("adm"), weights_cpu("hifigan"), DEV)
    clips = [((torch.rand(40000, generator=gen(21)) * 0.6 - 0.3).numpy(), 44100),
             ((torch.rand(20000, generator=gen(22)) * 2 - 1).numpy(), 16000)]
    mels, first = tts.prompt_mels(clips)
    refs = []
    for c, sr in clips:
        y = ref_audio.peak_normalize(ref_audio.resample(c, sr, 16000)).astype(np.float32)
        refs.append(R.mel_spectrogram(torch.from_numpy(y)[None])[0].transpose(0, 1))          # (frames, 80)
    ref = torch.cat(refs, 0)
    assert mels.shape == (1, ref.shape[0], 80) and first.shape == (1, refs[0].shape[0], 80)
    assert (mels[0].cpu() - ref).abs().mean().item() < 1e-4
    assert torch.equal(first[0], mels[0, :refs[0].shape[0]])
