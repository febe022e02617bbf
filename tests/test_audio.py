"""Audio front-end (SURVEY §8f N6): decoded samples -> log-mel -> audio encoder input.

CPU: the host tables (Slaney filterbank, periodic Hann window, twiddles) against independent implementations, frame counts,
webui's z_length rule, and argument validation of mugd_melspec.  GPU: the kernel against the CPU oracle (tests/audio_oracle.py)
at 3-minute and short lengths, padding, batching, and ``audio_features`` through the encoder and the sampler.

Parity with librosa itself is not tested: librosa is not installed where this suite runs, so no reference golden exists.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import audio_oracle
from mug_diffusion_b200 import audio, synth, wave
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.config import ModelConfig

SR = 22050
N_3MIN = 3 * 60 * SR                      # 3,969,000 samples -> 31,008 frames


# ---- seeded test signals ------------------------------------------------------------------------------------------------
def music_like(n: int, seed: int = 11) -> np.ndarray:
    """a silent first second, then notes of decaying partials every 0.25 s, noise bursts every 0.5 s and a 1e-4 noise floor"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    y = 1e-4 * rng.standard_normal(n)
    for start in np.arange(1.0, n / SR, 0.25):
        i0 = int(start * SR)
        i1 = min(n, i0 + 3 * SR)                                   # a note rings for 3 s (its envelope is below 2 % by then)
        tt = t[i0:i1] - start
        env = np.exp(-tt * rng.uniform(2.0, 8.0))
        f0 = 55.0 * 2 ** (rng.integers(0, 48) / 12)
        for k in range(1, 7):
            if k * f0 < SR / 2:
                y[i0:i1] += env * np.sin(2 * np.pi * k * f0 * tt + rng.uniform(0, 2 * np.pi)) * (0.3 / k)
    for start in np.arange(1.0, n / SR, 0.5):
        i0 = int(start * SR)
        m = min(n - i0, 2000)
        y[i0:i0 + m] += rng.standard_normal(m) * np.exp(-np.arange(m) / 300.0) * 0.5
    y[:min(n, SR)] = 0.0
    peak = np.abs(y).max()
    return (0.9 * y / peak if peak > 0 else y).astype(np.float32)


def white_noise(n: int, seed: int = 12) -> np.ndarray:
    return np.random.default_rng(seed).uniform(-1.0, 1.0, n).astype(np.float32)


def clipped_square(n: int) -> np.ndarray:
    t = np.arange(n) / SR
    return np.clip(1.5 * np.sign(np.sin(2 * np.pi * 220.0 * t)), -1.0, 1.0).astype(np.float32)


def silence(n: int) -> np.ndarray:
    return np.zeros(n, np.float32)


SIGNALS = {"music": music_like, "noise": white_noise, "square": clipped_square, "zeros": silence}


# ---- host tables --------------------------------------------------------------------------------------------------------
def _slaney_mel_basis_per_element(sr=22050, n_fft=512, n_mels=128) -> np.ndarray:
    """librosa.filters.mel(norm='slaney', htk=False) restated element by element with Python's math module"""
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0

    def to_mel(f):
        return min_log_mel + math.log(f / min_log_hz) / logstep if f >= min_log_hz else f / f_sp

    def to_hz(m):
        return min_log_hz * math.exp(logstep * (m - min_log_mel)) if m >= min_log_mel else f_sp * m

    lo, hi = to_mel(0.0), to_mel(sr / 2.0)
    mel_f = [to_hz(lo + (hi - lo) * i / (n_mels + 1)) for i in range(n_mels + 2)]
    freqs = [k * sr / n_fft for k in range(n_fft // 2 + 1)]
    out = np.zeros((n_mels, len(freqs)), np.float32)
    for i in range(n_mels):
        enorm = 2.0 / (mel_f[i + 2] - mel_f[i])
        for k, f in enumerate(freqs):
            ramp = max(0.0, min((f - mel_f[i]) / (mel_f[i + 1] - mel_f[i]), (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1])))
            out[i, k] = np.float32(float(np.float32(ramp)) * enorm)
    return out


def test_mel_basis_vs_torchaudio():
    taf = pytest.importorskip("torchaudio.functional")
    fb = taf.melscale_fbanks(257, 0.0, 11025.0, 128, 22050, norm="slaney", mel_scale="slaney").T.numpy()
    B = audio.mel_basis()
    assert B.dtype == np.float32 and B.shape == (128, 257)
    assert np.abs(fb - B).max() < 1e-6 and np.abs(fb - B).max() < 1e-5 * B.max()


def test_mel_basis_vs_per_element_restatement():
    B = audio.mel_basis() + np.float32(0.0)                       # -0.0 (a zero ramp negated) -> +0.0 before comparing bits
    ref = _slaney_mel_basis_per_element()
    assert np.array_equal(B != 0, ref != 0)
    ulps = np.abs(B.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1


def test_mel_basis_sparsity_and_csr():
    B = audio.mel_basis()
    nz = B != 0
    assert nz.sum(axis=1).min() >= 1                            # no empty band
    assert nz.sum() == 504 and nz.sum(axis=0).max() <= 2          # each rfft bin feeds at most two bands
    start, length, w = audio.filter_csr(B)
    assert start.min() >= 0 and (start + length).max() <= 257 and length.sum() == len(w)
    dense = np.zeros_like(B)
    off = 0
    for m in range(128):
        dense[m, start[m]:start[m] + length[m]] = w[off:off + length[m]]
        off += length[m]
    assert np.array_equal(dense, B)


def test_periodic_hann_window():
    w = audio.hann_window(512)
    signal = pytest.importorskip("scipy.signal")
    assert np.array_equal(w, signal.get_window("hann", 512, fftbins=True))      # what librosa's STFT uses
    assert np.abs(w - torch.hann_window(512, periodic=True, dtype=torch.float64).numpy()).max() < 1e-15


def test_fft_twiddles():
    tw = audio.fft_twiddles(512)
    ref = np.exp(-2j * np.pi * np.arange(256) / 512)
    assert tw.dtype == np.float64 and tw.shape == (256, 2)
    assert np.abs(tw[:, 0] + 1j * tw[:, 1] - ref).max() < 1e-15


@pytest.mark.parametrize("n", [1, 100, 127, 128, 129, 511, 512, 513, 1000, 5000 * 128, 5000 * 128 + 77])
def test_frame_count(n):
    T = audio.n_frames(n, 128)
    assert T == 1 + n // 128
    assert audio_oracle.log_mel(white_noise(n)).shape == (1, 128, T)


def test_z_length_rule_matches_webui():
    def webui(t, z_length=512, max_audio_frame=32768):       # webui.py:349-353
        audio_map_length_ratio = max_audio_frame // z_length
        test_map_length = t / audio_map_length_ratio
        return (int(test_map_length / 32) + 1) * 32

    per = audio.frames_per_latent(len(wave.WaveConfig().channel_mult), ModelConfig().unet.levels)
    assert per == 32768 // 512
    ts = list(range(1, 70000, 7)) + [2048 * k for k in range(1, 40)] + [2048 * k - 1 for k in range(1, 40)]
    for t in ts:
        assert audio.z_length_for(t, per) == webui(t), t
    assert audio.z_length_for(2048, per) == 64                   # an exact multiple still gains 32
    assert audio.z_length_for(1 + N_3MIN // 128, per) == 512


def _call(lib, **kw):
    a = dict(h=None, y=1 << 20, n=1000, ldy=1000, B=1, window=1 << 21, twiddle=1 << 22, n_fft=512, start=[0] * 128, length=[1] * 128,
             weights=1 << 23, n_mels=128, hop=128, out=1 << 24, ldo=128, T_out=8)
    a.update(kw)
    nm = max(a["n_mels"], 1)
    st = (C.c_int32 * nm)(*(a["start"] + [0] * nm)[:nm])
    ln = (C.c_int32 * nm)(*(a["length"] + [0] * nm)[:nm])
    return lib.mugd_melspec(a["h"], a["y"], a["n"], a["ldy"], a["B"], a["window"], a["twiddle"], a["n_fft"], st, ln,
                            a["weights"], a["n_mels"], a["hop"], a["out"], a["ldo"], a["T_out"], None)


@pytest.mark.parametrize("bad,msg", [
    (dict(y=None), "NULL"), (dict(out=None), "NULL"), (dict(weights=None), "NULL"), (dict(window=None), "NULL"),
    (dict(n_fft=1024), "n_fft"), (dict(n=0), "n >= 1"), (dict(B=0), "B >= 1"), (dict(hop=0), "hop >= 1"),
    (dict(B=2, ldy=999), "ldy"), (dict(T_out=7), "T_out"), (dict(ldo=127), "ldo"), (dict(n_mels=0), "n_mels"),
    (dict(n_mels=300), "n_mels"), (dict(start=[-1] + [0] * 127), "band 0"), (dict(start=[0] * 127 + [250], length=[1] * 127 + [8]), "band 127"),
    (dict(length=[1] * 5 + [-1] + [1] * 122), "band 5"), (dict(twiddle=(1 << 22) + 8), "alignment"), (dict(), "null handle"),
], ids=lambda v: None if isinstance(v, dict) else v.replace(" ", "_"))
def test_melspec_argument_validation(bad, msg):
    """every check runs on the host before the launch: no device is needed to see them fail"""
    lib = L_.load()
    rc = _call(lib, **bad)
    assert rc == 1, rc                                            # MUGD_ERR_INVALID
    assert msg in lib.mugd_last_error().decode()
    with pytest.raises(L_.MugdError):
        L_.check(rc, "mugd_melspec")


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _fp16_ulps(a: torch.Tensor, b: torch.Tensor) -> np.ndarray:
    """distance in fp16 steps between two float32 tensors of non-negative fp16 values"""
    ai = a.detach().cpu().numpy().astype(np.float16).view(np.int16).astype(np.int32)
    bi = b.detach().cpu().numpy().astype(np.float16).view(np.int16).astype(np.int32)
    return np.abs(ai - bi)


@pytest.fixture(scope="module")
def model():
    from mug_diffusion_b200.sampler import MugDiffusionB200
    sd = {**synth.synthetic_state_dict(96), **wave.synthetic_wave_state_dict()}
    return sd, MugDiffusionB200.from_state_dict(sd, z_length=96)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [N_3MIN, 100, 5000 * 128], ids=["3min", "n100", "n640000"])
@pytest.mark.parametrize("sig", list(SIGNALS))
def test_gpu_melspec_vs_oracle(model, sig, n):
    _, m = model
    y = SIGNALS[sig](n)
    got = m.model.melspectrogram(y)
    ref = audio_oracle.log_mel(y)
    assert got.shape == ref.shape == (1, 128, 1 + n // 128) and got.device.type == "cuda"
    g = got.cpu()
    assert torch.equal(g.half().float(), g)                      # fp16 values
    d = _fp16_ulps(g, ref)
    assert d.max() <= 1, d.max()
    assert (d == 0).mean() >= 0.9999, (d == 0).mean()
    if sig == "zeros":
        assert torch.count_nonzero(g) == 0
    if sig == "music" and n == N_3MIN:
        quiet = (SR - 256) // 128                                 # frames that see only the silent first second
        assert torch.count_nonzero(g[..., :quiet]) == 0
        assert g.abs().max() > 1.0


@pytest.mark.gpu
def test_gpu_melspec_padding_rows_and_leading_dimension(model):
    _, m = model
    fe = m.mel_frontend
    y = fe.samples(music_like(40000))
    T, T_out, ld = 1 + 40000 // 128, 448, 160
    buf = torch.full((T_out, ld), 7.0, device="cuda")
    from mug_diffusion_b200.engine import View
    fe.write_rows(y, View(buf.data_ptr(), ld, T_out, 128), T_out)
    torch.cuda.synchronize()
    ref = m.model.melspectrogram(y)[0].T
    assert torch.equal(buf[:T, :128], ref)
    assert torch.count_nonzero(buf[T:, :128]) == 0               # webui's zero pad
    assert bool((buf[:, 128:] == 7.0).all())                       # columns past n_mels untouched


@pytest.mark.gpu
def test_gpu_melspec_batch_rows_equal_single_calls(model):
    _, m = model
    n = 123457
    ys = np.stack([music_like(n, seed=3), white_noise(n, seed=4), clipped_square(n)])
    batch = m.model.melspectrogram(torch.from_numpy(ys).cuda())
    assert batch.shape == (3, 128, 1 + n // 128)
    for b in range(3):
        assert torch.equal(batch[b:b + 1], m.model.melspectrogram(ys[b]))


def _pad(mel: torch.Tensor, T: int) -> torch.Tensor:
    return torch.nn.functional.pad(mel, (0, T - mel.shape[-1]))


@pytest.mark.gpu
def test_gpu_audio_features_equals_wave_model_of_padded_mel(model):
    _, m = model
    y = music_like(5000 * 128)
    w, zl = m.model.audio_features(y, 4)
    assert zl == 96 and len(w) == 10 and all(h is None for h in w[:6])
    w_ref = m.model.wave_model(_pad(m.model.melspectrogram(y), 64 * zl))
    for h, r in zip(w[6:], w_ref[6:]):
        assert h.shape == (4,) + tuple(r.shape[1:])
        for b in range(4):
            assert torch.equal(h[b], r[0])


@pytest.mark.gpu
def test_gpu_audio_features_vs_wave_oracle(model):
    from oracle import wave_oracle as worc
    sd, m = model
    y = music_like(5000 * 128, seed=21)
    w, zl = m.model.audio_features(y, 1)
    assert zl == 96
    with torch.no_grad():
        ref = worc.wave_forward(sd, _pad(audio_oracle.log_mel(y), 64 * zl))
    for i in range(6, 10):
        err = float((w[i].cpu() - ref[i]).abs().max() / ref[i].abs().max())
        assert err < 1e-4, (i, err)


@pytest.mark.gpu
def test_gpu_samples_to_hit_objects(model):
    """webui's request path from decoded samples: audio_features -> DDIM (CFG) -> decode -> notes, bit-identical to the same
    chain fed the audio encoder's output for the kernel's own mel"""
    from mug_diffusion_b200.sampler import DDIMSampler
    _, m = model
    count = 2
    y = music_like(5000 * 128, seed=33)
    inp = synth.synthetic_inputs(count, 96)
    w, zl = m.model.audio_features(y, count)
    m.z_length = zl

    def chain(w_):
        z, _ = DDIMSampler(m).sample(S=2, c=inp["c"].cuda(), w=w_, batch_size=count, verbose=False, x_T=inp["x_T"].cuda(),
                                     unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
        return z, m.model.decode_to_hit_objects(z, 46.439909297052154)

    z, lines = chain(w)
    w_ref = m.model.wave_model(_pad(m.model.melspectrogram(y), 64 * zl))
    z_ref, lines_ref = chain([None if h is None else h.expand(count, -1, -1) for h in w_ref])
    assert bool(torch.isfinite(z).all()) and len(lines) == count
    assert torch.equal(z, z_ref) and lines == lines_ref
