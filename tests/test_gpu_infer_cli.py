"""GPU tests of the command line, `python -m f5_tts_b200.infer_cli`, end to end, and of `remove_silence` through
`F5TTS.infer`.

Checkpoint and vocoder files are synthetic, written in the released layouts as in tests/test_gpu_infer.py; the vocoder
sits at the CLI's local path `../checkpoints/vocos-mel-24khz`, relative to the working directory.  There are three
voices: the reference's `basic_ref_en.wav`, and two 16-bit wavs derived from it: `town` (scaled by 0.5, so its RMS is
under `target_rms` and the output gain path runs, and cut to 3 s) and `quiet` (scaled by 0.001 and cut to 3 s, so its
generated audio is scaled far below -50 dBFS and `remove_silence` has silence to cut).

The expected output is this package's `infer_process`, called piece by piece with the same voices and speeds after the
same `torch.manual_seed`: the sampler draws its noise from the device generator, and the engine is deterministic, so
the files must match sample for sample.
"""
import os
import shutil
import wave

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import synthdata as SD  # noqa: E402
from f5_tts_b200 import api, infer, infer_cli  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402

DEV = "cuda:0"
NFE = 4
REF_TEXTS = {"main": "Some call me nature, others call me mother nature.",
             "town": "Some call me nature,", "quiet": "Some call me nature,"}
STORY = ("I don't really care what you call me. [town] I've been a silent spectator, watching species evolve. "
         "[main] Empires rise and fall. [town] But always remember, I am mighty and enduring.")


def _write_pcm(path, pcm, rate=24000):
    with wave.open(path, "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(rate)
        f.writeframes(pcm.astype("<i2").tobytes())


def _read_pcm(path):
    with wave.open(path, "rb") as f:
        assert (f.getframerate(), f.getnchannels(), f.getsampwidth()) == (24000, 1, 2)
        return np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")


def _int16(wav):
    """What the writer of F5TTS.export_wav stores."""
    return (np.clip(np.asarray(wav), -1.0, 1.0) * 32767.0).astype("<i2")


@pytest.fixture(scope="module")
def assets(tmp_path_factory, golden_dir):
    from safetensors.torch import save_file

    d = tmp_path_factory.mktemp("cliassets")
    sd = SD.synthetic_state_dict(SD.f5tts_small(), seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(d / "model_1.safetensors")
    save_file(ema, ckpt)
    vcfg = {"feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                                  "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": 100,
                                                "padding": "center"}},
            "backbone": {"class_path": "vocos.models.VocosBackbone",
                         "init_args": {"input_channels": 100, "dim": 512, "intermediate_dim": 1536, "num_layers": 8}},
            "head": {"class_path": "vocos.heads.ISTFTHead",
                     "init_args": {"dim": 512, "n_fft": 1024, "hop_length": 256, "padding": "center"}}}
    vdir = d / "checkpoints" / "vocos-mel-24khz"
    vdir.mkdir(parents=True)
    (vdir / "config.yaml").write_text(yaml.safe_dump(vcfg))
    full = dict(SD.synthetic_vocos_state_dict())
    full["feature_extractor.mel_spec.spectrogram.window"] = torch.hann_window(1024)
    full["feature_extractor.mel_spec.mel_scale.fb"] = O.mel_filterbank()
    torch.save(full, str(vdir / "pytorch_model.bin"))
    (d / "work").mkdir()

    voices = {"main": str(d / "main.wav"), "town": str(d / "town.wav"), "quiet": str(d / "quiet.wav")}
    shutil.copy(os.path.join(golden_dir, "basic_ref_en.wav"), voices["main"])
    audio, sr = infer._load_wav(voices["main"])
    base = audio[0, : 3 * sr].numpy() * 32768.0
    _write_pcm(voices["town"], np.round(0.5 * base))
    _write_pcm(voices["quiet"], np.round(0.001 * base))

    vocab = os.path.join(golden_dir, "vocab.txt")
    cls, arch = api.MODEL_ARCH["F5TTS_Small"]
    model = infer.load_model(cls, arch, ckpt, vocab_file=vocab, device=DEV)
    vocoder = infer.load_vocoder("vocos", True, str(vdir), DEV)
    return dict(dir=d, ckpt=ckpt, vocab=vocab, vdir=str(vdir), voices=voices, model=model, vocoder=vocoder)


def _config(a, path, voices):
    lines = [f'ref_audio = "{a["voices"]["main"]}"', f'ref_text = "{REF_TEXTS["main"]}"', "speed = 0.9"]
    for name, speed in voices.items():
        lines += [f"[voices.{name}]", f'ref_audio = "{a["voices"][name]}"', f'ref_text = "{REF_TEXTS[name]}"']
        if speed is not None:
            lines.append(f"speed = {speed}")
    path.write_text("\n".join(lines) + "\n")
    return str(path)


def _run_cli(a, monkeypatch, seed, config, out_dir, text, *flags):
    monkeypatch.chdir(a["dir"] / "work")  # the vocoder is read from ../checkpoints/vocos-mel-24khz
    torch.manual_seed(seed)
    infer_cli.main(["-c", config, "-m", "F5TTS_Small", "-p", a["ckpt"], "-v", a["vocab"], "--load_vocoder_from_local",
                    "--nfe_step", str(NFE), "--device", DEV, "-o", str(out_dir), "-w", "out.wav", "-t", text, *flags])
    return str(out_dir / "out.wav")


def _expected(a, seed, pieces, speeds):
    """infer_process per piece, in order, after the same seed."""
    torch.manual_seed(seed)
    out = []
    for voice, text in pieces:
        ref_audio, ref_text = infer.preprocess_ref_audio_text(a["voices"][voice], REF_TEXTS[voice])
        wav, sr, _ = infer.infer_process(ref_audio, ref_text, text, a["model"], a["vocoder"], nfe_step=NFE,
                                         speed=speeds[voice], device=DEV, show_info=lambda *_: None)
        assert sr == 24000
        out.append(wav)
    return out


def test_cli_story_equals_infer_process(assets, tmp_path, monkeypatch):
    a = assets
    config = _config(a, tmp_path / "story.toml", {"town": 1.2})
    out = _run_cli(a, monkeypatch, 21, config, tmp_path / "out", STORY, "--save_chunk")
    pieces = infer_cli.split_voices(STORY, {"main": {}, "town": {}})
    assert [v for v, _ in pieces] == ["main", "town", "main", "town"]
    segs = _expected(a, 21, pieces, {"main": 0.9, "town": 1.2})
    for s in segs:
        assert s.ndim == 1 and np.isfinite(s).all() and float(np.abs(s).max()) > 0
    got = _read_pcm(out)
    want = _int16(np.concatenate(segs))
    print(f"[infer_cli] {len(pieces)} pieces, {len(got)} samples; piece lengths {[len(s) for s in segs]}")
    assert got.shape == want.shape and np.array_equal(got, want)
    chunk_dir = tmp_path / "out" / "out_chunks"
    names = [infer_cli.chunk_file_name(i, text, True) for i, (_, text) in enumerate(pieces)]
    assert sorted(os.listdir(chunk_dir)) == sorted(names)
    for name, s in zip(names, segs):
        assert np.array_equal(_read_pcm(str(chunk_dir / name)), _int16(s))


def test_cli_remove_silence(assets, tmp_path, monkeypatch):
    a = assets
    text = ("Some call me nature. [quiet] I've been a silent spectator, watching species evolve, empires rise and "
            "fall. [main] But always remember, I am mighty.")
    config = _config(a, tmp_path / "quiet.toml", {"quiet": None})
    out = _run_cli(a, monkeypatch, 5, config, tmp_path / "out", text, "--remove_silence")
    pieces = infer_cli.split_voices(text, {"main": {}, "quiet": {}})
    segs = _expected(a, 5, pieces, {"main": 0.9, "quiet": 0.9})
    untrimmed = str(tmp_path / "untrimmed.wav")
    infer._write_wav(untrimmed, np.concatenate(segs))
    full = _read_pcm(untrimmed)
    infer.remove_silence_for_generated_wav(untrimmed)
    got, want = _read_pcm(out), _read_pcm(untrimmed)
    print(f"[infer_cli --remove_silence] {len(full)} -> {len(got)} samples (quiet piece {len(segs[1])})")
    assert got.shape == want.shape and np.array_equal(got, want)
    assert len(got) < len(full) - 12000  # the quiet piece is over 1.5 s of silence


def test_f5tts_infer_remove_silence(assets, tmp_path):
    a = assets
    tts = api.F5TTS(model="F5TTS_Small", ckpt_file=a["ckpt"], vocab_file=a["vocab"], vocoder_local_path=a["vdir"],
                    device=DEV)
    gen = "I've been a silent spectator, watching species evolve, empires rise and fall."
    fw = str(tmp_path / "trimmed.wav")
    wav, sr, spec = tts.infer(a["voices"]["quiet"], REF_TEXTS["quiet"], gen, nfe_step=NFE, seed=3, file_wave=fw,
                              remove_silence=True, show_info=lambda *_: None)
    plain_wav, _, _ = tts.infer(a["voices"]["quiet"], REF_TEXTS["quiet"], gen, nfe_step=NFE, seed=3,
                                show_info=lambda *_: None)
    assert np.array_equal(wav, plain_wav)  # the returned array is not trimmed
    ref = str(tmp_path / "ref.wav")
    infer._write_wav(ref, wav)
    infer.remove_silence_for_generated_wav(ref)
    got = _read_pcm(fw)
    assert np.array_equal(got, _read_pcm(ref)) and len(got) < len(wav)
