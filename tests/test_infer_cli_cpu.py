"""CPU tests of the command line (`f5_tts_b200.infer_cli`) and of `infer.remove_silence_for_generated_wav`.

Silence removal is compared with `_PydubSegment` / `_pydub_split_on_silence` below: a direct transcription of pydub
0.25's `AudioSegment` slicing and `silence.detect_silence` / `detect_nonsilent` / `split_on_silence`, in which every
window's RMS comes from `audioop.rms` itself.  The CLI is run with the sampler and the loaders replaced by stand-ins,
so what is checked here is the settings, the voices, the piece list and the files; tests/test_gpu_infer_cli.py runs it
end to end on the GPU.
"""
import itertools
import os
import re
import shutil
import warnings
import wave

import numpy as np
import pytest

from f5_tts_b200 import api, infer, infer_cli

with warnings.catch_warnings():
    warnings.simplefilter("ignore", DeprecationWarning)
    import audioop


# ------------------------------------------------------------------------------------- pydub, transcribed
class _PydubSegment:
    """The parts of pydub.AudioSegment that split_on_silence uses, on raw 16-bit little-endian frames."""

    def __init__(self, data, frame_rate, channels):
        self._data, self.frame_rate, self.channels = data, frame_rate, channels
        self.sample_width, self.frame_width = 2, 2 * channels

    def frame_count(self, ms=None):
        if ms is not None:
            return ms * (self.frame_rate / 1000.0)
        return float(len(self._data) // self.frame_width)

    def __len__(self):
        return round(1000 * (self.frame_count() / self.frame_rate))

    def _parse_position(self, val):
        if val < 0:
            val = len(self) - abs(val)
        val = self.frame_count(ms=len(self)) if val == float("inf") else self.frame_count(ms=val)
        return int(val)

    def __getitem__(self, ms):
        start = ms.start if ms.start is not None else 0
        end = ms.stop if ms.stop is not None else len(self)
        start, end = min(start, len(self)), min(end, len(self))
        start = self._parse_position(start) * self.frame_width
        end = self._parse_position(end) * self.frame_width
        data = self._data[start:end]
        missing_frames = (end - start - len(data)) // self.frame_width
        if missing_frames:
            assert missing_frames <= self.frame_count(ms=2)
            data += audioop.mul(data[: self.frame_width], self.sample_width, 0) * missing_frames
        return _PydubSegment(data, self.frame_rate, self.channels)

    @property
    def rms(self):
        return audioop.rms(self._data, self.sample_width)


def _pydub_detect_silence(seg, min_silence_len, silence_thresh, seek_step):
    seg_len = len(seg)
    if seg_len < min_silence_len:
        return []
    silence_thresh = 10 ** (float(silence_thresh) / 20) * ((2 ** 16) / 2)
    silence_starts = []
    last_slice_start = seg_len - min_silence_len
    slice_starts = range(0, last_slice_start + 1, seek_step)
    if last_slice_start % seek_step:
        slice_starts = itertools.chain(slice_starts, [last_slice_start])
    for i in slice_starts:
        if seg[i:i + min_silence_len].rms <= silence_thresh:
            silence_starts.append(i)
    if not silence_starts:
        return []
    silent_ranges = []
    prev_i = silence_starts.pop(0)
    current_range_start = prev_i
    for silence_start_i in silence_starts:
        continuous = silence_start_i == prev_i + seek_step
        silence_has_gap = silence_start_i > (prev_i + min_silence_len)
        if not continuous and silence_has_gap:
            silent_ranges.append([current_range_start, prev_i + min_silence_len])
            current_range_start = silence_start_i
        prev_i = silence_start_i
    silent_ranges.append([current_range_start, prev_i + min_silence_len])
    return silent_ranges


def _pydub_detect_nonsilent(seg, min_silence_len, silence_thresh, seek_step):
    silent_ranges = _pydub_detect_silence(seg, min_silence_len, silence_thresh, seek_step)
    len_seg = len(seg)
    if not silent_ranges:
        return [[0, len_seg]]
    if silent_ranges[0][0] == 0 and silent_ranges[0][1] == len_seg:
        return []
    prev_end_i = 0
    nonsilent_ranges = []
    for start_i, end_i in silent_ranges:
        nonsilent_ranges.append([prev_end_i, start_i])
        prev_end_i = end_i
    if end_i != len_seg:
        nonsilent_ranges.append([prev_end_i, len_seg])
    if nonsilent_ranges[0] == [0, 0]:
        nonsilent_ranges.pop(0)
    return nonsilent_ranges


def _pydub_split_on_silence(seg, min_silence_len=1000, silence_thresh=-50, keep_silence=500, seek_step=10):
    output_ranges = [[start - keep_silence, end + keep_silence]
                     for (start, end) in _pydub_detect_nonsilent(seg, min_silence_len, silence_thresh, seek_step)]
    a, b = itertools.tee(output_ranges)
    next(b, None)
    for range_i, range_ii in zip(a, b):
        last_end = range_i[1]
        next_start = range_ii[0]
        if next_start < last_end:
            range_i[1] = (last_end + next_start) // 2
            range_ii[0] = range_i[1]
    return [seg[max(start, 0):min(end, len(seg))] for start, end in output_ranges]


# ------------------------------------------------------------------------------------- signals
def _signal(blocks, rate, channels=1, extra_frames=0, seed=0):
    """int16 [n, channels]: ("tone", ms) blocks are loud noise, ("quiet", ms) blocks stay just under the -50 dBFS
    threshold (RMS about 60), ("edge", ms) blocks sit at RMS 103-104, right at it; `extra_frames` adds frames that do
    not fill a millisecond."""
    g = np.random.default_rng(seed)
    parts = []
    for kind, ms in blocks:
        n = int(ms * rate / 1000)
        if kind == "tone":
            x = g.integers(-6000, 6000, (n, channels))
        elif kind == "quiet":
            x = g.integers(-100, 101, (n, channels))
        else:
            x = np.where(g.random((n, channels)) < 0.5, -104, 103)
        parts.append(x)
    parts.append(g.integers(-3000, 3000, (extra_frames, channels)))
    return np.concatenate(parts).astype(np.int16)


def _pydub_pieces(pcm, rate, **kw):
    seg = _PydubSegment(pcm.astype("<i2").tobytes(), rate, pcm.shape[1])
    return [np.frombuffer(s._data, dtype="<i2").reshape(-1, pcm.shape[1]) for s in _pydub_split_on_silence(seg, **kw)]


CASES = {
    "middle_long_and_short": ([("tone", 700), ("quiet", 1500), ("tone", 400), ("quiet", 600), ("tone", 900)], 24000, 1, 0),
    "start_and_end": ([("quiet", 2300), ("tone", 1200), ("quiet", 1800)], 24000, 1, 7),
    "exactly_one_second": ([("tone", 800), ("quiet", 1000), ("tone", 800)], 24000, 1, 0),
    "threshold_edge": ([("tone", 500), ("edge", 1400), ("tone", 300), ("quiet", 1100)], 24000, 1, 13),
    "all_silent": ([("quiet", 3000)], 24000, 1, 0),
    "no_silence": ([("tone", 2500)], 24000, 1, 0),
    "shorter_than_window": ([("quiet", 700)], 24000, 1, 5),
    "rate_22050": ([("tone", 300), ("quiet", 1250), ("tone", 600), ("quiet", 2000)], 22050, 1, 11),
    "rate_16000_stereo": ([("quiet", 1200), ("tone", 500), ("quiet", 1700), ("tone", 200)], 16000, 2, 3),
    "rate_44100": ([("tone", 1000), ("quiet", 1003), ("tone", 1000)], 44100, 1, 17),
    # 0.625 ms of extra frames round len() up to 2301 ms: the last piece is filled up to 2301 ms with zero frames
    "rounded_up_end": ([("quiet", 1500), ("tone", 800)], 24000, 1, 15),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_split_on_silence_matches_pydub(name):
    blocks, rate, ch, extra = CASES[name]
    pcm = _signal(blocks, rate, ch, extra)
    got = infer._split_on_silence(pcm, rate)
    want = _pydub_pieces(pcm, rate)
    assert [len(p) for p in got] == [len(p) for p in want]
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    if name == "all_silent":
        assert got == []
    if name in ("no_silence", "shorter_than_window"):
        assert len(got) == 1
    if name == "rounded_up_end":
        assert len(got[-1]) == 2301 * 24 - 1000 * 24 and not got[-1][-9:].any() and got[-1][-10].any()


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("keep_silence", [500, 800])
def test_split_on_silence_random_blocks(seed, keep_silence):
    """Random block patterns; keep_silence 800 makes the padded ranges of runs under 1.6 s overlap, so the midpoint
    split runs (at the reference's 500 ms two padded ranges at most touch, since a silent range is at least 1 s)."""
    g = np.random.default_rng(100 + seed)
    rate = [24000, 22050, 16000][seed % 3]
    blocks = [(["tone", "quiet", "edge"][g.integers(0, 3)], int(g.integers(50, 2600))) for _ in range(8)]
    pcm = _signal(blocks, rate, 1 + seed % 2, int(g.integers(0, 20)), seed=seed)
    got = infer._split_on_silence(pcm, rate, keep_silence=keep_silence)
    want = _pydub_pieces(pcm, rate, keep_silence=keep_silence)
    assert [len(p) for p in got] == [len(p) for p in want]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_midpoint_split_is_reached():
    blocks = [("tone", 600), ("quiet", 1200), ("tone", 600)]
    pcm = _signal(blocks, 24000)
    assert len(infer._split_on_silence(pcm, 24000, keep_silence=800)) == 2
    total = sum(len(p) for p in infer._split_on_silence(pcm, 24000, keep_silence=800))
    assert total == len(pcm)  # 1.2 s of silence < 2 x 0.8 s: the pieces meet at the midpoint and nothing is cut


@pytest.mark.parametrize("name", ["middle_long_and_short", "threshold_edge", "rate_22050", "rate_16000_stereo",
                                  "rate_44100"])
def test_window_rms_equals_audioop(name):
    blocks, rate, ch, extra = CASES[name]
    pcm = _signal(blocks, rate, ch, extra)
    starts, rms = infer._silence_window_rms(pcm, rate, 1000, 10)
    seg = _PydubSegment(pcm.astype("<i2").tobytes(), rate, ch)
    last = len(seg) - 1000
    want_starts = list(range(0, last + 1, 10)) + ([last] if last % 10 else [])
    assert starts == want_starts
    assert rms.tolist() == [seg[i:i + 1000].rms for i in starts]
    thresh = 10 ** (-50 / 20) * 32768
    if name == "threshold_edge":  # windows on both sides of the threshold
        assert (rms <= thresh).any() and (rms > thresh).any()


def _write_raw(path, pcm, rate):
    with wave.open(path, "wb") as f:
        f.setnchannels(pcm.shape[1])
        f.setsampwidth(2)
        f.setframerate(rate)
        f.writeframes(pcm.astype("<i2").tobytes())


def _read_raw(path):
    with wave.open(path, "rb") as f:
        params = (f.getframerate(), f.getnchannels(), f.getsampwidth())
        pcm = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2").reshape(-1, f.getnchannels())
    return params, pcm


@pytest.mark.parametrize("name", ["middle_long_and_short", "rate_16000_stereo", "all_silent", "no_silence"])
def test_remove_silence_round_trip(tmp_path, name):
    blocks, rate, ch, extra = CASES[name]
    pcm = _signal(blocks, rate, ch, extra)
    path = str(tmp_path / "x.wav")
    _write_raw(path, pcm, rate)
    infer.remove_silence_for_generated_wav(path)
    (r, c, w), back = _read_raw(path)
    assert (r, c, w) == (rate, ch, 2)
    pieces = _pydub_pieces(pcm, rate)
    want = np.concatenate(pieces) if pieces else pcm[:0]
    assert back.shape == want.shape and np.array_equal(back, want)


def _parent_export_bytes(wav, path):
    """F5TTS.export_wav as it was before silence removal existed."""
    pcm = (np.clip(np.asarray(wav), -1.0, 1.0) * 32767.0).astype("<i2")
    with wave.open(path, "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(24000)
        f.writeframes(pcm.tobytes())
    with open(path, "rb") as f:
        return f.read()


def test_export_wav(tmp_path):
    tts = object.__new__(api.F5TTS)  # export_wav needs no model
    tts.target_sample_rate = 24000
    g = np.random.default_rng(3)
    wav = np.concatenate([g.uniform(-1.2, 1.2, 30000), np.zeros(40000), g.uniform(-0.5, 0.5, 20000)]).astype(np.float32)
    plain, trimmed = str(tmp_path / "plain.wav"), str(tmp_path / "trimmed.wav")
    tts.export_wav(wav, plain)
    with open(plain, "rb") as f:
        assert f.read() == _parent_export_bytes(wav, str(tmp_path / "parent.wav"))
    tts.export_wav(wav, trimmed, remove_silence=True)
    _, full = _read_raw(plain)
    (r, c, w), back = _read_raw(trimmed)
    assert (r, c, w) == (24000, 1, 2)
    want = np.concatenate(_pydub_pieces(full, 24000))
    assert np.array_equal(back, want) and len(full) - len(back) > 15000  # 1.67 s of silence cut to about 1 s


# ------------------------------------------------------------------------------------- CLI settings
def _settings(argv, config=None):
    return infer_cli.resolve(infer_cli.parser.parse_args(argv), config or {})


def test_defaults_without_config():
    s = _settings([])
    assert s.model == "F5TTS_v1_Base" and s.ckpt_file == "" and s.vocab_file == "" and s.model_cfg == ""
    assert s.ref_audio == "infer/examples/basic/basic_ref_en.wav"
    assert s.ref_text == "Some call me nature, others call me mother nature."
    assert s.gen_text == "Here we generate something just for test."
    assert s.output_dir == "tests" and re.fullmatch(r"infer_cli_\d{8}_\d{6}\.wav", s.output_file)
    assert (s.save_chunk, s.use_legacy_text, s.remove_silence, s.load_vocoder_from_local) == (False, True, False, False)
    assert (s.vocoder_name, s.target_rms, s.cross_fade_duration, s.nfe_step, s.cfg_strength, s.sway_sampling_coef,
            s.speed, s.fix_duration, s.device) == ("vocos", 0.1, 0.15, 32, 2.0, -1.0, 1.0, None, infer.device)


def test_flag_over_config_and_falsy_fallback():
    config = {"model": "E2TTS_Base", "speed": 0.8, "nfe_step": 16, "cfg_strength": 3.0, "sway_sampling_coef": 0.5,
              "target_rms": 0.2, "output_dir": "out", "remove_silence": True, "gen_text": "from config",
              "ref_text": "config ref."}
    s = _settings(["-m", "F5TTS_Base", "--speed", "1.25", "--nfe_step", "8", "-t", "from flag"], config)
    assert (s.model, s.speed, s.nfe_step, s.gen_text) == ("F5TTS_Base", 1.25, 8, "from flag")
    assert (s.cfg_strength, s.sway_sampling_coef, s.target_rms, s.output_dir, s.remove_silence) == (3.0, 0.5, 0.2, "out", True)
    # a falsy flag value falls back to the config (the reference's `args.x or config.get(...)`)
    s = _settings(["--speed", "0", "--cfg_strength", "0", "--sway_sampling_coef", "0", "-t", ""], config)
    assert (s.speed, s.cfg_strength, s.sway_sampling_coef, s.gen_text) == (0.8, 3.0, 0.5, "from config")
    s = _settings(["--sway_sampling_coef", "0"])
    assert s.sway_sampling_coef == -1.0
    # ref_text is the exception: an empty flag is kept
    assert _settings(["-s", ""], config).ref_text == ""
    assert _settings([], config).ref_text == "config ref."


def test_legacy_text_flag():
    assert _settings([]).use_legacy_text is True
    assert _settings(["--no_legacy_text"]).use_legacy_text is False
    # no_legacy_text is store_false, so a config `no_legacy_text = true` turns legacy names ON, as in the reference
    assert _settings(["--no_legacy_text"], {"no_legacy_text": True}).use_legacy_text is True


def test_short_flags():
    s = _settings(["-c", "x.toml", "-m", "E2TTS_Base", "-mc", "m.yaml", "-p", "c.pt", "-v", "v.txt", "-r", "a.wav",
                   "-s", "rt.", "-t", "gt", "-o", "od", "-w", "of.wav"])
    assert (s.model, s.model_cfg, s.ckpt_file, s.vocab_file, s.ref_audio, s.ref_text, s.gen_text, s.output_dir,
            s.output_file) == ("E2TTS_Base", "m.yaml", "c.pt", "v.txt", "a.wav", "rt.", "gt", "od", "of.wav")
    assert str(s.wave_path) == os.path.join("od", "of.wav") and s.chunk_dir == os.path.join("od", "of_chunks")


def test_gen_file_overrides_gen_text(tmp_path, golden_dir):
    story = os.path.join(golden_dir, "story.txt")
    s = _settings(["-t", "ignored", "-f", story])
    with open(story, encoding="utf-8") as f:
        assert s.gen_text == f.read()
    config = infer_cli.load_config(os.path.join(golden_dir, "story.toml"))
    config["gen_file"] = story
    assert _settings([], config).gen_text == s.gen_text


def test_story_toml(golden_dir):
    config = infer_cli.load_config(os.path.join(golden_dir, "story.toml"))
    assert config["gen_file"] == "infer/examples/multi/story.txt"  # the reference's package path: not resolved here
    config["gen_file"] = os.path.join(golden_dir, "story.txt")
    s = _settings([], config)
    assert (s.model, s.ref_text, s.remove_silence, s.output_file) == ("F5TTS_v1_Base", "", True, "infer_cli_story.wav")
    assert config["voices"]["town"]["speed"] == 0.8 and "speed" not in config["voices"]["country"]


# ------------------------------------------------------------------------------------- voices and pieces
def test_story_split_matches_reference_regexes(golden_dir, capsys):
    with open(os.path.join(golden_dir, "story.txt"), encoding="utf-8") as f:
        text = f.read()
    voices = {"town": {}, "country": {}, "main": {}}
    pieces = infer_cli.split_voices(text, voices)
    expected = []
    for chunk in re.split(r"(?=\[\w+\])", text):  # infer_cli.py:323-342 of the reference
        if not chunk.strip():
            continue
        m = re.match(r"\[(\w+)\]", chunk)
        voice = m[1] if m and m[1] in voices else "main"
        expected.append((voice, re.sub(r"\[(\w+)\]", "", chunk).strip()))
    assert pieces == expected
    assert [v for v, _ in pieces] == ["main", "town", "main", "country", "main", "country"]
    assert pieces[0][1].startswith("A Town Mouse") and pieces[3][1] == '"Goodbye,"' and pieces[4][1] == "said he,"
    assert capsys.readouterr().out.count("No voice tag found, using main.") == 1


def test_unknown_untagged_and_blank_pieces(capsys):
    voices = {"town": {}, "main": {}}
    pieces = infer_cli.split_voices("Hello. [nobody] Who? [town] Here.  [main]   [town]\n Bye.", voices)
    assert pieces == [("main", "Hello."), ("main", "Who?"), ("town", "Here."), ("town", "Bye.")]
    out = capsys.readouterr().out
    assert "No voice tag found, using main." in out and "Voice nobody not found, using main." in out
    assert infer_cli.split_voices("   \n", voices) == []


def test_chunk_file_names():
    assert infer_cli.chunk_file_name(0, "Hello there.", True) == "0_Hello there..wav"
    long = "x" * 199 + "é" + "y" * 60
    assert infer_cli.chunk_file_name(3, long, False) == "3_" + "x" * 199 + "é ... .wav"
    assert infer_cli.chunk_file_name(3, long, True) == "3_" + "x" * 199 + "e ... .wav"
    assert infer_cli.chunk_file_name(1, "Café naïve – Ωmega", True) == "1_Cafe naive  mega.wav"
    assert infer_cli.chunk_file_name(1, "Café naïve", False) == "1_Café naïve.wav"


# ------------------------------------------------------------------------------------- errors
def test_missing_ckpt_vocab_and_hf_paths():
    with pytest.raises(FileNotFoundError, match="ckpt_file is required") as e:
        infer_cli.load_cli_model(_settings([]))
    assert str(e.value) == api.CKPT_REQUIRED
    with pytest.raises(FileNotFoundError, match="vocab_file is required"):
        infer_cli.load_cli_model(_settings(["-p", "model.safetensors", "-m", "F5TTS_Base"]))
    with pytest.raises(FileNotFoundError, match="hf:// paths are not downloaded"):
        infer_cli.load_cli_model(_settings(["-p", "hf://SWivid/F5-TTS/F5TTS_v1_Base/model_1250000.safetensors"]))
    with pytest.raises(FileNotFoundError, match="hf:// paths are not downloaded"):
        infer_cli.load_cli_model(_settings(["-p", "m.pt", "-v", "hf://SWivid/F5-TTS/vocab.txt"]))
    with pytest.raises(ValueError, match="unknown model"):
        infer_cli.load_cli_model(_settings(["-p", "m.pt", "-m", "F5TTS_Large"]))


def test_vocoder_path_errors(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError, match=re.escape("../checkpoints/vocos-mel-24khz")):
        infer_cli.load_cli_vocoder(_settings([]))
    with pytest.raises(FileNotFoundError, match=r"vocos-mel-24khz lacks config\.yaml, pytorch_model\.bin"):
        infer_cli.load_cli_vocoder(_settings(["--load_vocoder_from_local"]))
    with pytest.raises(NotImplementedError, match="only the Vocos back-end"):
        infer_cli.load_cli_vocoder(_settings(["--vocoder_name", "bigvgan"]))


def test_model_cfg_yaml(tmp_path):
    def write(backbone, arch, mel="vocos"):
        import yaml

        p = tmp_path / f"{backbone}.yaml"
        p.write_text(yaml.safe_dump({"model": {"name": "x", "backbone": backbone, "arch": arch,
                                               "mel_spec": {"mel_spec_type": mel, "target_sample_rate": 24000}}}))
        return str(p)

    cls, arch = infer_cli.model_class_and_arch(_settings([]))
    assert (cls, arch) == (api.MODEL_ARCH["F5TTS_v1_Base"][0], api.MODEL_ARCH["F5TTS_v1_Base"][1])
    dit = dict(dim=512, depth=4, heads=8, ff_mult=2, text_dim=256, text_mask_padding=True, qk_norm=None, conv_layers=4,
               pe_attn_head=None, attn_backend="torch", attn_mask_enabled=False, checkpoint_activations=False)
    assert infer_cli.model_class_and_arch(_settings(["--model_cfg", write("DiT", dit)])) == (infer_cli.DiT, dit)
    mm = dict(dim=512, depth=4, heads=8, ff_mult=2, text_mask_padding=True)
    assert infer_cli.model_class_and_arch(_settings(["-mc", write("MMDiT", mm)])) == (infer_cli.MMDiT, mm)
    un = dict(dim=512, depth=4, heads=8, ff_mult=4, text_mask_padding=False, pe_attn_head=1)
    cls, arch = infer_cli.model_class_and_arch(_settings([], {"model_cfg": write("UNetT", un)}))
    assert cls is infer_cli.UNetT and arch == un
    cls(**arch, text_num_embeds=10, mel_dim=100)  # the YAML's arguments build the backbone
    with pytest.raises(ValueError, match="model.backbone"):
        infer_cli.model_class_and_arch(_settings(["--model_cfg", write("Transformer", dit)]))
    with pytest.raises(ValueError, match="bigvgan mels"):
        infer_cli.model_class_and_arch(_settings(["--model_cfg", write("DiT", dit, mel="bigvgan")]))


def test_empty_ref_text_asks_for_asr(tmp_path, golden_dir):
    ref = str(tmp_path / "ref.wav")
    shutil.copy(os.path.join(golden_dir, "basic_ref_en.wav"), ref)
    config = infer_cli.load_config(os.path.join(golden_dir, "story.toml"))
    config["gen_file"] = os.path.join(golden_dir, "story.txt")
    for v in config["voices"].values():
        v["ref_audio"] = ref
    with pytest.raises(NotImplementedError, match="ASR"):
        infer_cli.prepare_voices(_settings(["-r", ref], config), config)


def test_non_wav_reference_audio(tmp_path):
    bad = tmp_path / "main.flac"
    bad.write_bytes(b"fLaC\x00\x00\x00\x22" + bytes(40))
    with pytest.raises(ValueError, match="16-bit PCM wav"):
        infer_cli.prepare_voices(_settings(["-r", str(bad)]), {})


# ------------------------------------------------------------------------------------- main, with stand-ins
def test_main_voices_speeds_and_files(tmp_path, golden_dir, monkeypatch):
    """main() with the loaders and `infer_process` replaced: every piece goes to its voice's preprocessed prompt with
    its voice's speed, in order; the output is the concatenation, the chunks are the pieces."""
    main_wav, town_wav = str(tmp_path / "main.wav"), str(tmp_path / "town.wav")
    shutil.copy(os.path.join(golden_dir, "basic_ref_en.wav"), main_wav)
    _write_raw(town_wav, _signal([("tone", 1500)], 24000), 24000)
    (tmp_path / "cfg.toml").write_text(
        'ref_text = "Main voice."\nspeed = 1.1\nnfe_step = 4\n'
        f'[voices.town]\nref_audio = "{town_wav}"\nref_text = "Town voice"\nspeed = 0.8\n')
    calls = []

    def fake_infer_process(ref_audio, ref_text, gen_text, model_obj, vocoder, **kw):
        calls.append((ref_audio, ref_text, gen_text, kw["speed"], kw["nfe_step"], kw["mel_spec_type"]))
        return np.full(1000 + 10 * len(calls), 0.01 * len(calls), np.float32), 24000, None

    monkeypatch.setattr(infer_cli._infer, "infer_process", fake_infer_process)
    monkeypatch.setattr(infer_cli, "load_cli_vocoder", lambda s: "vocoder")
    monkeypatch.setattr(infer_cli, "load_cli_model", lambda s: "model")
    out = tmp_path / "out"
    infer_cli.main(["-c", str(tmp_path / "cfg.toml"), "-r", main_wav, "-o", str(out), "-w", "story.wav",
                    "--save_chunk", "-t", "First. [town] Second “one”. [main] Third. [nobody] Fourth."])
    assert calls == [(main_wav, "Main voice. ", "First.", 1.1, 4, "vocos"),
                     (town_wav, "Town voice. ", "Second “one”.", 0.8, 4, "vocos"),
                     (main_wav, "Main voice. ", "Third.", 1.1, 4, "vocos"),
                     (main_wav, "Main voice. ", "Fourth.", 1.1, 4, "vocos")]
    segs = [np.full(1000 + 10 * k, 0.01 * k, np.float32) for k in range(1, 5)]
    (r, c, w), pcm = _read_raw(str(out / "story.wav"))
    assert (r, c, w) == (24000, 1, 2)
    assert np.array_equal(pcm[:, 0], (np.concatenate(segs) * 32767.0).astype(np.int16))
    names = sorted(os.listdir(out / "story_chunks"))
    assert names == ["0_First..wav", "1_Second one..wav", "2_Third..wav", "3_Fourth..wav"]
    for k, name in enumerate(["0_First..wav", "1_Second one..wav", "2_Third..wav", "3_Fourth..wav"]):
        _, chunk = _read_raw(str(out / "story_chunks" / name))
        assert np.array_equal(chunk[:, 0], (segs[k] * 32767.0).astype(np.int16))
