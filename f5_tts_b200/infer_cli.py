"""Command-line inference — mirror of the reference's ``f5_tts/infer/infer_cli.py`` (``f5-tts_infer-cli``): one text,
or a multi-voice story, to one wav file.

    python -m f5_tts_b200.infer_cli -c story.toml -p model_1250000.safetensors -v vocab.txt --load_vocoder_from_local

Same flags and short forms (infer_cli.py:36-175), TOML keys, defaults and precedence (infer_cli.py:187-223): a flag
wins over the config, and a falsy flag value (``--speed 0``, ``--cfg_strength 0``) falls back to the config, as in the
reference.  ``--no_legacy_text`` is a store_false flag there, and so it is here.  A text splits into pieces at voice
tags (``[town] ...``); each piece runs through ``infer.infer_process`` with its voice's prompt and speed, one after
another, and the pieces are concatenated without a cross-fade (infer_cli.py:307-384).

What differs from the reference, because this package depends on none of hydra, omegaconf, cached_path, soundfile,
tomli, unidecode and pydub, and downloads nothing:
- The config is read with ``tomllib``.  The reference's packaged ``basic.toml`` is not shipped: without ``-c`` the
  config is empty and the reference's fallbacks apply.  Paths under ``infer/examples/`` are not resolved against
  package data.
- Architectures come from ``api.MODEL_ARCH``, or from ``--model_cfg``: a YAML file in the layout of the reference's
  ``configs/*.yaml``, read with PyYAML, whose ``model.backbone`` picks ``DiT``, ``UNetT`` or ``MMDiT`` and whose
  ``model.arch`` gives its arguments.
- ``--ckpt_file`` and ``--vocab_file`` are required local paths; ``hf://`` paths raise, since nothing is downloaded.
  The vocoder is read from the reference's local path ``../checkpoints/vocos-mel-24khz`` with
  ``--load_vocoder_from_local`` and is not downloaded without it.
- Reference audio is read by ``infer._load_wav``: 16-bit PCM wav only.  The reference's ``examples/multi/*.flac``
  must be converted to wav first.
- Files are written as 16-bit PCM by the writer of ``F5TTS.export_wav``; ``remove_silence`` then trims the output
  with ``infer.remove_silence_for_generated_wav``.  Legacy ``--save_chunk`` file names use ``unidecode`` when it is
  installed, and otherwise keep the ASCII characters of the text's NFKD form (accents are dropped, other non-ASCII
  characters are removed).
- A voice tag with no text after it is skipped; the reference fails on the empty result of such a piece.
"""
from __future__ import annotations

import argparse
import os
import re
import tomllib
import unicodedata
import wave
from datetime import datetime
from pathlib import Path
from types import SimpleNamespace

import numpy as np

from . import api as _api
from . import infer as _infer
from .model import DiT, MMDiT, UNetT

BACKBONES = {"DiT": DiT, "UNetT": UNetT, "MMDiT": MMDiT}
VOCODER_LOCAL_PATHS = {"vocos": "../checkpoints/vocos-mel-24khz",  # infer_cli.py:256-259
                       "bigvgan": "../checkpoints/bigvgan_v2_24khz_100band_256x"}
VOICE_SPLIT = r"(?=\[\w+\])"  # infer_cli.py:323-325
VOICE_TAG = r"\[(\w+)\]"

parser = argparse.ArgumentParser(
    prog="python -m f5_tts_b200.infer_cli",
    description="Commandline interface for E2/F5 TTS with Advanced Batch Processing.",
    epilog="Specify options above to override one or more settings from config.",
)
parser.add_argument("-c", "--config", type=str, default=None,
                    help="The configuration file (TOML), default none: every setting takes its default")
# no defaults below, so that the config file's values apply (infer_cli.py:49)
parser.add_argument("-m", "--model", type=str, help="The model name: F5TTS_v1_Base | F5TTS_Base | E2TTS_Base | etc.")
parser.add_argument("-mc", "--model_cfg", type=str, help="The path to F5-TTS model config file .yaml")
parser.add_argument("-p", "--ckpt_file", type=str, help="The path to model checkpoint .pt or .safetensors (required)")
parser.add_argument("-v", "--vocab_file", type=str, help="The path to vocab file .txt (required)")
parser.add_argument("-r", "--ref_audio", type=str, help="The reference audio file (16-bit PCM wav).")
parser.add_argument("-s", "--ref_text", type=str, help="The transcript/subtitle for the reference audio")
parser.add_argument("-t", "--gen_text", type=str, help="The text to make model synthesize a speech")
parser.add_argument("-f", "--gen_file", type=str, help="The file with text to generate, will ignore --gen_text")
parser.add_argument("-o", "--output_dir", type=str, help="The path to output folder")
parser.add_argument("-w", "--output_file", type=str, help="The name of output file")
parser.add_argument("--save_chunk", action="store_true", help="To save each audio chunks during inference")
parser.add_argument("--no_legacy_text", action="store_false",
                    help="Not to use lossy ASCII transliterations of unicode text in saved file names.")
parser.add_argument("--remove_silence", action="store_true", help="To remove long silence found in ouput")
parser.add_argument("--load_vocoder_from_local", action="store_true",
                    help=f"To load vocoder from local dir, default to {VOCODER_LOCAL_PATHS['vocos']}")
parser.add_argument("--vocoder_name", type=str, choices=["vocos", "bigvgan"],
                    help=f"Used vocoder name: vocos | bigvgan, default {_infer.mel_spec_type}")
parser.add_argument("--target_rms", type=float,
                    help=f"Target output speech loudness normalization value, default {_infer.target_rms}")
parser.add_argument("--cross_fade_duration", type=float,
                    help=f"Duration of cross-fade between audio segments in seconds, default {_infer.cross_fade_duration}")
parser.add_argument("--nfe_step", type=int,
                    help=f"The number of function evaluation (denoising steps), default {_infer.nfe_step}")
parser.add_argument("--cfg_strength", type=float,
                    help=f"Classifier-free guidance strength, default {_infer.cfg_strength}")
parser.add_argument("--sway_sampling_coef", type=float,
                    help=f"Sway Sampling coefficient, default {_infer.sway_sampling_coef}")
parser.add_argument("--speed", type=float, help=f"The speed of the generated audio, default {_infer.speed}")
parser.add_argument("--fix_duration", type=float,
                    help=f"Fix the total duration (ref and gen audios) in seconds, default {_infer.fix_duration}")
parser.add_argument("--device", type=str, help="Specify the device to run on")


def load_config(path):
    """The TOML config as a dict; empty without ``-c``."""
    if not path:
        return {}
    with open(path, "rb") as f:
        return tomllib.load(f)


def resolve(args, config):
    """Settings from flags over config over defaults, with the reference's ``args.x or config.get(...)`` rule
    (infer_cli.py:187-223); ``gen_file``, when set, replaces ``gen_text`` with its contents."""
    d = _infer
    s = SimpleNamespace()
    s.model = args.model or config.get("model", "F5TTS_v1_Base")
    s.model_cfg = args.model_cfg or config.get("model_cfg", "")
    s.ckpt_file = args.ckpt_file or config.get("ckpt_file", "")
    s.vocab_file = args.vocab_file or config.get("vocab_file", "")
    s.ref_audio = args.ref_audio or config.get("ref_audio", "infer/examples/basic/basic_ref_en.wav")
    s.ref_text = (args.ref_text if args.ref_text is not None
                  else config.get("ref_text", "Some call me nature, others call me mother nature."))
    s.gen_text = args.gen_text or config.get("gen_text", "Here we generate something just for test.")
    s.gen_file = args.gen_file or config.get("gen_file", "")
    s.output_dir = args.output_dir or config.get("output_dir", "tests")
    s.output_file = args.output_file or config.get("output_file",
                                                   f"infer_cli_{datetime.now().strftime(r'%Y%m%d_%H%M%S')}.wav")
    s.save_chunk = args.save_chunk or config.get("save_chunk", False)
    s.use_legacy_text = args.no_legacy_text or config.get("no_legacy_text", False)  # store_false flag
    s.remove_silence = args.remove_silence or config.get("remove_silence", False)
    s.load_vocoder_from_local = args.load_vocoder_from_local or config.get("load_vocoder_from_local", False)
    s.vocoder_name = args.vocoder_name or config.get("vocoder_name", d.mel_spec_type)
    s.target_rms = args.target_rms or config.get("target_rms", d.target_rms)
    s.cross_fade_duration = args.cross_fade_duration or config.get("cross_fade_duration", d.cross_fade_duration)
    s.nfe_step = args.nfe_step or config.get("nfe_step", d.nfe_step)
    s.cfg_strength = args.cfg_strength or config.get("cfg_strength", d.cfg_strength)
    s.sway_sampling_coef = args.sway_sampling_coef or config.get("sway_sampling_coef", d.sway_sampling_coef)
    s.speed = args.speed or config.get("speed", d.speed)
    s.fix_duration = args.fix_duration or config.get("fix_duration", d.fix_duration)
    s.device = args.device or config.get("device", d.device)
    if s.gen_file:
        with open(s.gen_file, "r", encoding="utf-8", newline="") as f:
            s.gen_text = f.read()
    s.wave_path = Path(s.output_dir) / s.output_file
    s.chunk_dir = os.path.join(s.output_dir, f"{Path(s.output_file).stem}_chunks")
    return s


def split_voices(gen_text, voices):
    """[(voice, text)] in order: the text split before every ``[name]`` tag, the tag removed and the text stripped.
    Untagged text and unknown voices go to ``main`` (infer_cli.py:322-342)."""
    pieces = []
    for text in re.split(VOICE_SPLIT, gen_text):
        if not text.strip():
            continue
        match = re.match(VOICE_TAG, text)
        if match:
            voice = match[1]
        else:
            print("No voice tag found, using main.")
            voice = "main"
        if voice not in voices:
            print(f"Voice {voice} not found, using main.")
            voice = "main"
        text = re.sub(VOICE_TAG, "", text).strip()
        if text:
            pieces.append((voice, text))
    return pieces


def _ascii_fold(text):
    try:
        from unidecode import unidecode
    except ImportError:
        return unicodedata.normalize("NFKD", text).encode("ascii", "ignore").decode("ascii")
    return unidecode(text)


def chunk_file_name(index, text, use_legacy_text):
    """``<index>_<text>.wav`` of ``--save_chunk`` (infer_cli.py:362-371): text over 200 characters is cut to 200 and
    followed by " ... "; legacy names are folded to ASCII."""
    if len(text) > 200:
        text = text[:200] + " ... "
    if use_legacy_text:
        text = _ascii_fold(text)
    return f"{index}_{text}.wav"


def prepare_voices(s, config):
    """``main`` from ref_audio / ref_text plus the config's ``[voices.<name>]`` tables, each through
    ``preprocess_ref_audio_text`` once (infer_cli.py:308-320).  An empty ref_text raises, as ASR is not mirrored."""
    voices = {name: dict(v) for name, v in config.get("voices", {}).items()}
    voices["main"] = {"ref_audio": s.ref_audio, "ref_text": s.ref_text}
    for name, v in voices.items():
        print("Voice:", name)
        print("ref_audio ", v["ref_audio"])
        try:
            _infer._load_wav(v["ref_audio"])
        except wave.Error as e:
            raise ValueError(f"{v['ref_audio']}: reference audio must be 16-bit PCM wav ({e})") from None
        v["ref_audio"], v["ref_text"] = _infer.preprocess_ref_audio_text(v["ref_audio"], v["ref_text"])
        print("ref_audio_", v["ref_audio"], "\n\n")
    return voices


def load_cli_vocoder(s):
    """infer_cli.py:256-263, from the reference's local vocoder path only."""
    path = VOCODER_LOCAL_PATHS.get(s.vocoder_name, "")
    if s.vocoder_name == "vocos":
        if not s.load_vocoder_from_local:
            raise FileNotFoundError(f"the vocoder is not downloaded: put charactr/vocos-mel-24khz's config.yaml and "
                                    f"pytorch_model.bin in {path} and pass --load_vocoder_from_local")
        missing = [f for f in ("config.yaml", "pytorch_model.bin") if not os.path.isfile(os.path.join(path, f))]
        if missing:
            raise FileNotFoundError(f"--load_vocoder_from_local: {path} lacks {', '.join(missing)}")
    return _infer.load_vocoder(vocoder_name=s.vocoder_name, is_local=s.load_vocoder_from_local, local_path=path,
                               device=s.device)


def model_class_and_arch(s):
    """(backbone class, constructor arguments): from ``--model_cfg`` when given, else ``api.MODEL_ARCH[model]``."""
    if not s.model_cfg:
        if s.model not in _api.MODEL_ARCH:
            raise ValueError(f"unknown model {s.model!r}; shipped configs: {sorted(_api.MODEL_ARCH)}; "
                             "pass --model_cfg for others")
        cls, arch = _api.MODEL_ARCH[s.model]
        return cls, dict(arch)
    import yaml

    with open(s.model_cfg, "r", encoding="utf-8") as f:
        cfg = yaml.safe_load(f)["model"]
    if cfg["backbone"] not in BACKBONES:
        raise ValueError(f"model.backbone {cfg['backbone']!r} in {s.model_cfg}: expected one of {sorted(BACKBONES)}")
    mel_type = cfg.get("mel_spec", {}).get("mel_spec_type", _infer.mel_spec_type)
    if s.model != "F5TTS_Base" and mel_type != s.vocoder_name:  # infer_cli.py:276-277
        raise ValueError(f"{s.model_cfg} is trained on {mel_type} mels, but the vocoder is {s.vocoder_name}")
    return BACKBONES[cfg["backbone"]], dict(cfg["arch"])


def load_cli_model(s):
    """infer_cli.py:268-301 with local files only."""
    for name in ("ckpt_file", "vocab_file"):
        if getattr(s, name).startswith("hf://"):
            raise FileNotFoundError(f"{name} {getattr(s, name)!r}: hf:// paths are not downloaded; pass a local file")
    if not s.ckpt_file:
        raise FileNotFoundError(_api.CKPT_REQUIRED)
    cls, arch = model_class_and_arch(s)
    print(f"Using {s.model}...")
    return _infer.load_model(cls, arch, s.ckpt_file, mel_spec_type=s.vocoder_name, vocab_file=s.vocab_file,
                             device=s.device)


def main(argv=None):
    args = parser.parse_args(argv)
    config = load_config(args.config)
    s = resolve(args, config)
    if s.save_chunk and s.use_legacy_text:
        print("\nWarning to --save_chunk: lossy ASCII transliterations of unicode text for legacy (.wav) file names, "
              "--no_legacy_text to disable.\n")
    if s.save_chunk:
        os.makedirs(s.chunk_dir, exist_ok=True)
    voices = prepare_voices(s, config)
    pieces = split_voices(s.gen_text, voices)
    vocoder = load_cli_vocoder(s)
    ema_model = load_cli_model(s)

    segments, sample_rate = [], _infer.target_sample_rate
    for voice, text in pieces:
        v = voices[voice]
        print(f"Voice: {voice}")
        segment, sample_rate, _ = _infer.infer_process(
            v["ref_audio"], v["ref_text"], text, ema_model, vocoder, mel_spec_type=s.vocoder_name,
            target_rms=s.target_rms, cross_fade_duration=s.cross_fade_duration, nfe_step=s.nfe_step,
            cfg_strength=s.cfg_strength, sway_sampling_coef=s.sway_sampling_coef, speed=v.get("speed", s.speed),
            fix_duration=s.fix_duration, device=s.device)
        segments.append(segment)
        if s.save_chunk:
            name = chunk_file_name(len(segments) - 1, text, s.use_legacy_text)
            _infer._write_wav(os.path.join(s.chunk_dir, name), segment, sample_rate)

    if segments:
        os.makedirs(s.output_dir, exist_ok=True)
        _infer._write_wav(str(s.wave_path), np.concatenate(segments), sample_rate)
        if s.remove_silence:
            _infer.remove_silence_for_generated_wav(str(s.wave_path))
        print(s.wave_path)


if __name__ == "__main__":
    main()
