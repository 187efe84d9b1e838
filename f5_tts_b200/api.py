"""``F5TTS`` — mirror of the reference's top-level API class (f5_tts/api.py:23-149) over the H100 sampler.

Same constructor / ``infer`` signature and return value ``(wav np.float32[nw], sr, spec np[100, n])``.  Differences,
all forced by the offline image and the scope of this build: model configs are the six shipped architectures
(Base and Small of F5TTS_v1, F5TTS and E2TTS) hard-coded below (hydra/omegaconf are not installed; values copied from configs/*.yaml ``model.arch``); checkpoints
and the vocoder must be given as local paths (no network); ``transcribe`` and silence removal are not mirrored.
"""
from __future__ import annotations

import random
import sys

import numpy as np

from . import infer as _infer
from .model import DiT, UNetT

MODEL_ARCH = {
    # configs/F5TTS_v1_Base.yaml:26-36
    "F5TTS_v1_Base": (DiT, dict(dim=1024, depth=22, heads=16, ff_mult=2, text_dim=512, text_mask_padding=True,
                               qk_norm=None, conv_layers=4, pe_attn_head=None, attn_backend="torch",
                               attn_mask_enabled=False)),
    # configs/F5TTS_Base.yaml:25-35
    "F5TTS_Base": (DiT, dict(dim=1024, depth=22, heads=16, ff_mult=2, text_dim=512, text_mask_padding=False,
                            conv_layers=4, pe_attn_head=1, attn_backend="torch", attn_mask_enabled=False)),
    # configs/E2TTS_Base.yaml:25-31
    "E2TTS_Base": (UNetT, dict(dim=1024, depth=24, heads=16, ff_mult=4, text_mask_padding=False, pe_attn_head=1)),
    # configs/F5TTS_v1_Small.yaml:26-36
    "F5TTS_v1_Small": (DiT, dict(dim=768, depth=18, heads=12, ff_mult=2, text_dim=512, text_mask_padding=True,
                                qk_norm=None, conv_layers=4, pe_attn_head=None, attn_backend="torch",
                                attn_mask_enabled=False)),
    # configs/F5TTS_Small.yaml:25-35
    "F5TTS_Small": (DiT, dict(dim=768, depth=18, heads=12, ff_mult=2, text_dim=512, text_mask_padding=False,
                             conv_layers=4, pe_attn_head=1, attn_backend="torch", attn_mask_enabled=False)),
    # configs/E2TTS_Small.yaml:25-31
    "E2TTS_Small": (UNetT, dict(dim=768, depth=20, heads=12, ff_mult=4, text_mask_padding=False, pe_attn_head=1)),
}


def seed_everything(seed=0):
    """model/utils.py:19-26"""
    import torch

    random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


class F5TTS:
    def __init__(self, model="F5TTS_v1_Base", ckpt_file="", vocab_file="", ode_method="euler", use_ema=True,
                 vocoder_local_path=None, device=None, hf_cache_dir=None):
        if model not in MODEL_ARCH:
            raise ValueError(f"unknown model {model!r}; shipped configs: {sorted(MODEL_ARCH)}")
        model_cls, model_arc = MODEL_ARCH[model]
        self.mel_spec_type = "vocos"
        self.target_sample_rate = 24000
        self.ode_method, self.use_ema = ode_method, use_ema
        self.device = device if device is not None else _infer.device
        self.vocoder = _infer.load_vocoder(self.mel_spec_type, vocoder_local_path is not None, vocoder_local_path,
                                           self.device, hf_cache_dir)
        if not ckpt_file:
            raise FileNotFoundError("ckpt_file is required: there is no network here to fetch hf://SWivid/... "
                                    "(api.py:65-81 in the reference downloads it)")
        self.ema_model = _infer.load_model(model_cls, model_arc, ckpt_file, self.mel_spec_type, vocab_file,
                                           self.ode_method, self.use_ema, self.device)
        self.seed = None

    def export_wav(self, wav, file_wave, remove_silence=False):
        import wave

        pcm = (np.clip(np.asarray(wav), -1.0, 1.0) * 32767.0).astype("<i2")
        with wave.open(file_wave, "wb") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(self.target_sample_rate)
            f.writeframes(pcm.tobytes())

    def export_spectrogram(self, spec, file_spec):
        np.save(file_spec, spec)

    def infer(self, ref_file, ref_text, gen_text, show_info=print, progress=None, target_rms=0.1,
              cross_fade_duration=0.15, sway_sampling_coef=-1, cfg_strength=2, nfe_step=32, speed=1.0,
              fix_duration=None, remove_silence=False, file_wave=None, file_spec=None, seed=None):
        if seed is None:
            seed = random.randint(0, sys.maxsize)
        seed_everything(seed)
        self.seed = seed
        ref_file, ref_text = _infer.preprocess_ref_audio_text(ref_file, ref_text, show_info=show_info)
        wav, sr, spec = _infer.infer_process(ref_file, ref_text, gen_text, self.ema_model, self.vocoder,
                                             self.mel_spec_type, show_info=show_info, progress=progress,
                                             target_rms=target_rms, cross_fade_duration=cross_fade_duration,
                                             nfe_step=nfe_step, cfg_strength=cfg_strength,
                                             sway_sampling_coef=sway_sampling_coef, speed=speed,
                                             fix_duration=fix_duration, device=self.device)
        if file_wave is not None:
            self.export_wav(wav, file_wave, remove_silence)
        if file_spec is not None:
            self.export_spectrogram(spec, file_spec)
        return wav, sr, spec
