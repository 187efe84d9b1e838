"""f5_tts_b200 — H100-native (sm_90a) implementation of the F5-TTS / E2-TTS ODE-sampling hot path.

Drop-in surface (same names / signatures as the reference's f5_tts package for this path):
    f5_tts_b200.model.{CFM, DiT, UNetT, MMDiT, MelSpec}     <- f5_tts.model
    f5_tts_b200.vocoder.Vocos                          <- vocos.Vocos (decode)
    f5_tts_b200.infer.{load_model, load_vocoder, load_checkpoint, infer_process, infer_batch_process, ...}
    f5_tts_b200.api.F5TTS                              <- f5_tts.api.F5TTS
All arithmetic runs in libf5tts_b200.so (include/f5tts_b200.h); importing the package does not load it, calling any
operator does, and raises if it is missing — there is no CPU or PyTorch fallback.
"""
from . import _lib  # noqa: F401
from .model import CFM, DiT, MelSpec, MMDiT, UNetT  # noqa: F401

__all__ = ["CFM", "DiT", "UNetT", "MMDiT", "MelSpec"]
__version__ = "0.1.0"
