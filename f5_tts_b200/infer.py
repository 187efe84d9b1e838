"""Inference-process layer on top of the H100 sampler — mirror of the reference's ``f5_tts.infer.utils_infer`` for the
functions on (or feeding) the hot path: same names, arguments, defaults and return values.

Reference anchors (relative to /root/reference/src/f5_tts/infer/utils_infer.py):
  module constants 52-65 · chunk_text 73-102 · load_vocoder 106-145 · load_checkpoint 190-232 · load_model 238-276 ·
  infer_process 384-434 · infer_batch_process 440-593 (``_infer_basic`` 477-520).
  remove_silence_for_generated_wav 599-608.
Out of scope here (SURVEY.md §2 rows 7, 10-12): ASR transcription, the pydub clipping of the reference audio,
matplotlib spectrogram dumps, BigVGAN.  ``preprocess_ref_audio_text`` keeps only the text normalisation of
utils_infer.py:369-376.
"""
from __future__ import annotations

import os
import re
import wave

import numpy as np
import torch

from .model import CFM, DiT, MMDiT, UNetT  # noqa: F401
from . import vocoder as _vocoder
from .vocoder import Vocos

# ------------------------------------------------------------------------------------------- constants (52-65)
target_sample_rate = 24000
n_mel_channels = 100
hop_length = 256
win_length = 1024
n_fft = 1024
mel_spec_type = "vocos"
target_rms = 0.1
cross_fade_duration = 0.15
ode_method = "euler"
nfe_step = 32
cfg_strength = 2.0
sway_sampling_coef = -1.0
speed = 1.0
fix_duration = None
device = "cuda" if torch.cuda.is_available() else "cpu"


# ------------------------------------------------------------------------------------------------ text helpers
def chunk_text(text: str, max_chars: int = 135) -> list[str]:
    """Greedy sentence packing by UTF-8 byte length (utils_infer.py:73-102)."""
    chunks, cur = [], ""
    for sentence in re.split(r"(?<=[;:,.!?])\s+|(?<=[；：，。！？])", text):
        if not sentence:
            continue
        piece = sentence + " " if len(sentence[-1].encode("utf-8")) == 1 else sentence
        if len(cur.encode("utf-8")) + len(sentence.encode("utf-8")) <= max_chars:
            cur += piece
        else:
            if cur:
                chunks.append(cur.strip())
            cur = piece
    if cur:
        chunks.append(cur.strip())
    return chunks


def get_tokenizer(dataset_name: str, tokenizer: str = "custom"):
    """'custom' (path to vocab.txt) and 'byte' tokenizers of model/utils.py:112-142."""
    if tokenizer == "byte":
        return None, 256
    if tokenizer != "custom":
        raise NotImplementedError("pass the vocab.txt path with tokenizer='custom' (dataset-relative lookup not mirrored)")
    vocab = {}
    with open(dataset_name, "r", encoding="utf-8") as f:
        for i, line in enumerate(f):
            vocab[line[:-1]] = i
    return vocab, len(vocab)


_RE_HAN_DEFAULT = re.compile(r"([\u4E00-\u9FD5a-zA-Z0-9+#&\._%\-]+)")  # jieba: blocks that go through the word graph
_RE_SKIP_DEFAULT = re.compile(r"(\r\n|\s)")                            # jieba: separators kept between blocks
_RE_FINALSEG_SKIP = re.compile(r"([a-zA-Z0-9]+(?:\.\d+)?%?)")           # jieba.finalseg: latin / number runs


def _segment_no_chinese(text: str) -> list[str]:
    """Segmentation jieba's `cut(text, HMM=True)` (and its Rust port rjieba, model/utils.py:160) produces for text WITHOUT
    Chinese characters, restated from jieba's published algorithm (jieba/__init__.py `cut` / `__cut_DAG`,
    jieba/finalseg `cut`; the package is absent from this image): the text is split into blocks of
    [han letters digits + # & . _ % -]; such a block is unknown to the dictionary, so it goes to finalseg, which
    splits it into latin / number runs — a decimal part and a trailing % stay attached ("3.14", "50%") — and the
    characters between them; everything else is emitted whitespace by whitespace, character by character.
    Not covered: the handful of ASCII entries of jieba's dictionary ("C++", "AT&T"), which jieba keeps whole."""
    out: list[str] = []
    for blk in _RE_HAN_DEFAULT.split(text):
        if not blk:
            continue
        if _RE_HAN_DEFAULT.fullmatch(blk):
            out.extend(x for x in _RE_FINALSEG_SKIP.split(blk) if x)
        else:
            for x in _RE_SKIP_DEFAULT.split(blk):
                if _RE_SKIP_DEFAULT.fullmatch(x):
                    out.append(x)
                else:
                    out.extend(x)
    return out


def convert_char_to_pinyin(text_list, polyphone=True):
    """model/utils.py:148-185.  With rjieba + pypinyin installed this is the reference's function line for line; this
    image has neither, so non-Chinese text is segmented by `_segment_no_chinese` (jieba's algorithm restated — decimals
    and quoted words included) and Chinese text raises a clear error instead of silently producing different tokens."""
    trans = str.maketrans({";": ",", "“": '"', "”": '"', "‘": "'", "’": "'"})
    try:
        import rjieba
        from pypinyin import Style, lazy_pinyin

        if not callable(getattr(rjieba, "cut", None)):  # an empty stand-in module is not the package
            rjieba = None
    except Exception:  # noqa: BLE001
        rjieba = None

    def is_chinese(c):
        return "\u3100" <= c <= "\u9fff"

    out = []
    for text in text_list:
        text = text.translate(trans)
        chars: list[str] = []
        if rjieba is None:
            if any(is_chinese(c) for c in text):
                raise RuntimeError("Chinese text needs the rjieba + pypinyin packages (text front-end, out of scope)")
            segs = _segment_no_chinese(text)
        else:
            segs = rjieba.cut(text)
        for seg in segs:
            nbytes = len(bytes(seg, "UTF-8"))
            if nbytes == len(seg):  # pure alphabets and symbols
                if chars and nbytes > 1 and chars[-1] not in " :'\"":
                    chars.append(" ")
                chars.extend(seg)
            elif rjieba is not None and polyphone and nbytes == 3 * len(seg):
                py = lazy_pinyin(seg, style=Style.TONE3, tone_sandhi=True)
                for i, c in enumerate(seg):
                    if is_chinese(c):
                        chars.append(" ")
                    chars.append(py[i])
            else:
                for c in seg:
                    if ord(c) < 256:
                        chars.extend(c)
                    elif is_chinese(c):
                        chars.append(" ")
                        chars.extend(lazy_pinyin(c, style=Style.TONE3, tone_sandhi=True))
                    else:
                        chars.append(c)
        out.append(chars)
    return out


# ------------------------------------------------------------------------------------------------ loading
def load_vocoder(vocoder_name="vocos", is_local=False, local_path="", device=device, hf_cache_dir=None):
    """utils_infer.py:106-145 for vocoder_name='vocos' (config.yaml + pytorch_model.bin of charactr/vocos-mel-24khz)."""
    if vocoder_name != "vocos":
        raise NotImplementedError("only the Vocos back-end is on the H100 path (BigVGAN: SURVEY.md §2 row 16)")
    if is_local:
        config_path, model_path = f"{local_path}/config.yaml", f"{local_path}/pytorch_model.bin"
    else:
        from huggingface_hub import hf_hub_download

        repo_id = "charactr/vocos-mel-24khz"
        config_path = hf_hub_download(repo_id=repo_id, cache_dir=hf_cache_dir, filename="config.yaml")
        model_path = hf_hub_download(repo_id=repo_id, cache_dir=hf_cache_dir, filename="pytorch_model.bin")
    vocoder = Vocos.from_hparams(config_path)
    state_dict = torch.load(model_path, map_location="cpu", weights_only=True)
    vocoder.load_state_dict(state_dict)
    return vocoder.eval().to(device)


def load_checkpoint(model, ckpt_path, device: str, dtype=None, use_ema=True):
    """utils_infer.py:190-232: .safetensors (flat EMA dict) or .pt; strips the `ema_model.` prefix, drops
    `initted`/`step` and the legacy mel_spec buffers; fp16 parameters on CUDA like the reference."""
    if dtype is None:
        dtype = torch.float16 if "cuda" in str(device) else torch.float32
    model = model.to(dtype)
    ckpt_type = ckpt_path.split(".")[-1]
    if ckpt_type == "safetensors":
        from safetensors.torch import load_file

        checkpoint = load_file(ckpt_path, device=str(device))
    else:
        checkpoint = torch.load(ckpt_path, map_location=device, weights_only=True)
    if use_ema:
        if ckpt_type == "safetensors":
            checkpoint = {"ema_model_state_dict": checkpoint}
        sd = {k.replace("ema_model.", ""): v for k, v in checkpoint["ema_model_state_dict"].items()
              if k not in ("initted", "step")}
        for key in ("mel_spec.mel_stft.mel_scale.fb", "mel_spec.mel_stft.spectrogram.window"):
            sd.pop(key, None)
    else:
        sd = checkpoint if ckpt_type == "safetensors" else checkpoint["model_state_dict"]
    model.load_state_dict(sd)
    return model.to(device)


def load_model(model_cls, model_cfg, ckpt_path, mel_spec_type=mel_spec_type, vocab_file="", ode_method=ode_method,
               use_ema=True, device=device, packed_cache_dir=None, cfg_parallel_device=None,
               sample_parallel_devices=None):
    """utils_infer.py:238-276.  `packed_cache_dir` (extra, default off): keep the kernel-layout operands of this
    checkpoint (fp16 K-major weights, stacked QKV / AdaLN matrices, re-tiled conv weights; weights.py) in that folder and
    read them straight onto the GPU on later loads instead of re-packing 0.67 GB through conversion kernels.
    `cfg_parallel_device` (extra, default off): run the unconditional CFG half of every sampler call on that GPU
    (CFM.enable_cfg_parallel).  `sample_parallel_devices` (extra, default off): run the samples of every batched sampler
    call in groups on those GPUs (CFM.enable_sample_parallel)."""
    if vocab_file == "":
        raise FileNotFoundError("vocab_file is required (the reference defaults to its packaged "
                                "infer/examples/vocab.txt, utils_infer.py:248-249; that data file is not vendored here)")
    vocab_char_map, vocab_size = get_tokenizer(vocab_file, "custom")
    model = CFM(
        transformer=model_cls(**model_cfg, text_num_embeds=vocab_size, mel_dim=n_mel_channels),
        mel_spec_kwargs=dict(n_fft=n_fft, hop_length=hop_length, win_length=win_length, n_mel_channels=n_mel_channels,
                             target_sample_rate=target_sample_rate, mel_spec_type=mel_spec_type),
        odeint_kwargs=dict(method=ode_method),
        vocab_char_map=vocab_char_map,
    ).to(device)
    if ckpt_path:
        model = load_checkpoint(model, ckpt_path, device, dtype=None, use_ema=use_ema)
        if packed_cache_dir and "cuda" in str(device):
            from . import weights as _w

            os.makedirs(packed_cache_dir, exist_ok=True)
            path = os.path.join(packed_cache_dir, f"f5pack_{_w.cache_key(ckpt_path, model.transformer)}.safetensors")
            if not (os.path.exists(path) and _w.attach_packed(model.transformer, path, device)):
                _w.save_packed(model.transformer, path)
    if cfg_parallel_device is not None:
        model.enable_cfg_parallel(cfg_parallel_device)
    if sample_parallel_devices is not None:
        model.enable_sample_parallel(sample_parallel_devices)
    return model


def preprocess_ref_audio_text(ref_audio_orig, ref_text, show_info=print):
    """Text normalisation of utils_infer.py:369-376 (the audio clipping / ASR part needs pydub + whisper: not mirrored)."""
    if not ref_text.strip():
        raise NotImplementedError("empty ref_text would trigger ASR transcription in the reference (out of scope)")
    if not ref_text.endswith(". ") and not ref_text.endswith("。"):
        ref_text += " " if ref_text.endswith(".") else ". "
    return ref_audio_orig, ref_text


def _load_wav(path):
    """(float32 [channels, n], sample_rate) for 16-bit PCM wav via the stdlib (torchaudio.load needs a codec backend)."""
    with wave.open(path, "rb") as f:
        sr, ch, width, n = f.getframerate(), f.getnchannels(), f.getsampwidth(), f.getnframes()
        raw = f.readframes(n)
    if width != 2:
        raise NotImplementedError("only 16-bit PCM wav is read natively")
    data = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    return torch.from_numpy(data.reshape(-1, ch).T.copy()), sr


def _write_wav(path, wav, sample_rate=target_sample_rate):
    """Mono 16-bit PCM wav of a float waveform: clipped to [-1, 1], scaled by 32767 and truncated toward zero."""
    pcm = (np.clip(np.asarray(wav), -1.0, 1.0) * 32767.0).astype("<i2")
    with wave.open(path, "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sample_rate)
        f.writeframes(pcm.tobytes())


# ------------------------------------------------------------------------------------------------ silence removal
def _ms_to_frame(ms, rate):
    """pydub's millisecond -> frame position (AudioSegment._parse_position: int(frame_count(ms=ms)))."""
    return (np.asarray(ms, dtype=np.float64) * (rate / 1000.0)).astype(np.int64)


def _pydub_len(n_frames, rate):
    """len(AudioSegment) in milliseconds: round(1000 * frames / rate), Python's round (half to even)."""
    return round(1000 * (float(n_frames) / rate))


def _slice_frames(pcm, rate, start_ms, end_ms):
    """AudioSegment[start_ms:end_ms] on [n, channels] int16 frames.  Both ends are clamped to len(segment); an end
    that the millisecond rounding puts past the last frame is filled with zero frames, as pydub does, unless the slice
    is empty."""
    seg_len = _pydub_len(len(pcm), rate)
    fs, fe = (int(v) for v in _ms_to_frame([min(start_ms, seg_len), min(end_ms, seg_len)], rate))
    data = pcm[fs:fe]
    if 0 < len(data) < fe - fs:
        data = np.concatenate([data, np.zeros((fe - fs - len(data), pcm.shape[1]), pcm.dtype)])
    return data


def _silence_window_rms(pcm, rate, min_silence_len=1000, seek_step=10):
    """(window starts in ms, audioop.rms of each window) for pydub's `detect_silence` scan: windows of
    `min_silence_len` ms every `seek_step` ms, plus a final window ending at len(segment) when the steps miss it.

    The RMS is audioop.rms's: the integer part of sqrt(sum of squares / samples) over every sample of every channel
    in the window, zero for an empty window.  The sums come from int64 prefix sums of squares, so the scan is O(n);
    they convert to float64 exactly while a window has fewer than 2**23 samples, as audioop's double accumulator
    does."""
    seg_len = _pydub_len(len(pcm), rate)
    last = seg_len - min_silence_len
    starts = list(range(0, last + 1, seek_step))
    if last % seek_step:
        starts.append(last)
    sq = np.square(pcm.astype(np.int64)).sum(axis=1)
    prefix = np.concatenate([np.zeros(1, np.int64), np.cumsum(sq)])
    s = np.asarray(starts, dtype=np.int64)
    fs = _ms_to_frame(np.minimum(s, seg_len), rate)
    fe = _ms_to_frame(np.minimum(s + min_silence_len, seg_len), rate)
    n = len(pcm)
    lo, hi = np.minimum(fs, n), np.minimum(fe, n)
    frames = np.where(hi > lo, np.maximum(fe - fs, 0), 0)  # zero-filled ends count as samples (_slice_frames)
    total = (prefix[hi] - prefix[lo]).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        rms = np.where(frames > 0, np.floor(np.sqrt(total / (frames * pcm.shape[1]))), 0.0)
    return starts, rms.astype(np.int64)


def _split_on_silence(pcm, rate, min_silence_len=1000, silence_thresh=-50, keep_silence=500, seek_step=10):
    """pydub.silence.split_on_silence on [n, channels] int16 frames: the list of kept [m, channels] pieces.

    Restated from pydub 0.25's published `detect_silence` / `detect_nonsilent` / `split_on_silence` (pydub is not a
    dependency of this package): a window is silent when its RMS is at most db_to_float(silence_thresh) * 32768; consecutive silent
    windows merge into ranges; the non-silent ranges between them are padded by `keep_silence` ms each way, and two
    padded ranges that overlap are split at their midpoint."""
    seg_len = _pydub_len(len(pcm), rate)
    silent = []
    if seg_len >= min_silence_len:
        thresh = 10 ** (float(silence_thresh) / 20) * 32768.0
        starts, rms = _silence_window_rms(pcm, rate, min_silence_len, seek_step)
        silence_starts = [i for i, r in zip(starts, rms) if r <= thresh]
        if silence_starts:
            prev = cur = silence_starts[0]
            for i in silence_starts[1:]:
                if i != prev + seek_step and i > prev + min_silence_len:
                    silent.append([cur, prev + min_silence_len])
                    cur = i
                prev = i
            silent.append([cur, prev + min_silence_len])
    if not silent:
        nonsilent = [[0, seg_len]]
    elif silent[0] == [0, seg_len]:
        nonsilent = []
    else:
        nonsilent, prev_end = [], 0
        for start, end in silent:
            nonsilent.append([prev_end, start])
            prev_end = end
        if silent[-1][1] != seg_len:
            nonsilent.append([prev_end, seg_len])
        if nonsilent[0] == [0, 0]:
            nonsilent.pop(0)
    ranges = [[start - keep_silence, end + keep_silence] for start, end in nonsilent]
    for a, b in zip(ranges, ranges[1:]):
        if b[0] < a[1]:
            a[1] = (a[1] + b[0]) // 2
            b[0] = a[1]
    return [_slice_frames(pcm, rate, max(start, 0), min(end, seg_len)) for start, end in ranges]


def remove_silence_for_generated_wav(filename):
    """utils_infer.py:599-608: cut every silence of 1 s or more in a 16-bit wav down to 0.5 s on each side, in place.

    The reference runs pydub's split_on_silence(min_silence_len=1000, silence_thresh=-50, keep_silence=500,
    seek_step=10), concatenates the pieces and writes the file back.  pydub is not a dependency here, so its loop logic
    (window placement, range merging, padding, midpoint split, millisecond-to-frame rounding) is restated in
    `_split_on_silence`; the window RMS is pinned against `audioop.rms` itself, window by window.  The file keeps its
    rate, channel count and width.  (pydub concatenates onto an empty 11025 Hz segment, so it would write a result at
    11025 Hz when the input rate is lower or every piece is dropped.)"""
    with wave.open(filename, "rb") as f:
        rate, ch, width = f.getframerate(), f.getnchannels(), f.getsampwidth()
        raw = f.readframes(f.getnframes())
    if width != 2:
        raise NotImplementedError("only 16-bit PCM wav is read natively")
    pcm = np.frombuffer(raw, dtype="<i2").reshape(-1, ch)
    pieces = _split_on_silence(pcm, rate)
    out = np.concatenate(pieces) if pieces else pcm[:0]
    with wave.open(filename, "wb") as f:
        f.setnchannels(ch)
        f.setsampwidth(2)
        f.setframerate(rate)
        f.writeframes(out.astype("<i2").tobytes())


# ------------------------------------------------------------------------------------------------ inference
def infer_process(ref_audio, ref_text, gen_text, model_obj, vocoder, mel_spec_type=mel_spec_type, show_info=print,
                  progress=None, target_rms=target_rms, cross_fade_duration=cross_fade_duration, nfe_step=nfe_step,
                  cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef, speed=speed,
                  fix_duration=fix_duration, device=device):
    """utils_infer.py:384-434: chunk the text by the reference-audio speaking rate, then run the batch process."""
    audio, sr = _load_wav(ref_audio) if isinstance(ref_audio, str) else ref_audio
    secs = audio.shape[-1] / sr
    max_chars = int(len(ref_text.encode("utf-8")) / secs * (22 - secs) * speed)
    gen_text_batches = chunk_text(gen_text, max_chars=max_chars)
    show_info(f"Generating audio in {len(gen_text_batches)} batches...")
    if not gen_text_batches:
        return None, target_sample_rate, None
    return next(infer_batch_process((audio, sr), ref_text, gen_text_batches, model_obj, vocoder,
                                    mel_spec_type=mel_spec_type, progress=progress, target_rms=target_rms,
                                    cross_fade_duration=cross_fade_duration, nfe_step=nfe_step, cfg_strength=cfg_strength,
                                    sway_sampling_coef=sway_sampling_coef, speed=speed, fix_duration=fix_duration,
                                    device=device))


def cross_fade_concat(waves: list, fade: int):
    """utils_infer.py:549-585 on tensors that stay where they are (device or host): sequentially, the tail of the running
    result and the head of the next chunk are blended over `fade` samples with linear ramps."""
    final = waves[0]
    for nxt in waves[1:]:
        n = min(fade, final.shape[-1], nxt.shape[-1])
        if n <= 0:
            final = torch.cat([final, nxt])
            continue
        ramp = torch.linspace(0.0, 1.0, n, device=final.device, dtype=final.dtype)
        mixed = final[-n:] * (1.0 - ramp) + nxt[:n] * ramp
        final = torch.cat([final[:-n], mixed, nxt[n:]])
    return final


MAX_CHUNK_BATCH = 16  # text chunks per batched sampler call


def infer_batch_process(ref_audio, ref_text, gen_text_batches, model_obj, vocoder, mel_spec_type="vocos", progress=None,
                        target_rms=0.1, cross_fade_duration=0.15, nfe_step=32, cfg_strength=2.0, sway_sampling_coef=-1,
                        speed=1, fix_duration=None, device=None, streaming=False, chunk_size=2048):
    """utils_infer.py:440-593 — generator yielding (final_wave, sr, spectrogram) or streaming (chunk, sr).

    The reference samples every text chunk in its own B = 1 call from a thread pool (utils_infer.py:540-541) and
    cross-fades the chunks on the host.  Here all chunks of a request go through ONE batched sampler call
    (`exact_varlen=True`: each chunk is computed exactly as if it were alone, so the result equals the per-chunk loop),
    sharing the prompt mel; the vocoder output, RMS gain and cross-fade stay on the device and the finished waveform
    crosses to the host once."""
    if mel_spec_type != "vocos":
        raise NotImplementedError("bigvgan mel/vocoder is out of scope")
    audio, sr = ref_audio
    if audio.shape[0] > 1:
        audio = torch.mean(audio, dim=0, keepdim=True)
    rms = torch.sqrt(torch.mean(torch.square(audio)))
    if rms < target_rms:
        audio = audio * target_rms / rms
    if sr != target_sample_rate:
        import torchaudio

        audio = torchaudio.transforms.Resample(sr, target_sample_rate)(audio)
    audio = audio.to(device)
    if len(ref_text[-1].encode("utf-8")) == 1:
        ref_text = ref_text + " "
    ref_audio_len = audio.shape[-1] // hop_length

    def plan(gen_text):  # duration heuristic of `_infer_basic`, utils_infer.py:477-493
        local_speed = 0.3 if len(gen_text.encode("utf-8")) < 10 else speed
        if fix_duration is not None:
            return int(fix_duration * target_sample_rate / hop_length)
        ref_text_len, gen_text_len = len(ref_text.encode("utf-8")), len(gen_text.encode("utf-8"))
        return ref_audio_len + int(ref_audio_len / ref_text_len * gen_text_len / local_speed)

    def synth(gen_texts):
        """[(wave tensor [n], generated mel tensor [100, frames])] for a group of chunks — one sampler call."""
        tokens = convert_char_to_pinyin([ref_text + t for t in gen_texts])
        durations = [plan(t) for t in gen_texts]
        with torch.inference_mode():
            if len(gen_texts) == 1:
                generated, _ = model_obj.sample(cond=audio, text=tokens, duration=durations[0], steps=nfe_step,
                                                cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef)
                # the sampler may lengthen a chunk (cfm.py:134-137): the row count is its answer
                durations = [generated.shape[1]]
            else:
                cond = model_obj.mel_spec(audio, frames_last=False)  # prompt mel, once: [1, n_ref, 100]
                cond = cond.expand(len(gen_texts), -1, -1).contiguous()
                dur = torch.tensor(durations, dtype=torch.long, device=cond.device)
                lens = torch.full((len(gen_texts),), cond.shape[1], dtype=torch.long, device=cond.device)
                n_text = [len(t) for t in tokens]
                durations = [max(max(nt, cond.shape[1]) + 1, d) for nt, d in zip(n_text, durations)]  # cfm.py:134-137
                generated, _ = model_obj.sample(cond=cond, text=tokens, duration=dur, lens=lens, steps=nfe_step,
                                                cfg_strength=cfg_strength, sway_sampling_coef=sway_sampling_coef,
                                                exact_varlen=True)
            mels = [generated[i, ref_audio_len:d, :].to(torch.float32).permute(1, 0) for i, d in enumerate(durations)]
            out = []
            # one vocoder call for the group: each chunk's audio is bit-identical to decoding its mel alone
            for wave_out, mel in zip(_vocoder.decode_each(vocoder, mels), mels):
                if rms < target_rms:
                    wave_out = wave_out * rms / target_rms
                out.append((wave_out, mel))
            return out

    batches = list(gen_text_batches)
    if streaming:
        it = progress.tqdm(batches) if progress is not None else batches
        for gen_text in it:
            wave_np = synth([gen_text])[0][0].cpu().numpy()
            for j in range(0, len(wave_np), chunk_size):
                yield wave_np[j: j + chunk_size], target_sample_rate
        return

    groups = [batches[i: i + MAX_CHUNK_BATCH] for i in range(0, len(batches), MAX_CHUNK_BATCH)]
    results = []
    for grp in (progress.tqdm(groups) if progress is not None else groups):
        results.extend(synth(grp))
    if not results:
        yield None, target_sample_rate, None
        return
    fade = int(cross_fade_duration * target_sample_rate) if cross_fade_duration > 0 else 0
    final = cross_fade_concat([w for w, _ in results], fade)
    spec = torch.cat([m for _, m in results], dim=1)
    yield final.cpu().numpy(), target_sample_rate, spec.cpu().numpy()
