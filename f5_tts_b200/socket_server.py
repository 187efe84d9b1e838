"""Streaming TCP front door on top of the H100 sampler — mirror of the reference's ``f5_tts/socket_server.py`` (wire
protocol and chunking policy), SURVEY.md §8(f)-3.

Wire protocol (socket_server.py:150-177): the client sends UTF-8 text (at most 1024 bytes per request) on a TCP
connection; the server answers with the synthesised audio as raw little-endian float32 samples, sent in pieces of at
most 2048 samples as they become available, and terminates each request with the three bytes ``END``.  The connection
stays open for further requests; closing it resets the "first package" state.

Chunking policy (socket_server.py:116-140): the text is cut into chunks sized for the reference voice's speaking rate
(``max_chars`` = bytes of reference text per second of reference audio x (25 s - reference length)); the FIRST chunk
of a connection is cut again at half and then a quarter of that size so that the first audio leaves early.

What differs from the reference, by necessity of this image: model architectures come from ``api.MODEL_ARCH`` (no
hydra / omegaconf), the reference wave is read with the stdlib reader of ``infer._load_wav`` (no torchaudio codec),
checkpoints / vocoder are local paths (no network).  Sampling runs through ``infer.infer_batch_process(...,
streaming=True)``, i.e. the same kernels as every other entry point.  Each client's chunks are B = 1 sampler calls made
from that client's thread; ``--batch_clients`` merges the calls of concurrent clients into shared engine calls
(``CFM.enable_batching``); the wire protocol is unchanged and each call computes what it would compute alone.
"""
from __future__ import annotations

import argparse
import logging
import queue
import socket
import struct
import threading
import traceback
import wave

import numpy as np
import torch

from . import api as _api
from . import infer as _infer

logger = logging.getLogger(__name__)
END_MARKER = b"END"
REQUEST_BYTES = 1024
CHUNK_SAMPLES = 2048


class AudioFileWriterThread(threading.Thread):
    """Writes the streamed chunks to a 16-bit wav without holding up the sender (socket_server.py:32-70)."""

    def __init__(self, output_file, sampling_rate):
        super().__init__(daemon=True)
        self.output_file, self.sampling_rate = output_file, sampling_rate
        self.queue: queue.Queue = queue.Queue()
        self.stop_event = threading.Event()

    def run(self):
        with wave.open(self.output_file, "wb") as wf:
            wf.setnchannels(1)
            wf.setsampwidth(2)
            wf.setframerate(self.sampling_rate)
            while not self.stop_event.is_set() or not self.queue.empty():
                try:
                    chunk = self.queue.get(timeout=0.1)
                except queue.Empty:
                    continue
                if chunk is not None:
                    wf.writeframes(np.int16(np.asarray(chunk) * 32767).tobytes())

    def add_chunk(self, chunk):
        self.queue.put(chunk)

    def stop(self):
        self.stop_event.set()
        self.join()


class TTSStreamingProcessor:
    """socket_server.py:72-148.  `model` names an entry of api.MODEL_ARCH; `model_obj` / `vocoder` may be passed in
    ready-made (tests, embedding into a larger server) instead of being loaded from `ckpt_file` / `vocoder_local_path`."""

    def __init__(self, model, ckpt_file, vocab_file, ref_audio, ref_text, device=None, dtype=torch.float32,
                 vocoder_local_path=None, model_obj=None, vocoder=None, output_file=None):
        self.device = device or _infer.device
        self.mel_spec_type = "vocos"
        self.sampling_rate = _infer.target_sample_rate
        if model_obj is None:
            model_cls, model_arc = _api.MODEL_ARCH[model]
            model_obj = _infer.load_model(model_cls, model_arc, ckpt_path=ckpt_file, mel_spec_type=self.mel_spec_type,
                                          vocab_file=vocab_file, ode_method="euler", use_ema=True,
                                          device=self.device).to(self.device, dtype=dtype)
        self.model = model_obj
        self.vocoder = vocoder if vocoder is not None else _infer.load_vocoder(
            self.mel_spec_type, vocoder_local_path is not None, vocoder_local_path, self.device)
        self.output_file = output_file  # None: no wav copy of the stream is kept (the reference always writes output.wav)
        self.update_reference(ref_audio, ref_text)
        self._warm_up()
        self.file_writer_thread = None
        self.first_package = True

    def update_reference(self, ref_audio, ref_text):
        self.ref_audio, self.ref_text = _infer.preprocess_ref_audio_text(ref_audio, ref_text)
        self.audio, self.sr = _infer._load_wav(self.ref_audio) if isinstance(self.ref_audio, str) else self.ref_audio
        seconds = self.audio.shape[-1] / self.sr
        rate = len(self.ref_text.encode("utf-8")) / seconds
        self.max_chars = int(rate * (25 - seconds))
        self.few_chars = int(rate * (25 - seconds) / 2)
        self.min_chars = int(rate * (25 - seconds) / 4)

    def _stream(self, text_batches):
        return _infer.infer_batch_process((self.audio, self.sr), self.ref_text, text_batches, self.model, self.vocoder,
                                          progress=None, device=self.device, streaming=True, chunk_size=CHUNK_SAMPLES)

    def _warm_up(self):
        for _ in self._stream(["Warm-up text for the model."]):
            pass

    def plan_chunks(self, text):
        batches = _infer.chunk_text(text, max_chars=self.max_chars)
        if self.first_package and batches:
            batches = _infer.chunk_text(batches[0], max_chars=self.few_chars) + batches[1:]
            batches = _infer.chunk_text(batches[0], max_chars=self.min_chars) + batches[1:]
            self.first_package = False
        return batches

    def generate_stream(self, text, conn):
        if self.file_writer_thread is not None:
            self.file_writer_thread.stop()
            self.file_writer_thread = None
        if self.output_file:
            self.file_writer_thread = AudioFileWriterThread(self.output_file, self.sampling_rate)
            self.file_writer_thread.start()
        for audio_chunk, _ in self._stream(self.plan_chunks(text)):
            if len(audio_chunk) > 0:
                conn.sendall(np.asarray(audio_chunk, dtype="<f4").tobytes())  # == struct.pack(f"{n}f", *chunk)
                if self.file_writer_thread is not None:
                    self.file_writer_thread.add_chunk(audio_chunk)
        conn.sendall(END_MARKER)
        if self.file_writer_thread is not None:
            self.file_writer_thread.stop()
            self.file_writer_thread = None


def handle_client(conn, processor):
    """socket_server.py:150-177: one request per recv(1024); an empty read ends the session."""
    try:
        with conn:
            conn.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)
            while True:
                data = conn.recv(REQUEST_BYTES)
                if not data:
                    processor.first_package = True
                    break
                try:
                    processor.generate_stream(data.decode("utf-8").strip(), conn)
                except Exception as inner:  # noqa: BLE001
                    logger.error("error during processing: %s", inner)
                    traceback.print_exc()
                    break
    except Exception as e:  # noqa: BLE001
        logger.error("error handling client: %s", e)
        traceback.print_exc()


def start_server(host, port, processor, ready: threading.Event | None = None, stop: threading.Event | None = None):
    """socket_server.py:180-189: accept loop, one thread per client.  `ready` / `stop` let a test run it in-process."""
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        s.bind((host, port))
        s.listen()
        s.settimeout(0.2)
        if ready is not None:
            ready.port = s.getsockname()[1]
            ready.set()
        while stop is None or not stop.is_set():
            try:
                conn, _addr = s.accept()
            except socket.timeout:
                continue
            threading.Thread(target=handle_client, args=(conn, processor), daemon=True).start()


def receive_stream(sock) -> np.ndarray:
    """Client side of the protocol: float32 samples until the END marker (the reference's socket_client.py logic)."""
    buf = b""
    while not buf.endswith(END_MARKER):
        data = sock.recv(8192)
        if not data:
            break
        buf += data
    payload = buf[: -len(END_MARKER)] if buf.endswith(END_MARKER) else buf
    return np.frombuffer(payload[: len(payload) // 4 * 4], dtype="<f4")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", default="0.0.0.0")
    ap.add_argument("--port", default=9998, type=int)
    ap.add_argument("--model", default="F5TTS_v1_Base")
    ap.add_argument("--ckpt_file", required=True)
    ap.add_argument("--vocab_file", required=True)
    ap.add_argument("--vocoder_local_path", required=True)
    ap.add_argument("--ref_audio", required=True)
    ap.add_argument("--ref_text", required=True)
    ap.add_argument("--device", default=None)
    ap.add_argument("--dtype", default=torch.float32)
    ap.add_argument("--batch_clients", action="store_true",
                    help="merge the sampler calls of concurrent clients into shared engine calls (CFM.enable_batching)")
    a = ap.parse_args()
    logging.basicConfig(level=logging.INFO)
    proc = TTSStreamingProcessor(a.model, a.ckpt_file, a.vocab_file, a.ref_audio, a.ref_text, device=a.device,
                                 dtype=a.dtype, vocoder_local_path=a.vocoder_local_path, output_file="output.wav")
    if a.batch_clients:
        proc.model.enable_batching()
    start_server(a.host, a.port, proc)


if __name__ == "__main__":
    main()
