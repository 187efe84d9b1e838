"""CPU model of the engine's fp16 storage — TEST INFRASTRUCTURE ONLY (same rules as oracle/f5_oracle.py).

The engine keeps the residual streams, norms, softmax statistics and every accumulator in fp32, and stores only GEMM
operands and a few intermediates as fp16.  This module runs the unchanged oracle forwards (oracle/f5_oracle.py,
arch_options.py, unett_skip.py, mmdit.py), normally in float64, with exactly those values rounded to fp16:

(a) the parameters weights.packed_tensors stores through ``_h`` (``fp16_weight_keys``); the ``_f`` ones (text table,
    dwconv, norm gains, GRN, biases, qk-norm gains) stay as they are;
(b) the activations at each point where csrc/engine.cu stores a ``__half`` (``fp16_storage``):
    * every GEMM A operand, i.e. every linear's input: ``xin`` (engine.cu:89-90, the input projection), ``a`` (:52, the
      normalised copy read by QKV, FF1 and proj_out), ``ao`` (:52, attention output), ``g`` (:52, FF hidden), ``cat``
      (:97, the UNetT skip and DiT long-skip concat), ``temb_silu`` (:81, the AdaLN table GEMM, :853-859), ``ta`` and
      ``tg`` (:86, the text blocks' pointwise GEMMs) — except the two time-MLP linears, whose inputs ``tfeat`` and
      ``th1`` are fp32 (:80, run_small_linear at :850-851);
    * the grouped conv position embedding's inputs ``h0h`` and ``c1`` (:92, conv1 / conv2 at :590-614), not the text
      blocks' depthwise conv, which reads the fp32 ``tx`` (:84);
    * q, k and v after qk-norm and RoPE (``qkv``, :52, written by the QKV GEMM's epilogue at :517-531);
    * the GELU outputs: FF1's ``g`` and the text blocks' GRN input ``tg`` (:907-915; GRN rewrites ``tg`` in place,
      and pwconv2 reads it as an A operand).
Everything else is computed in the state dict's dtype.  What this leaves out — fp32 accumulation order in the GEMMs,
the attention kernel's fp16 probabilities and its online softmax, fast-math transcendentals — is the part of the
engine's error this model does not predict; tests compare the engine with this model's error by a measured factor.
"""
from __future__ import annotations

import contextlib
import types

import torch
import torch.nn.functional as TF

from oracle import arch_options as OA
from oracle import f5_oracle as O
from oracle import mmdit as OMM
from oracle import unett_skip as OU

# the oracle modules whose `F` (torch.nn.functional) fp16_storage replaces while it is active
MODULES = (O, OA, OU, OMM)
_TIME_MLP = ("transformer.time_embed.time_mlp.0.weight", "transformer.time_embed.time_mlp.2.weight")


def to_fp16(x: torch.Tensor) -> torch.Tensor:
    """Round to the nearest fp16 value (ties to even, subnormals kept, |x| > 65504 -> inf) and back to x's dtype."""
    return x.to(torch.float16).to(x.dtype)


def fp16_weight_keys(sd: dict) -> list:
    """The keys of `sd` that weights.packed_tensors stores as fp16: every GEMM weight matrix (time MLP, text
    pwconv1/pwconv2, input projection, conv position embedding, QKV, out-projection, FF, UNetT skip_proj, AdaLN
    linears, proj_out, long skip), i.e. every weight of two or more axes except the text table and the text blocks'
    depthwise conv (and the 1-d norm gains, which are fp32 too)."""
    return [k for k, v in sd.items() if k.endswith(".weight") and v.ndim >= 2
            and not k.endswith("text_embed.text_embed.weight") and not k.endswith("dwconv.weight")]


def engine_state_dict(sd: dict, dtype=torch.float64, rnd=to_fp16) -> dict:
    """`sd` in `dtype`, with the engine's fp16 parameters passed through `rnd` (part (a) above)."""
    keys = set(fp16_weight_keys(sd))
    return {k: (rnd(v.to(dtype)) if k in keys else v.to(dtype)) for k, v in sd.items()}


def _functional(sd: dict, rnd) -> types.SimpleNamespace:
    keep = {id(sd[k]) for k in _TIME_MLP if k in sd}  # linears whose input stays fp32

    def linear(x, w, b=None):
        return TF.linear(x if id(w) in keep else rnd(x), w, b)

    def conv1d(x, w, b=None, *args, **kw):
        grouped_pos = w.shape[-1] == 31  # ConvPositionEmbedding (k = 31); the text dwconv has k = 7
        return TF.conv1d(rnd(x) if grouped_pos else x, w, b, *args, **kw)

    def scaled_dot_product_attention(q, k, v, *args, **kw):
        return TF.scaled_dot_product_attention(rnd(q), rnd(k), rnd(v), *args, **kw)

    def gelu(x, approximate="none"):
        return rnd(TF.gelu(x, approximate=approximate))

    ns = types.SimpleNamespace(**{n: getattr(TF, n) for n in dir(TF) if not n.startswith("__")})
    ns.linear, ns.conv1d, ns.scaled_dot_product_attention, ns.gelu = linear, conv1d, scaled_dot_product_attention, gelu
    return ns


@contextlib.contextmanager
def fp16_storage(sd: dict, rnd=to_fp16):
    """Inside the block the oracle forwards round the engine's fp16 activations (part (b) above) with `rnd`.  `sd` is
    the state dict the forwards will be called with (its time-MLP weights are recognised by identity).  The modules'
    own `F` is restored on exit, also when the block raises."""
    ns = _functional(sd, rnd)
    saved = [m.F for m in MODULES]
    try:
        for m in MODULES:
            m.F = ns
        yield ns
    finally:
        for m, f in zip(MODULES, saved):
            m.F = f


def forward(sd, cfg, x, cond, text, time, mask, cfg_infer: bool):
    """The backbone operator transformer(x, cond, text, time, mask, cfg_infer=...) of any config, text embeddings
    included: DiT through oracle/arch_options (which equals oracle/f5_oracle with the options off), UNetT through
    oracle/unett_skip, MMDiT through oracle/mmdit.  Computed in sd's dtype (x, cond and time are cast to it)."""
    dt = next(iter(sd.values())).dtype
    x, cond, time = x.to(dt), cond.to(dt), time.to(dt)
    N = x.shape[1]
    if cfg.backbone == "DiT":
        seq = mask.sum(1) if mask is not None else N
        te = tuple(OA.text_embedding_dit(sd, cfg, text, seq, d) for d in (False, True))
        return OA.dit_forward(sd, cfg, x, cond, te, time, mask, cfg_infer)
    if cfg.backbone == "UNetT":
        te = tuple(O.text_embedding_unett(sd, cfg, text, N, d) for d in (False, True))
        return OU.unett_forward(sd, cfg, x, cond, te, time, mask, cfg_infer)
    te = tuple(OMM.text_embedding(sd, cfg, text, d) for d in (False, True))
    return OMM.mmdit_forward(sd, cfg, x, cond, text, te, time, mask, cfg_infer)


# ---------------------------------------------------------------------------------------------------------------------
# stress weights: synthdata's weights with attention made peaked and position-sensitive and every block's contribution
# made O(1), so that wiring errors in attention, RoPE and masking move the output well past the fp16 noise
# ---------------------------------------------------------------------------------------------------------------------
def stress_configs() -> dict:
    """Real widths, short stacks: the backbones and options the frame tests cover."""
    import synthdata as SD

    def with_(cfg, **kw):
        for k, v in kw.items():
            setattr(cfg, k, v)
        return cfg

    return {
        "f5base": with_(SD.f5tts_base(), depth=4),
        "f5v1": with_(SD.f5tts_v1_base(), depth=4),
        "e2_concat": with_(SD.e2tts_base(), depth=4),
        "e2_add": with_(SD.e2tts_base(), depth=4, skip_connect_type="add"),
        "mmdit": with_(SD.mmdit_v1_base_widths(), depth=3),
        "dh128": with_(SD.f5tts_v1_base_dh128(), depth=3),
        "options": with_(SD.f5tts_v1_base_all_options(), depth=4, pe_attn_head=1),
        "small": with_(SD.f5tts_v1_small(), depth=4),
    }


def stress_state_dict(cfg, seed: int = 1234, beta: float = 2.0, gate: float = 1.0, qk_gain: float = 1.6,
                      roped_out: float = 4.0) -> dict:
    """synthdata.synthetic_state_dict(cfg, seed) with four changes (fp32, like the original):

    * the q and k biases of the roped heads are one shared vector of N(0, beta^2) entries per head (MMDiT: the text
      stream's q_c / k_c biases too, the same vector), so q . k has a term sum_i |u_i|^2 cos((m - n) theta_i): every
      roped head attends mostly to its neighbours, and a position error changes which ones;
    * qk-norm gains are multiplied by qk_gain (qk-norm divides the bias out otherwise);
    * the AdaLN gates gate_msa and gate_mlp get +gate on their bias, so each DiT / MMDiT block adds O(1) to its stream;
    * with fewer roped heads than heads (pe_attn_head), the out-projection columns of the roped heads are multiplied by
      roped_out, so RoPE still moves the output."""
    import synthdata as SD

    sd = SD.synthetic_state_dict(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    H, dh, D = cfg.heads, cfg.dim_head, cfg.dim
    pn = H if (cfg.pe_attn_head is None or cfg.backbone == "MMDiT") else cfg.pe_attn_head
    for k in list(sd):
        if k.endswith("to_q.bias"):
            base = k[: -len("to_q.bias")]
            u = beta * torch.randn(pn * dh, generator=g)
            for nm in ("to_q.bias", "to_k.bias", "to_q_c.bias", "to_k_c.bias"):
                if base + nm in sd:
                    sd[base + nm][: pn * dh] = u
        elif k.endswith(("q_norm.weight", "k_norm.weight")):
            sd[k] = sd[k] * qk_gain
        elif k.endswith("to_out.0.weight") and pn < H:
            sd[k][:, : pn * dh] *= roped_out
        elif k.endswith(("attn_norm.linear.bias", "attn_norm_x.linear.bias", "attn_norm_c.linear.bias")) \
                and sd[k].numel() == 6 * D:
            sd[k][2 * D:3 * D] += gate  # gate_msa (modules.py:323 chunk order)
            sd[k][5 * D:6 * D] += gate  # gate_mlp
    return sd
