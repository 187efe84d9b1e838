"""Re-pack a loaded ``state_dict`` (released checkpoint layout) into the kernels' operand layouts.

 * GEMM weights -> fp16, row-major [N, K] (K-major operands for wgmma); to_q|to_k|to_v stacked into one
   [3*inner, D] matrix so QKV is a single GEMM; all AdaLN linears of a DiT stacked into one
   [depth*6D + 2D, D] matrix (rows per block in the reference's chunk order shift_msa, scale_msa, gate_msa,
   shift_mlp, scale_mlp, gate_mlp — model/modules.py:323; final: scale, shift — modules.py:344);
 * input_embed.proj K padded with zero columns to a multiple of 64;
 * grouped Conv1d(k=31, g=16) weight [D, G, 31] -> [31][D][G], G = D/16 channels per group, so that tap t / group g
   is a K-major G x G block (64 x 64 at D = 1024);
 * biases, norm gains, GRN parameters, embedding table -> fp32;
 * MMDiT: the audio stream fills the per-layer slots of DiT (audio_embed.linear is the input projection, its K = 2*mel
   zero-padded to 256), the text stream goes to `C{i}.*` (to_q_c|to_k_c|to_v_c stacked), and the AdaLN table is
   [attn_norm_x 6D | attn_norm_c 6D (2D in the last block)] per block, then norm_out.
The packed tensors are owned by Python (kept alive in the returned dict); the C engine only stores pointers.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def _h(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float16).contiguous()


def _f(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def packed_tensors(m) -> dict[str, torch.Tensor]:
    """Every operand the engine reads, in kernel layout, as a flat name -> tensor dict (the unit that is cached on disk).
    Names: `time_w0`, `text_table`, `tb{i}.pw1_w`, `proj_w`, `conv_w{0,1}`, `L{i}.w_qkv`, `C{i}.w_qkv_c`, `mod_w`,
    `out_w`, ..."""
    sd = {k: v for k, v in m.state_dict().items()}
    dev = next(m.parameters()).device
    if dev.type != "cuda":
        raise _lib.F5LibraryError("the backbone must live on a CUDA (H100) device before sampling; no CPU path exists")
    D, depth = m.dim, m.depth
    mmdit, unett = m.KIND == "MMDiT", m.KIND == "UNetT"
    T: dict[str, torch.Tensor] = {}
    T["time_w0"], T["time_b0"] = _h(sd["time_embed.time_mlp.0.weight"]), _f(sd["time_embed.time_mlp.0.bias"])
    T["time_w1"], T["time_b1"] = _h(sd["time_embed.time_mlp.2.weight"]), _f(sd["time_embed.time_mlp.2.bias"])
    T["text_table"] = _f(sd["text_embed.text_embed.weight"])
    for i in range(m.conv_layers):
        p, q = f"text_embed.text_blocks.{i}.", f"tb{i}."
        T[q + "dw_w"], T[q + "dw_b"] = _f(sd[p + "dwconv.weight"].reshape(m.text_dim, 7)), _f(sd[p + "dwconv.bias"])
        T[q + "ln_w"], T[q + "ln_b"] = _f(sd[p + "norm.weight"]), _f(sd[p + "norm.bias"])
        T[q + "pw1_w"], T[q + "pw1_b"] = _h(sd[p + "pwconv1.weight"]), _f(sd[p + "pwconv1.bias"])
        T[q + "grn_gamma"], T[q + "grn_beta"] = _f(sd[p + "grn.gamma"].reshape(-1)), _f(sd[p + "grn.beta"].reshape(-1))
        T[q + "pw2_w"], T[q + "pw2_b"] = _h(sd[p + "pwconv2.weight"]), _f(sd[p + "pwconv2.bias"])
    embed, proj = ("audio_embed.", "audio_embed.linear.") if mmdit else ("input_embed.", "input_embed.proj.")
    pw = sd[proj + "weight"]
    kin = pw.shape[1]
    kpad = (kin + 63) // 64 * 64
    pwp = torch.zeros((D, kpad), dtype=torch.float16, device=dev)
    pwp[:, :kin] = pw.to(torch.float16)
    T["proj_w"], T["proj_b"] = pwp, _f(sd[proj + "bias"])
    for j, idx in enumerate((0, 2)):
        cw = sd[f"{embed}conv_pos_embed.conv1d.{idx}.weight"]  # [D_out, G, 31]
        T[f"conv_w{j}"] = _h(cw.permute(2, 0, 1))              # [31, D_out, G]
        T[f"conv_b{j}"] = _f(sd[f"{embed}conv_pos_embed.conv1d.{idx}.bias"])
    mod = []  # AdaLN linears in table order (DiT, MMDiT)
    for i in range(depth):
        q = f"L{i}."
        if unett:
            p, a, f = f"layers.{i}.", f"layers.{i}.2.", f"layers.{i}.4."
        else:
            p, a = f"transformer_blocks.{i}.", f"transformer_blocks.{i}.attn."
            f = p + ("ff_x." if mmdit else "ff.")
        T[q + "w_qkv"] = _h(torch.cat([sd[a + "to_q.weight"], sd[a + "to_k.weight"], sd[a + "to_v.weight"]], dim=0))
        T[q + "b_qkv"] = _f(torch.cat([sd[a + "to_q.bias"], sd[a + "to_k.bias"], sd[a + "to_v.bias"]], dim=0))
        T[q + "w_out"], T[q + "b_out"] = _h(sd[a + "to_out.0.weight"]), _f(sd[a + "to_out.0.bias"])
        T[q + "w_ff1"], T[q + "b_ff1"] = _h(sd[f + "ff.0.0.weight"]), _f(sd[f + "ff.0.0.bias"])
        T[q + "w_ff2"], T[q + "b_ff2"] = _h(sd[f + "ff.2.weight"]), _f(sd[f + "ff.2.bias"])
        if unett:
            if (p + "0.weight") in sd:
                T[q + "w_skip"] = _h(sd[p + "0.weight"])
            T[q + "g_attn"], T[q + "g_ff"] = _f(sd[p + "1.g"]), _f(sd[p + "3.g"])
        if m.qk_norm is not None:
            T[q + "q_norm_w"], T[q + "k_norm_w"] = _f(sd[a + "q_norm.weight"]), _f(sd[a + "k_norm.weight"])
        if not mmdit:
            mod.append(p + "attn_norm.linear.")
            continue
        c = f"C{i}."  # the text stream; the last block has only its QKV (context_pre_only)
        T[c + "w_qkv_c"] = _h(torch.cat([sd[a + "to_q_c.weight"], sd[a + "to_k_c.weight"], sd[a + "to_v_c.weight"]], 0))
        T[c + "b_qkv_c"] = _f(torch.cat([sd[a + "to_q_c.bias"], sd[a + "to_k_c.bias"], sd[a + "to_v_c.bias"]], 0))
        if i < depth - 1:
            T[c + "w_out_c"], T[c + "b_out_c"] = _h(sd[a + "to_out_c.weight"]), _f(sd[a + "to_out_c.bias"])
            T[c + "w_ff1_c"], T[c + "b_ff1_c"] = _h(sd[p + "ff_c.ff.0.0.weight"]), _f(sd[p + "ff_c.ff.0.0.bias"])
            T[c + "w_ff2_c"], T[c + "b_ff2_c"] = _h(sd[p + "ff_c.ff.2.weight"]), _f(sd[p + "ff_c.ff.2.bias"])
        if m.qk_norm is not None:
            T[c + "q_norm_c"], T[c + "k_norm_c"] = _f(sd[a + "c_q_norm.weight"]), _f(sd[a + "c_k_norm.weight"])
        mod += [p + "attn_norm_x.linear.", p + "attn_norm_c.linear."]
    if unett:
        T["g_out"] = _f(sd["norm_out.g"])
    else:
        mod.append("norm_out.linear.")
        T["mod_w"] = _h(torch.cat([sd[k + "weight"] for k in mod], dim=0))
        T["mod_b"] = _f(torch.cat([sd[k + "bias"] for k in mod], dim=0))
    T["out_w"], T["out_b"] = _h(sd["proj_out.weight"]), _f(sd["proj_out.bias"])
    if m.long_skip:
        T["long_skip_w"] = _h(sd["long_skip_connection.weight"])
    return T


def engine_from_packed(m, T: dict[str, torch.Tensor]) -> dict:
    """Create the C engine over already-packed tensors (fresh from `packed_tensors` or read back from the disk cache)."""
    dev = next(iter(T.values())).device
    depth = m.depth
    dit = m.KIND != "UNetT"  # DiT and MMDiT: AdaLN table
    P = lambda k: T[k].data_ptr() if k in T else None  # noqa: E731
    W = _lib.Weights()
    W.time_w0, W.time_b0, W.time_w1, W.time_b1 = P("time_w0"), P("time_b0"), P("time_w1"), P("time_b1")
    W.text_table = P("text_table")
    for i in range(m.conv_layers):
        tb, q = W.text_blocks[i], f"tb{i}."
        for name in ("dw_w", "dw_b", "ln_w", "ln_b", "pw1_w", "pw1_b", "grn_gamma", "grn_beta", "pw2_w", "pw2_b"):
            setattr(tb, name, P(q + name))
    W.proj_w, W.proj_b, W.proj_kpad = P("proj_w"), P("proj_b"), T["proj_w"].shape[1]
    for j in range(2):
        W.conv_w[j], W.conv_b[j] = P(f"conv_w{j}"), P(f"conv_b{j}")
    layers = (_lib.LayerWeights * depth)()
    for i in range(depth):
        lw, q = layers[i], f"L{i}."
        for name in ("w_qkv", "b_qkv", "w_out", "b_out", "w_ff1", "b_ff1", "w_ff2", "b_ff2", "w_skip", "g_attn", "g_ff",
                     "q_norm_w", "k_norm_w"):
            setattr(lw, name, P(q + name))
    W.layers = C.cast(layers, C.POINTER(_lib.LayerWeights))
    if dit:
        W.mod_w, W.mod_b = P("mod_w"), P("mod_b")
    else:
        W.g_out = P("g_out")
    W.out_w, W.out_b = P("out_w"), P("out_b")
    W.long_skip_w = P("long_skip_w")
    ctx = None
    if m.KIND == "MMDiT":
        ctx = (_lib.CtxLayerWeights * depth)()
        for i in range(depth):
            for name in ("w_qkv_c", "b_qkv_c", "w_out_c", "b_out_c", "w_ff1_c", "b_ff1_c", "w_ff2_c", "b_ff2_c",
                         "q_norm_c", "k_norm_c"):
                setattr(ctx[i], name, P(f"C{i}." + name))
        W.ctx_layers = C.cast(ctx, C.POINTER(_lib.CtxLayerWeights))

    A = _lib.Arch()
    A.backbone = _lib.BACKBONES[m.KIND]
    A.dim, A.depth, A.heads, A.dim_head, A.ff_inner = m.dim, depth, m.heads, m.dim_head, m.ff_inner
    A.mel_dim, A.text_dim, A.text_num_embeds, A.conv_layers = m.mel_dim, m.text_dim, m.text_num_embeds, m.conv_layers
    A.text_mask_padding = 1 if m.text_mask_padding else 0
    A.pe_attn_head = -1 if m.pe_attn_head is None else int(m.pe_attn_head)
    A.attn_mask_enabled = 1 if m.attn_mask_enabled else 0
    A.qk_norm = 1 if m.qk_norm is not None else 0
    A.long_skip = 1 if m.long_skip else 0
    A.text_avg_upsample = 1 if m.text_embedding_average_upsampling else 0
    A.skip_type = _lib.SKIP_TYPES[m.skip_connect_type] if m.KIND == "UNetT" else 0
    handle = C.c_void_p()
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().f5_engine_create(C.byref(A), C.byref(W), C.byref(handle)), "f5_engine_create")
    return {"handle": handle, "keep": T, "layers": layers, "ctx": ctx, "weights": W, "arch": A}


def pack_backbone(m) -> dict:
    return engine_from_packed(m, packed_tensors(m))


# ---- on-disk cache of the packed operands (SURVEY.md §8f-4) ------------------------------------------------------------
PACK_FORMAT = 1  # bump when a kernel operand layout changes


def cache_key(ckpt_path: str, m) -> str:
    """Identifies (checkpoint file, architecture, pack format): path + size + mtime of the checkpoint, arch fields."""
    import hashlib
    import os

    st = os.stat(ckpt_path)
    arch = (m.KIND, m.dim, m.depth, m.heads, m.dim_head, m.ff_inner, m.mel_dim, m.text_dim, m.text_num_embeds,
            m.conv_layers, m.text_mask_padding, m.pe_attn_head)
    options = (m.qk_norm, m.long_skip, m.text_embedding_average_upsampling)
    if any(options):  # appended only when an option is on: packed caches of other models keep their keys
        arch += options
    if m.KIND == "UNetT" and m.skip_connect_type != "concat":  # likewise: concat models keep their keys
        arch += (f"skip_connect_type={m.skip_connect_type}",)
    raw = f"{os.path.abspath(ckpt_path)}|{st.st_size}|{st.st_mtime_ns}|{arch}|fmt{PACK_FORMAT}"
    return hashlib.sha256(raw.encode()).hexdigest()[:24]


def save_packed(m, path: str) -> None:
    """Write the packed operands of `m` (already on the GPU) as one safetensors file."""
    from safetensors.torch import save_file

    st = m.engine()
    save_file({k: v.detach().cpu().contiguous() for k, v in st["keep"].items()}, path,
              metadata={"format": str(PACK_FORMAT), "kind": m.KIND})


def attach_packed(m, path: str, device) -> bool:
    """Read a packed-operand file straight onto `device` and hand it to the engine: no fp32 -> fp16 conversion, no
    concatenation / permutation kernels at load time.  Returns False (and leaves `m` untouched) if the file does not fit."""
    from safetensors import safe_open
    from safetensors.torch import load_file

    with safe_open(path, framework="pt") as f:
        meta = f.metadata() or {}
    if meta.get("format") != str(PACK_FORMAT) or meta.get("kind") != m.KIND:
        return False
    T = load_file(path, device=str(device))
    with m._engine_lock:
        if m._engine_state is not None:
            _lib.lib().f5_engine_destroy(m._engine_state["handle"])
        st = engine_from_packed(m, T)
        st["fp"] = m._fingerprint()
        m._engine_state = st
    return True
