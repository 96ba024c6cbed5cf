"""B200TextEncoders — the T5 encoder and the CLIP text model on the device (rf_text_* in
include/rf_b200.h).

Replaces `pipe.text_encoder_2(ids)[0]` (T5-v1.1-XXL, prompt_embeds [B, 512, 4096]) and
`pipe.text_encoder(ids).pooler_output` (CLIP-L, [B, 768]) inside diffusers
FluxPipeline.encode_prompt, which train_flux/flux/generate.py:148-161 calls through
pipeline_tools.py:33-52 for every candidate prompt (each reflection candidate has its own refined
prompt: tts/tts_reflectionflow.py:286-294).  Tokenisation stays on the host (sentencepiece / BPE
vocabularies are checkpoint assets); ids go in, embeddings come out.  State-dict keys are the
transformers ones (`T5EncoderModel`, `CLIPTextModel`)."""
from __future__ import annotations

import ctypes
import math
from typing import Callable, Dict, Optional, Tuple

import torch

from . import _lib as L


class _TextCfg(ctypes.Structure):
    _fields_ = [("t5_layers", ctypes.c_int), ("t5_d_model", ctypes.c_int), ("t5_d_ff", ctypes.c_int),
                ("t5_heads", ctypes.c_int), ("t5_vocab", ctypes.c_int), ("t5_eps", ctypes.c_float),
                ("clip_layers", ctypes.c_int), ("clip_d_model", ctypes.c_int), ("clip_heads", ctypes.c_int),
                ("clip_vocab", ctypes.c_int), ("clip_max_pos", ctypes.c_int)]


T5_XXL = dict(t5_layers=24, t5_d_model=4096, t5_d_ff=10240, t5_heads=64, t5_vocab=32128, t5_eps=1e-6)
CLIP_L = dict(clip_layers=12, clip_d_model=768, clip_heads=12, clip_vocab=49408, clip_max_pos=77)


def t5_bucket_table(seq: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """[seq, seq] long: bucket of (key position - query position) for a bidirectional T5 encoder
    (transformers T5Attention._relative_position_bucket / compute_bias): half the buckets per sign;
    within a sign, distances below nb/2 get their own bucket and the rest are spaced logarithmically
    up to max_distance."""
    pos = torch.arange(seq)
    rel = pos[None, :] - pos[:, None]
    nb = num_buckets // 2
    out = (rel > 0).long() * nb
    dist = rel.abs()
    exact = nb // 2
    far = exact + (torch.log(dist.float() / exact) / math.log(max_distance / exact) * (nb - exact)).long()
    far = far.clamp(max=nb - 1)
    return out + torch.where(dist < exact, dist, far)


class B200TextEncoders:
    def __init__(self, device="cuda:0", **cfg):
        if not torch.cuda.is_available():
            raise L.RFError("B200TextEncoders needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device)
        full = dict(T5_XXL, **CLIP_L)
        full.update(cfg)
        self.cfg = full
        self._lib = L.load()
        self._h = ctypes.c_void_p()
        self._bias: Dict[int, torch.Tensor] = {}
        self._rel_bias: Optional[torch.Tensor] = None
        self.clip_eos_token_id = 2
        with torch.cuda.device(self.device):
            c = _TextCfg(**full)
            L.check(self._lib.rf_text_create(ctypes.byref(c), ctypes.byref(self._h)), "rf_text_create")

    @classmethod
    def from_pretrained(cls, text_encoder_dir: str, text_encoder_2_dir: str, device="cuda:0"):
        """The diffusers `text_encoder/` (transformers CLIPTextModel) and `text_encoder_2/` (T5EncoderModel)
        directories: shapes from their config.json (what the kernels do not implement is refused before the
        handle is created), weights streamed from their safetensors.  `clip_eos_token_id` is CLIP's
        eos_token_id, for the pooling rule of clip_encode."""
        import os
        from . import checkpoint as ck
        fields, eos = ck.text_config(ck.read_json(os.path.join(text_encoder_dir, "config.json")),
                                     ck.read_json(os.path.join(text_encoder_2_dir, "config.json")))
        clip = ck.SafetensorsStream(text_encoder_dir, ck.clip_key)
        t5 = ck.SafetensorsStream(text_encoder_2_dir, ck.t5_key)
        enc = cls(device=device, **fields)
        enc.clip_eos_token_id = eos
        return enc.load_clip_state_dict(clip).load_t5_state_dict(t5)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.rf_text_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights -------------------------------------------------------------------------------
    def _put(self, key: str, t: torch.Tensor):
        t = t.detach().to(self.device, torch.bfloat16).contiguous()
        L.check(self._lib.rf_text_load_weight(self._h, key.encode(), L.ptr(t), t.numel()),
                f"rf_text_load_weight({key})")

    _REL = "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"

    def load_t5_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """transformers T5EncoderModel keys"""
        with torch.cuda.device(self.device):
            for k, v in sd.items():
                if k == self._REL:
                    self._rel_bias = v.detach().to(self.device, torch.bfloat16)  # [buckets, heads]
                    self._bias.clear()
                elif k == "encoder.embed_tokens.weight":
                    continue  # tied to shared.weight
                else:
                    self._put("t5." + k, v)
            if strict:
                if self._rel_bias is None:
                    raise L.RFError("missing T5 weight: " + self._REL)
                if self._lib.rf_text_missing_weights(self._h, b"t5.") != 0:
                    L.check(-4, "load_t5_state_dict (missing weights)")
        return self

    def load_clip_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """transformers CLIPTextModel keys"""
        with torch.cuda.device(self.device):
            for k, v in sd.items():
                if k.endswith("position_ids"):
                    continue
                self._put("clip." + k, v)
            if strict and self._lib.rf_text_missing_weights(self._h, b"clip.") != 0:
                L.check(-4, "load_clip_state_dict (missing weights)")
        return self

    def init_synthetic_weights(self, seed: int = 0):
        """random-init encoders of the configured shape (no checkpoints exist offline); one layer's
        worth of memory at a time on the device"""
        g = torch.Generator(device=self.device).manual_seed(seed)
        c = self.cfg

        def rn(*shape, scale=1.0):
            return torch.randn(*shape, generator=g, device=self.device) * scale

        D, F, I = c["t5_d_model"], c["t5_d_ff"], c["t5_heads"] * 64
        self._put("t5.shared.weight", rn(c["t5_vocab"], D))
        for i in range(c["t5_layers"]):
            p = f"t5.encoder.block.{i}.layer."
            for n in "qkv":
                self._put(p + f"0.SelfAttention.{n}.weight", rn(I, D, scale=D ** -0.5 * (0.35 if n != "v" else 1)))
            self._put(p + "0.SelfAttention.o.weight", rn(D, I, scale=I ** -0.5))
            self._put(p + "0.layer_norm.weight", 1 + 0.1 * rn(D))
            self._put(p + "1.DenseReluDense.wi_0.weight", rn(F, D, scale=D ** -0.5))
            self._put(p + "1.DenseReluDense.wi_1.weight", rn(F, D, scale=D ** -0.5))
            self._put(p + "1.DenseReluDense.wo.weight", rn(D, F, scale=F ** -0.5))
            self._put(p + "1.layer_norm.weight", 1 + 0.1 * rn(D))
        self._put("t5.encoder.final_layer_norm.weight", 1 + 0.1 * rn(D))
        self._rel_bias = rn(32, c["t5_heads"]).to(torch.bfloat16)
        self._bias.clear()
        C = c["clip_d_model"]
        self._put("clip.text_model.embeddings.token_embedding.weight", rn(c["clip_vocab"], C, scale=0.02))
        self._put("clip.text_model.embeddings.position_embedding.weight", rn(c["clip_max_pos"], C, scale=0.01))
        for i in range(c["clip_layers"]):
            p = f"clip.text_model.encoder.layers.{i}."
            for n in ("layer_norm1", "layer_norm2"):
                self._put(p + n + ".weight", 1 + 0.1 * rn(C))
                self._put(p + n + ".bias", 0.02 * rn(C))
            for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                self._put(p + f"self_attn.{n}.weight", rn(C, C, scale=C ** -0.5))
                self._put(p + f"self_attn.{n}.bias", 0.02 * rn(C))
            self._put(p + "mlp.fc1.weight", rn(4 * C, C, scale=C ** -0.5))
            self._put(p + "mlp.fc1.bias", 0.02 * rn(4 * C))
            self._put(p + "mlp.fc2.weight", rn(C, 4 * C, scale=(4 * C) ** -0.5))
            self._put(p + "mlp.fc2.bias", 0.02 * rn(C))
        self._put("clip.text_model.final_layer_norm.weight", 1 + 0.1 * rn(C))
        self._put("clip.text_model.final_layer_norm.bias", 0.02 * rn(C))
        return self

    # ---- encode --------------------------------------------------------------------------------
    def _position_bias(self, seq: int) -> torch.Tensor:
        """[heads, seq, seq] bf16 = relative_attention_bias[bucket(j - i)], shared by every layer"""
        if seq not in self._bias:
            if self._rel_bias is None:
                raise L.RFError("T5 relative_attention_bias not loaded")
            idx = t5_bucket_table(seq).to(self.device)
            self._bias[seq] = self._rel_bias[idx].permute(2, 0, 1).contiguous()
        return self._bias[seq]

    @staticmethod
    def _check_ids(input_ids: torch.Tensor, vocab: int, what: str):
        """the embedding kernel indexes its table with the ids unchecked: refuse an id outside [0, vocab) before any
        launch (on the caller's tensor, before the copy to the device)"""
        if input_ids.numel() and (int(input_ids.min()) < 0 or int(input_ids.max()) >= vocab):
            raise L.RFError(f"{what}: token id outside [0, {vocab}) (min {int(input_ids.min())}, "
                            f"max {int(input_ids.max())})")

    def t5_encode(self, input_ids: torch.Tensor) -> torch.Tensor:
        """ids [B, S] -> last_hidden_state [B, S, d_model] bf16 (no attention mask: FLUX passes none)"""
        self._check_ids(input_ids, self.cfg["t5_vocab"], "t5_encode")
        ids = input_ids.to(self.device, torch.int32).contiguous()
        B, S = ids.shape
        out = torch.empty(B, S, self.cfg["t5_d_model"], device=self.device, dtype=torch.bfloat16)
        bias = self._position_bias(S)
        with torch.cuda.device(self.device):
            s = torch.cuda.current_stream().cuda_stream
            L.check(self._lib.rf_t5_encode(self._h, L.ptr(ids), B, S, L.ptr(bias), L.ptr(out), s), "rf_t5_encode")
        return out

    def clip_encode(self, input_ids: torch.Tensor, eos_token_id: int = 2,
                    return_hidden: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """ids [B, S<=77] -> pooler_output [B, d] (hidden state at the EOS position), optionally
        last_hidden_state.  eos_token_id == 2 is the stock CLIP-L config, for which transformers
        pools at ids.argmax(-1); otherwise at the first occurrence of eos_token_id."""
        self._check_ids(input_ids, self.cfg["clip_vocab"], "clip_encode")
        ids = input_ids.to(self.device, torch.int32).contiguous()
        B, S = ids.shape
        if eos_token_id == 2:
            pos = ids.argmax(dim=-1).to(torch.int32)
        else:
            pos = (ids == eos_token_id).int().argmax(dim=-1).to(torch.int32)
        C = self.cfg["clip_d_model"]
        pooled = torch.empty(B, C, device=self.device, dtype=torch.bfloat16)
        hidden = torch.empty(B, S, C, device=self.device, dtype=torch.bfloat16) if return_hidden else None
        with torch.cuda.device(self.device):
            s = torch.cuda.current_stream().cuda_stream
            L.check(self._lib.rf_clip_encode(self._h, L.ptr(ids), L.ptr(pos), B, S, L.ptr(pooled),
                                             L.ptr(hidden) if hidden is not None else None, s), "rf_clip_encode")
        return pooled, hidden

    # ---- pipeline hook ---------------------------------------------------------------------------
    def as_hook(self, tokenizer: Callable, tokenizer_2: Callable) -> Callable:
        """text_encoder_hook for B200FluxPipeline: (prompt, prompt_2, max_len) -> (prompt_embeds,
        pooled).  tokenizer(prompts, max_len) -> LongTensor ids [B, 77] (CLIP BPE, padded);
        tokenizer_2(prompts, max_len) -> ids [B, max_len] (T5 sentencepiece, padded).  Mirrors
        FluxPipeline._get_clip_prompt_embeds / _get_t5_prompt_embeds; CLIP pools by clip_eos_token_id."""

        def hook(prompt, prompt_2, max_len):
            prompt = [prompt] if isinstance(prompt, str) else list(prompt)
            prompt_2 = prompt if prompt_2 is None else ([prompt_2] if isinstance(prompt_2, str) else list(prompt_2))
            pooled, _ = self.clip_encode(tokenizer(prompt, 77), self.clip_eos_token_id)
            embeds = self.t5_encode(tokenizer_2(prompt_2, max_len))
            return embeds, pooled

        return hook
