"""B200FluxTransformer2DModel — the DiT behind the two call surfaces the reference uses:

  entry A  `pipe.transformer(hidden_states=..., timestep=..., guidance=..., pooled_projections=...,
            encoder_hidden_states=..., txt_ids=..., img_ids=..., joint_attention_kwargs=...,
            return_dict=False)[0]`   — stock diffusers FluxTransformer2DModel.forward, as called by
            FluxPipeline.__call__ (tts/tts_t2i_noise_scaling.py:60)
  entry B  `tranformer_forward(transformer, condition_latents, condition_ids, condition_type_ids,
            model_config, c_t, **params)`  — train_flux/flux/transformer.py:47-55

Both run the same C-ABI call (rf_dit_forward, include/rf_b200.h) on hand-written sm_90a
kernels.  There is no PyTorch fallback: without librf_b200.so or without a GPU this raises.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Any, Dict, Optional

import torch

from . import _lib as L
from .config import FluxDiTConfig


class _RfDitConfig(ctypes.Structure):
    _fields_ = [("num_layers", ctypes.c_int), ("num_single_layers", ctypes.c_int),
                ("num_heads", ctypes.c_int), ("in_channels", ctypes.c_int),
                ("joint_attention_dim", ctypes.c_int), ("pooled_projection_dim", ctypes.c_int),
                ("guidance_embeds", ctypes.c_int), ("lora_rank", ctypes.c_int)]


@dataclass
class Transformer2DModelOutput:
    sample: torch.Tensor


class _ConfigView(dict):
    __getattr__ = dict.__getitem__


def _bf16c(t: torch.Tensor, device) -> torch.Tensor:
    return t.detach().to(device=device, dtype=torch.bfloat16).contiguous()


class B200FluxTransformer2DModel:
    """Owns one rf_dit handle (weights resident in HBM, packed for the kernels)."""

    def __init__(self, config=None, lora_rank: int = 0, device="cuda:0"):
        if not torch.cuda.is_available():
            raise L.RFError("B200FluxTransformer2DModel needs a CUDA device; there is no CPU fallback")
        self.cfg = FluxDiTConfig.from_any(config or FluxDiTConfig())
        if self.cfg.attention_head_dim != 128:
            raise ValueError("attention_head_dim must be 128")
        self.device = torch.device(device)
        self.dtype = torch.bfloat16
        self.config = _ConfigView(**self.cfg.to_dict())
        self.lora_rank = int(lora_rank)
        self._lib = L.load()
        self._h = ctypes.c_void_p()
        self._geom_key = None
        self._geom_ids = None
        # "exact": y = Wx + b + B(A x) with peft's three bf16 roundings (bit-faithful to the reference);
        # "merged": condition tokens use W + BA (peft fuse_lora; the reference leaves that call
        # commented out at tts_reflectionflow.py:506) — no extra kernels, +11.5 GB of weights.
        self.lora_mode = "exact"
        with torch.cuda.device(self.device):
            c = _RfDitConfig(self.cfg.num_layers, self.cfg.num_single_layers,
                             self.cfg.num_attention_heads, self.cfg.in_channels,
                             self.cfg.joint_attention_dim, self.cfg.pooled_projection_dim,
                             int(self.cfg.guidance_embeds), self.lora_rank)
            L.check(self._lib.rf_dit_create(ctypes.byref(c), ctypes.byref(self._h)), "rf_dit_create")

    # ------------------------------------------------------------------ lifetime
    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.rf_dit_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def to(self, *a, **k):  # diffusers-style no-op: weights already live on the device
        return self

    def eval(self):
        return self

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """`sd` uses diffusers' FluxTransformer2DModel keys.  Tensors may live anywhere; each is
        staged to the device in bf16 and copied into the handle's packed storage."""
        self._geom_key = None
        with torch.cuda.device(self.device):
            for k, v in sd.items():
                if ".lora_" in k:
                    continue
                t = _bf16c(v, self.device)
                rc = self._lib.rf_dit_load_weight(self._h, k.encode(), L.ptr(t), t.numel())
                if rc != 0 and strict:
                    L.check(rc, f"rf_dit_load_weight({k})")
            torch.cuda.synchronize(self.device)
            if strict:
                n = self._lib.rf_dit_missing_weights(self._h)
                if n != 0:
                    L.check(-4, "load_state_dict (missing weights)")
        return self

    def init_synthetic_weights(self, seed: int = 0):
        """Random-init weights of the right architecture directly on the GPU (no checkpoint exists
        offline): N(0, 1/fan_in) matrices, small biases, RMSNorm scales near 1."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        d, c = self.cfg.inner_dim, self.cfg

        def lin(name, out, inp, wscale=1.0):
            w = torch.randn(out, inp, generator=g, device=self.device, dtype=torch.float32)
            w = (w * (wscale / inp ** 0.5)).to(torch.bfloat16)
            b = (0.05 * torch.randn(out, generator=g, device=self.device)).to(torch.bfloat16)
            for k, t in ((name + ".weight", w), (name + ".bias", b)):
                L.check(self._lib.rf_dit_load_weight(self._h, k.encode(), L.ptr(t), t.numel()), k)

        def rms(name):
            t = (1 + 0.1 * torch.randn(128, generator=g, device=self.device)).to(torch.bfloat16)
            L.check(self._lib.rf_dit_load_weight(self._h, name.encode(), L.ptr(t), 128), name)

        with torch.cuda.device(self.device):
            lin("x_embedder", d, c.in_channels)
            lin("context_embedder", d, c.joint_attention_dim)
            tte = "time_text_embed."
            lin(tte + "timestep_embedder.linear_1", d, 256)
            lin(tte + "timestep_embedder.linear_2", d, d)
            if c.guidance_embeds:
                lin(tte + "guidance_embedder.linear_1", d, 256)
                lin(tte + "guidance_embedder.linear_2", d, d)
            lin(tte + "text_embedder.linear_1", d, c.pooled_projection_dim)
            lin(tte + "text_embedder.linear_2", d, d)
            for i in range(c.num_layers):
                p = f"transformer_blocks.{i}."
                lin(p + "norm1.linear", 6 * d, d, 0.5)
                lin(p + "norm1_context.linear", 6 * d, d, 0.5)
                for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj",
                          "to_out.0", "to_add_out"):
                    lin(p + "attn." + n, d, d)
                for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
                    rms(p + "attn." + n + ".weight")
                lin(p + "ff.net.0.proj", 4 * d, d)
                lin(p + "ff.net.2", d, 4 * d)
                lin(p + "ff_context.net.0.proj", 4 * d, d)
                lin(p + "ff_context.net.2", d, 4 * d)
            for i in range(c.num_single_layers):
                p = f"single_transformer_blocks.{i}."
                lin(p + "norm.linear", 3 * d, d, 0.5)
                for n in ("to_q", "to_k", "to_v"):
                    lin(p + "attn." + n, d, d)
                rms(p + "attn.norm_q.weight")
                rms(p + "attn.norm_k.weight")
                lin(p + "proj_mlp", 4 * d, d)
                lin(p + "proj_out", d, 5 * d)
            lin("norm_out.linear", 2 * d, d, 0.5)
            lin("proj_out", c.in_channels, d)
            torch.cuda.synchronize(self.device)
            if self._lib.rf_dit_missing_weights(self._h) != 0:
                L.check(-4, "init_synthetic_weights")
        return self

    def load_lora(self, lora: Dict[str, Any], alpha: Optional[float] = None, mode: Optional[str] = None):
        """`lora`: {module_path: (A [r,in], B [out,r])}  or a peft/diffusers LoRA state dict with
        keys `[transformer.]<module>.lora_A.weight` / `.lora_B.weight`.  scaling = alpha / r
        (train_flux/config.yaml:50-51: r = alpha = 32 -> 1)."""
        if self.lora_rank <= 0:
            raise L.RFError("model was created with lora_rank=0")
        if mode is not None:
            if mode not in ("exact", "merged"):
                raise ValueError("lora mode must be 'exact' or 'merged'")
            self.lora_mode = mode
        self._geom_key = None  # adapters changed: rf_dit_prepare must re-run (merged copies, graph)
        pairs = {}
        if lora and all(isinstance(v, (tuple, list)) for v in lora.values()):
            pairs = dict(lora)
        else:
            tmp: Dict[str, Dict[str, torch.Tensor]] = {}
            for k, v in lora.items():
                k = k[len("transformer."):] if k.startswith("transformer.") else k
                for tag in (".lora_A", ".lora_B"):
                    if tag in k:
                        mod = k.split(tag)[0]
                        tmp.setdefault(mod, {})[tag] = v
            pairs = {m: (d[".lora_A"], d[".lora_B"]) for m, d in tmp.items()}
        with torch.cuda.device(self.device):
            for mod, (A, B) in pairs.items():
                r = A.shape[0]
                if A.ndim != 2 or B.ndim != 2 or B.shape[1] != r:
                    raise ValueError(f"LoRA factors of {mod}: A {tuple(A.shape)} / B {tuple(B.shape)} "
                                     "are not [r, in] / [out, r]")
                scale = 1.0 if alpha is None else float(alpha) / r
                a, b = _bf16c(A, self.device), _bf16c(B, self.device)
                L.check(self._lib.rf_dit_set_lora(self._h, mod.encode(), L.ptr(a), L.ptr(b), r,
                                                  int(A.shape[1]), int(B.shape[0]),
                                                  ctypes.c_float(scale)), f"rf_dit_set_lora({mod})")
            torch.cuda.synchronize(self.device)
        return self

    # ------------------------------------------------------------------ geometry
    def _flags(self, model_config: Optional[Dict[str, Any]]) -> int:
        mc = model_config or {}
        f = 8 if self.lora_mode == "merged" else 0
        if mc.get("latent_lora", False):
            f |= 1
        if mc.get("add_cond_attn", False):
            f |= 2
        if not mc.get("union_cond_attn", True):
            f |= 4
        return f

    def prepare(self, batch: int, txt_ids: torch.Tensor, img_ids: torch.Tensor,
                cond_ids: Optional[torch.Tensor] = None, model_config=None,
                condition_scale: float = 1.0):
        if txt_ids.ndim == 3:  # deprecated 3-D ids (transformer.py:117-128)
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3:
            img_ids = img_ids[0]
        n_cond = 0 if cond_ids is None else cond_ids.shape[0]
        key = (batch, txt_ids.shape[0], img_ids.shape[0], n_cond, self._flags(model_config),
               float(condition_scale))
        t = _bf16c(txt_ids, self.device)
        i = _bf16c(img_ids, self.device)
        c = _bf16c(cond_ids, self.device) if cond_ids is not None else None
        if self._geom_key == key and self._geom_ids is not None:
            ot, oi, oc = self._geom_ids
            if torch.equal(ot, t) and torch.equal(oi, i) and (c is None or torch.equal(oc, c)):
                return
        with torch.cuda.device(self.device):
            L.check(self._lib.rf_dit_prepare(self._h, batch, t.shape[0], i.shape[0], n_cond, L.ptr(t),
                                             L.ptr(i), L.ptr(c), key[4],
                                             ctypes.c_float(condition_scale), L.cur_stream()),
                    "rf_dit_prepare")
        self._geom_key, self._geom_ids = key, (t, i, c)

    # ------------------------------------------------------------------ forward
    def _forward(self, hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids,
                 txt_ids, guidance, condition_latents=None, condition_ids=None, model_config=None,
                 condition_scale: float = 1.0) -> torch.Tensor:
        B = hidden_states.shape[0]
        self.prepare(B, txt_ids, img_ids, condition_ids, model_config, condition_scale)
        dev = self.device
        lat = _bf16c(hidden_states, dev)
        txt = _bf16c(encoder_hidden_states, dev)
        pool = _bf16c(pooled_projections, dev)
        ts = _bf16c(timestep.reshape(-1).expand(B) if timestep.numel() == 1 else timestep, dev)
        g = None
        if self.cfg.guidance_embeds:
            if guidance is None:
                raise ValueError("guidance is required when guidance_embeds=True")
            g = guidance.detach().to(device=dev, dtype=torch.float32).reshape(-1).expand(B).contiguous()
        cond = _bf16c(condition_latents, dev) if condition_latents is not None else None
        out = torch.empty_like(lat)
        with torch.cuda.device(dev):
            L.check(self._lib.rf_dit_forward(self._h, L.ptr(lat), L.ptr(txt), L.ptr(pool), L.ptr(ts),
                                             L.ptr(g), L.ptr(cond), L.ptr(out), L.cur_stream()),
                    "rf_dit_forward")
        return out

    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None,
                timestep=None, img_ids=None, txt_ids=None, guidance=None,
                joint_attention_kwargs=None, controlnet_block_samples=None,
                controlnet_single_block_samples=None, return_dict: bool = True, **_):
        """Entry A: diffusers FluxTransformer2DModel.forward keyword surface."""
        if controlnet_block_samples is not None or controlnet_single_block_samples is not None:
            raise NotImplementedError("ControlNet residuals are never fed on this path")
        out = self._forward(hidden_states, encoder_hidden_states, pooled_projections, timestep,
                            img_ids, txt_ids, guidance)
        return Transformer2DModelOutput(sample=out) if return_dict else (out,)

    __call__ = forward

    def denoise(self, latents, prompt_embeds, pooled, timesteps_bf16: torch.Tensor,
                sigmas_f32: torch.Tensor, guidance_scale: float, img_ids, txt_ids,
                condition_latents=None, condition_ids=None, model_config=None,
                condition_scale: float = 1.0) -> torch.Tensor:
        """Whole denoise loop on the device (rf_dit_denoise): one CUDA graph per step, replayed."""
        B = latents.shape[0]
        self.prepare(B, txt_ids, img_ids, condition_ids, model_config, condition_scale)
        dev = self.device
        lat = _bf16c(latents, dev).clone()
        txt = _bf16c(prompt_embeds, dev)
        pool = _bf16c(pooled, dev)
        cond = _bf16c(condition_latents, dev) if condition_latents is not None else None
        ts = timesteps_bf16.detach().to("cpu", torch.bfloat16).contiguous().view(torch.int16)
        sg = sigmas_f32.detach().to("cpu", torch.float32).contiguous()
        n = ts.numel()
        assert sg.numel() == n + 1
        with torch.cuda.device(dev):
            L.check(self._lib.rf_dit_denoise(self._h, L.ptr(lat), L.ptr(txt), L.ptr(pool),
                                             ctypes.c_void_p(ts.data_ptr()),
                                             ctypes.c_void_p(sg.data_ptr()), n,
                                             ctypes.c_float(guidance_scale), L.ptr(cond),
                                             L.cur_stream()), "rf_dit_denoise")
            torch.cuda.current_stream().synchronize()  # ts/sg host buffers must outlive the copies
        return lat


def tranformer_forward(transformer: B200FluxTransformer2DModel, condition_latents, condition_ids,
                       condition_type_ids, model_config: Optional[Dict[str, Any]] = {}, c_t=0,
                       **params):
    """Entry B — same name (typo included), arguments and return convention as
    train_flux/flux/transformer.py:47-55,250-252."""
    if c_t != 0:
        raise NotImplementedError("c_t != 0 is never used by the reference's callers")
    jak = params.get("joint_attention_kwargs")
    if jak is not None and jak.get("scale", 1.0) != 1.0:
        raise NotImplementedError("joint_attention_kwargs['scale'] != 1 is not supported")
    if params.get("controlnet_block_samples") is not None or \
            params.get("controlnet_single_block_samples") is not None:
        raise NotImplementedError("controlnet residuals (transformer.py:26-27,182,226) are not on the tts path")
    cscale = float(getattr(transformer, "condition_scale", 1.0))
    out = transformer._forward(params["hidden_states"], params.get("encoder_hidden_states"),
                               params.get("pooled_projections"), params.get("timestep"),
                               params.get("img_ids"), params.get("txt_ids"), params.get("guidance"),
                               condition_latents, condition_ids, model_config or {}, cscale)
    if not params.get("return_dict", True):
        return (out,)
    return Transformer2DModelOutput(sample=out)
