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
import math
from contextlib import contextmanager
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


MAX_LORA_RANK = 128


def _lora_pairs(lora: Dict[str, Any], max_rank: int) -> Dict[str, Any]:
    """{module_path: (A [r, in], B [out, r])} from either that mapping or a peft / diffusers LoRA state dict with
    keys `[transformer.]<module>.lora_A.weight` / `.lora_B.weight`; refuses factors that are not [r, in] / [out, r]
    and ranks above `max_rank`."""
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
    for mod, (A, B) in pairs.items():
        if A.ndim != 2 or B.ndim != 2 or B.shape[1] != A.shape[0]:
            raise ValueError(f"LoRA factors of {mod}: A {tuple(A.shape)} / B {tuple(B.shape)} "
                             "are not [r, in] / [out, r]")
        if A.shape[0] > max_rank:
            raise ValueError(f"LoRA rank {A.shape[0]} of {mod} exceeds the model's lora_rank {max_rank}: "
                             f"create the model with lora_rank >= {A.shape[0]} (at most {MAX_LORA_RANK})")
    return pairs


class B200FluxTransformer2DModel:
    """Owns one rf_dit handle (weights resident in HBM, packed for the kernels)."""

    def __init__(self, config=None, lora_rank: int = 0, device="cuda:0"):
        if not 0 <= int(lora_rank) <= MAX_LORA_RANK:
            raise ValueError(f"lora_rank must be 0..{MAX_LORA_RANK}, got {lora_rank}")
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
        self.has_lora = False  # an adapter is loaded: the call-level LoRA scale has something to act on
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

    @classmethod
    def from_pretrained(cls, transformer_dir: str, lora_rank: int = 0, device="cuda:0"):
        """A diffusers `transformer/` directory: FluxDiTConfig from its config.json (values the kernels do not
        implement are refused before the handle is created), weights streamed from its safetensors."""
        import os
        from . import checkpoint as ck
        cfg = ck.dit_config(ck.read_json(os.path.join(transformer_dir, "config.json")))
        stream = ck.SafetensorsStream(transformer_dir, ck.dit_key)
        return cls(cfg, lora_rank=lora_rank, device=device).load_state_dict(stream)

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
        keys `[transformer.]<module>.lora_A.weight` / `.lora_B.weight`.  scaling = alpha / r per module, r
        taken from that module's factors (alpha None: scaling 1; train_flux/config.yaml:50-51 r = alpha = 32).
        Ranks up to the model's lora_rank (<= 128)."""
        if self.lora_rank <= 0:
            raise L.RFError("model was created with lora_rank=0")
        if mode is not None:
            if mode not in ("exact", "merged"):
                raise ValueError("lora mode must be 'exact' or 'merged'")
            self.lora_mode = mode
        pairs = _lora_pairs(lora, self.lora_rank)
        self._geom_key = None  # adapters changed: rf_dit_prepare must re-run (merged copies, graph)
        with torch.cuda.device(self.device):
            for mod, (A, B) in pairs.items():
                r = A.shape[0]
                scale = 1.0 if alpha is None else float(alpha) / r
                a, b = _bf16c(A, self.device), _bf16c(B, self.device)
                L.check(self._lib.rf_dit_set_lora(self._h, mod.encode(), L.ptr(a), L.ptr(b), r,
                                                  int(A.shape[1]), int(B.shape[0]),
                                                  ctypes.c_float(scale)), f"rf_dit_set_lora({mod})")
                self.has_lora = True
            torch.cuda.synchronize(self.device)
        return self

    def unload_lora(self):
        """Unset every LoRA target (diffusers' unload_lora_weights): the model computes without an adapter until
        load_lora is called again.  load_lora itself only adds or replaces targets, so switching from an adapter
        on more modules to one on fewer goes through here."""
        L.check(self._lib.rf_dit_clear_lora(self._h), "rf_dit_clear_lora")
        self._geom_key = None  # the LoRA workspace, merged copies and captured step follow the new adapter set
        self.has_lora = False
        return self

    def set_lora_scale(self, scale: float):
        """diffusers' LoRA strength (joint_attention_kwargs["scale"]): multiplies every adapter's alpha / r from
        the next call on, until set again (1 = as loaded).  A captured denoise step built for another scale is
        re-captured, merged weights are re-merged."""
        L.check(self._lib.rf_dit_set_lora_scale(self._h, ctypes.c_double(float(scale))), "rf_dit_set_lora_scale")

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
                condition_scale: float = 1.0, image_guidance_scale: float = 1.0,
                uncond_condition_latents=None, step_hook=None) -> torch.Tensor:
        """Whole denoise loop on the device (rf_dit_denoise): one CUDA graph per step, replayed.

        `image_guidance_scale` s != 1: image classifier-free guidance over the condition stream (generate.py:250-272,
        rf_dit_denoise_image_guidance).  Every step adds a forward with the condition latents U_i of
        `uncond_condition_latents` [B, n_steps, n_cond, 64] and guidance 1, and steps on u + s * (c - u).  Without
        them U_i = condition_latents for every step.  s == 1 is the plain loop and ignores them.

        `step_hook(i, latents, prompt_embeds)` runs the loop step by step (rf_dit_denoise_begin / _step): see
        `run_steps`.  Without a hook the loop is one rf_dit_denoise call."""
        B = latents.shape[0]
        ts = timesteps_bf16.detach().to("cpu", torch.bfloat16).contiguous().view(torch.int16)
        sg = sigmas_f32.detach().to("cpu", torch.float32).contiguous()
        n = ts.numel()
        assert sg.numel() == n + 1
        guided = image_guidance_scale != 1.0
        if guided:
            if not math.isfinite(image_guidance_scale):
                raise ValueError(f"image_guidance_scale must be finite, got {image_guidance_scale}")
            if condition_latents is None or condition_ids is None:
                raise ValueError("image_guidance_scale != 1 guides over the condition stream: it needs a condition")
            if not self.cfg.guidance_embeds:
                raise ValueError("image_guidance_scale != 1 runs its uncond branch at guidance 1, which needs a model "
                                 "with guidance_embeds=True")
            shape = (B, condition_ids.shape[-2], self.cfg.in_channels)
            if tuple(condition_latents.shape) != shape:
                raise ValueError(f"condition_latents has shape {tuple(condition_latents.shape)}, image guidance "
                                 f"needs {shape} (batch, condition tokens, channels)")
            if uncond_condition_latents is None:
                uncond_condition_latents = condition_latents[:, None].expand(B, n, *shape[1:])
            if tuple(uncond_condition_latents.shape) != (B, n) + shape[1:]:
                raise ValueError(f"uncond_condition_latents has shape {tuple(uncond_condition_latents.shape)}, "
                                 f"expected {(B, n) + shape[1:]} (batch, steps, condition tokens, channels)")
        self.prepare(B, txt_ids, img_ids, condition_ids, model_config, condition_scale)
        dev = self.device
        lat = _bf16c(latents, dev).clone()
        txt = _bf16c(prompt_embeds, dev)
        pool = _bf16c(pooled, dev)
        cond = _bf16c(condition_latents, dev) if condition_latents is not None else None
        if step_hook is not None:
            unc = _bf16c(uncond_condition_latents, dev) if guided else None
            return self._denoise_steps(lat, txt, pool, ts, sg, guidance_scale, cond, image_guidance_scale if guided
                                       else 1.0, unc, step_hook)
        with torch.cuda.device(dev):
            if guided:
                unc = _bf16c(uncond_condition_latents, dev)
                L.check(self._lib.rf_dit_denoise_image_guidance(
                    self._h, L.ptr(lat), L.ptr(txt), L.ptr(pool), ctypes.c_void_p(ts.data_ptr()),
                    ctypes.c_void_p(sg.data_ptr()), n, ctypes.c_float(guidance_scale), L.ptr(cond), L.ptr(unc),
                    ctypes.c_float(image_guidance_scale), L.cur_stream()), "rf_dit_denoise_image_guidance")
            else:
                L.check(self._lib.rf_dit_denoise(self._h, L.ptr(lat), L.ptr(txt), L.ptr(pool),
                                                 ctypes.c_void_p(ts.data_ptr()),
                                                 ctypes.c_void_p(sg.data_ptr()), n,
                                                 ctypes.c_float(guidance_scale), L.ptr(cond),
                                                 L.cur_stream()), "rf_dit_denoise")
            torch.cuda.current_stream().synchronize()  # ts/sg host buffers must outlive the copies
        return lat

    def _denoise_steps(self, lat, txt, pool, ts, sg, guidance_scale, cond, image_guidance_scale, unc, step_hook):
        """The loop of `denoise` with a step hook: one session, then one rf_dit_denoise_step per executed step."""
        n = ts.numel()
        with torch.cuda.device(self.device):
            L.check(self._lib.rf_dit_denoise_begin(
                self._h, L.ptr(pool), ctypes.c_void_p(ts.data_ptr()), ctypes.c_void_p(sg.data_ptr()), n,
                ctypes.c_float(guidance_scale), L.ptr(cond), ctypes.c_float(image_guidance_scale), L.cur_stream()),
                "rf_dit_denoise_begin")
            torch.cuda.current_stream().synchronize()  # ts/sg host buffers must outlive the copies

            def step(i, lat, txt):
                u_i = None if unc is None else unc[:, i].contiguous()
                L.check(self._lib.rf_dit_denoise_step(self._h, i, L.ptr(lat), L.ptr(txt), L.ptr(u_i),
                                                      L.cur_stream()), "rf_dit_denoise_step")
            return run_steps(n, step, step_hook, lat, txt)


def run_steps(n: int, step, step_hook, lat: torch.Tensor, txt: torch.Tensor) -> torch.Tensor:
    """The step-wise loop of `denoise` (generate.py:217-290).  For i < n: `step(i, lat, txt)` advances a new copy of
    the latents in place (a new tensor per step, as the reference's scheduler.step returns one: a callback may keep
    it), then `step_hook(i, lat, txt)` returns (latents, prompt_embeds, stop).  The returned tensors feed the next
    step, or are the result when `stop` is set or i is the last step, as the reference pops the callback's outputs
    before its interrupt check.  They must keep the shapes and be bf16, else ValueError."""
    for i in range(n):
        lat = lat.clone()
        step(i, lat, txt)
        new_lat, new_txt, stop = step_hook(i, lat, txt)
        # the next step reads these through raw pointers
        lat, txt = step_input(new_lat, lat, "latents"), step_input(new_txt, txt, "prompt_embeds")
        if stop:
            break
    return lat


def step_input(t, ref: torch.Tensor, name: str) -> torch.Tensor:
    """A tensor a step callback hands to the next denoise step, on `ref`'s device and contiguous.  Its shape and dtype
    must be `ref`'s: the step reads that many bf16 rows."""
    if not torch.is_tensor(t) or t.shape != ref.shape or t.dtype != torch.bfloat16:
        got = f"{tuple(t.shape)} {t.dtype}" if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"`{name}` returned by callback_on_step_end must be a bf16 tensor of shape "
                         f"{tuple(ref.shape)}, got {got}")
    return t.detach().to(ref.device).contiguous()


@contextmanager
def lora_scale(transformer, joint_attention_kwargs: Optional[Dict[str, Any]]):
    """joint_attention_kwargs["scale"] for one call: diffusers' scale_lora_layers before it, unscale after
    (train_flux/flux/transformer.py:73-81,248).  Without a scale (or with 1) the transformer is not touched.  A
    scale other than 1 needs a loaded adapter: without one it could have no effect, so it is refused."""
    s = 1.0 if joint_attention_kwargs is None else joint_attention_kwargs.get("scale", 1.0)
    if s is None or s == 1.0:
        yield
        return
    if not getattr(transformer, "has_lora", False):
        raise NotImplementedError("joint_attention_kwargs['scale'] != 1 scales a LoRA adapter, and none is loaded")
    transformer.set_lora_scale(float(s))
    try:
        yield
    finally:
        transformer.set_lora_scale(1.0)


def tranformer_forward(transformer: B200FluxTransformer2DModel, condition_latents, condition_ids,
                       condition_type_ids, model_config: Optional[Dict[str, Any]] = {}, c_t=0,
                       **params):
    """Entry B — same name (typo included), arguments and return convention as
    train_flux/flux/transformer.py:47-55,250-252."""
    if c_t != 0:
        raise NotImplementedError("c_t != 0 is never used by the reference's callers")
    if params.get("controlnet_block_samples") is not None or \
            params.get("controlnet_single_block_samples") is not None:
        raise NotImplementedError("controlnet residuals (transformer.py:26-27,182,226) are not on the tts path")
    cscale = float(getattr(transformer, "condition_scale", 1.0))
    with lora_scale(transformer, params.get("joint_attention_kwargs")):
        out = transformer._forward(params["hidden_states"], params.get("encoder_hidden_states"),
                                   params.get("pooled_projections"), params.get("timestep"),
                                   params.get("img_ids"), params.get("txt_ids"), params.get("guidance"),
                                   condition_latents, condition_ids, model_config or {}, cscale)
    if not params.get("return_dict", True):
        return (out,)
    return Transformer2DModelOutput(sample=out)
