"""not-gpu: the LoRA scale and rank surface that needs no device: the C ABI exports rf_dit_set_lora_scale and refuses
lora_rank > 128, the Python model refuses such ranks and adapters of a higher rank than it was built for, and
joint_attention_kwargs["scale"] is applied around one call and then restored."""
import ctypes

import pytest
import torch

from reflectionflow_b200 import _lib
from reflectionflow_b200 import pipeline as P
from reflectionflow_b200 import transformer as T


class _Cfg(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("a", "b", "c", "d", "e", "f", "g", "lora_rank")]


def test_set_lora_scale_is_exported():
    lib = _lib.load()
    assert hasattr(lib, "rf_dit_set_lora_scale")
    assert lib.rf_dit_set_lora_scale(None, ctypes.c_double(0.5)) != 0
    assert b"null handle" in lib.rf_last_error()


@pytest.mark.parametrize("rank", [-1, 129, 256])
def test_c_abi_refuses_lora_rank_above_128(rank):
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.rf_dit_create(ctypes.byref(_Cfg(1, 1, 2, 64, 128, 64, 1, rank)), ctypes.byref(h)) == -1
    assert b"lora_rank must be 0..128" in lib.rf_last_error()


@pytest.mark.parametrize("rank", [-1, 129])
def test_model_refuses_lora_rank_above_128(rank):
    with pytest.raises(ValueError, match="lora_rank must be 0..128"):
        T.B200FluxTransformer2DModel(lora_rank=rank)


def test_adapter_rank_above_the_model_rank_is_refused():
    pairs = {"x_embedder": (torch.zeros(96, 64), torch.zeros(256, 96))}
    assert T._lora_pairs(pairs, 128) == pairs
    with pytest.raises(ValueError, match="LoRA rank 96 of x_embedder exceeds the model's lora_rank 64"):
        T._lora_pairs(pairs, 64)
    sd = {"transformer.x_embedder.lora_A.weight": torch.zeros(128, 64),
          "transformer.x_embedder.lora_B.weight": torch.zeros(256, 128)}
    assert list(T._lora_pairs(sd, 128)) == ["x_embedder"]
    with pytest.raises(ValueError, match="exceeds the model's lora_rank 32"):
        T._lora_pairs(sd, 32)


class _Fake:
    """records the call scale seen by each forward / denoise"""
    condition_scale = 1.0
    has_lora = True

    def __init__(self):
        self.scale, self.seen = 1.0, []

    def set_lora_scale(self, s):
        self.scale = s

    def _forward(self, *a):
        self.seen.append(self.scale)
        if a[0] is None:
            raise RuntimeError("boom")
        return torch.zeros(1, 4, 64)


def _kw(scale, hidden=torch.zeros(1, 4, 64)):
    return dict(hidden_states=hidden, encoder_hidden_states=1, pooled_projections=2, timestep=3, img_ids=4,
                txt_ids=5, guidance=6, return_dict=False,
                joint_attention_kwargs=None if scale is None else {"scale": scale})


def test_tranformer_forward_applies_the_scale_for_one_call():
    f = _Fake()
    for s in (0.75, None, 1.0, 0.0, -0.5):
        T.tranformer_forward(f, None, None, None, {}, 0, **_kw(s))
        assert f.scale == 1.0
    assert f.seen == [0.75, 1.0, 1.0, 0.0, -0.5]
    with pytest.raises(RuntimeError):  # restored even when the call fails
        T.tranformer_forward(f, None, None, None, {}, 0, **_kw(0.5, hidden=None))
    assert f.seen[-1] == 0.5 and f.scale == 1.0


def test_scale_without_an_adapter_is_refused():
    f = _Fake()
    f.has_lora = False
    T.tranformer_forward(f, None, None, None, {}, 0, **_kw(1.0))
    with pytest.raises(NotImplementedError):
        T.tranformer_forward(f, None, None, None, {}, 0, **_kw(0.5))
    assert f.seen == [1.0]


def test_load_lora_weights_reads_a_save_lora_directory(tmp_path):
    from safetensors.torch import save_file
    sd = {"transformer.x_embedder.lora_A.weight": torch.ones(4, 64),
          "transformer.x_embedder.lora_B.weight": torch.ones(256, 4)}
    save_file(sd, str(tmp_path / "pytorch_lora_weights.safetensors"))
    got = []

    class _T:
        def load_lora(self, lora, alpha):
            got.append((lora, alpha))

    pipe = P.B200FluxPipeline.__new__(P.B200FluxPipeline)
    pipe.transformer = _T()
    for path in (str(tmp_path), tmp_path, str(tmp_path / "pytorch_lora_weights.safetensors")):
        pipe.load_lora_weights(path, alpha=8)
    for lora, alpha in got:
        assert alpha == 8 and sorted(lora) == sorted(sd)
        assert all(torch.equal(lora[k], sd[k]) for k in sd)
