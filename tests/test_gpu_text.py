"""T5 encoder / CLIP text model on the device vs transformers' own T5EncoderModel / CLIPTextModel.

The reference gets its text embeddings from diffusers FluxPipeline.encode_prompt, i.e. from the
transformers classes (train_flux/flux/generate.py:148-161) — transformers is installed in this image,
so it is imported directly as the oracle (CPU, eager attention, bf16 like the reference loads it, and
fp32 as the "true value"; the bf16 model also runs on the device, where the reference runs it, and
the distance to it is printed).  Floating-point bar, as for the DiT (DESIGN.md §5): our error against the
fp32 model may not exceed 1.25x the error of the reference's own bf16 arithmetic against it, and the
two bf16 results agree to a few 1e-3 of the mean magnitude."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().mean() / b.abs().mean()).item()


def _vs_cuda_bf16(m16, ids, ours, pick):
    """the bf16 transformers model run on the device, where the reference runs it: (mean error of ours against it
    relative to its mean magnitude, fraction of bit-identical elements)"""
    import copy
    mc = copy.deepcopy(m16).to("cuda")
    with torch.no_grad():
        ref = pick(mc(input_ids=ids.to("cuda"))).reshape(ours.shape)
    same = (ours.view(torch.int16) == ref.view(torch.int16)).float().mean().item()
    del mc
    return _rel(ours, ref), same


def _t5_models(layers, d_model, d_ff, heads, vocab, seed):
    from transformers import T5Config, T5EncoderModel
    cfg = T5Config(vocab_size=vocab, d_model=d_model, d_kv=64, d_ff=d_ff, num_layers=layers, num_heads=heads,
                   feed_forward_proj="gated-gelu", layer_norm_epsilon=1e-6, relative_attention_num_buckets=32,
                   relative_attention_max_distance=128, dropout_rate=0.0)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m32 = T5EncoderModel(cfg).eval()
    with torch.no_grad():
        for n, p in m32.named_parameters():  # HF init is tiny for a random model; use unit-variance activations
            if n.endswith("layer_norm.weight"):
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif "relative_attention_bias" in n or "shared" in n:
                p.copy_(torch.randn_like(p))
            elif n.endswith(".q.weight") or n.endswith(".k.weight"):
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5 * 0.6)
            else:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
            p.copy_(p.to(torch.bfloat16).float())  # both models hold the same bf16-representable weights
    import copy
    m16 = copy.deepcopy(m32).to(torch.bfloat16)
    return cfg, m32, m16


@pytest.mark.parametrize("layers,d_model,d_ff,heads,B,S", [
    (3, 1024, 2560, 16, 2, 128),
    (2, 512, 1024, 8, 1, 512),     # the FLUX sequence length
    (1, 4096, 10240, 64, 1, 64),   # one block at T5-v1.1-XXL width
    (2, 256, 512, 4, 3, 77),       # ragged: S not a multiple of 32
])
def test_t5_encoder_matches_transformers(layers, d_model, d_ff, heads, B, S):
    from reflectionflow_b200.text import B200TextEncoders
    vocab = 1024
    cfg, m32, m16 = _t5_models(layers, d_model, d_ff, heads, vocab, seed=layers * 7 + S)
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    with torch.no_grad():
        ref32 = m32(input_ids=ids)[0]
        ref16 = m16(input_ids=ids)[0]
    enc = B200TextEncoders(t5_layers=layers, t5_d_model=d_model, t5_d_ff=d_ff, t5_heads=heads, t5_vocab=vocab,
                           clip_layers=1, clip_d_model=256, clip_heads=4, clip_vocab=64, clip_max_pos=77)
    enc.load_t5_state_dict(m16.state_dict())
    out = enc.t5_encode(ids)
    torch.cuda.synchronize()
    assert out.shape == ref16.shape and out.dtype == torch.bfloat16
    e_ref, e_ours, e_pair = _rel(ref16, ref32), _rel(out, ref32), _rel(out, ref16)
    e_cuda, same = _vs_cuda_bf16(m16, ids, out, lambda r: r[0])
    print(f"t5 L{layers} d{d_model} S{S}: ref-bf16 vs fp32 {e_ref:.3e}, ours vs fp32 {e_ours:.3e}, ours vs ref-bf16 {e_pair:.3e}, "
          f"ours vs CUDA bf16 {e_cuda:.3e} (bit-identical {same:.4f})")
    assert e_ours <= 1.25 * e_ref + 1e-4
    assert e_pair <= 2.0 * e_ref + 1e-4      # two independent bf16 roundings of the same fp32 function


def test_t5_missing_weights_fail_loudly():
    from reflectionflow_b200 import _lib as L
    from reflectionflow_b200.text import B200TextEncoders
    enc = B200TextEncoders(t5_layers=1, t5_d_model=256, t5_d_ff=512, t5_heads=4, t5_vocab=64,
                           clip_layers=1, clip_d_model=256, clip_heads=4, clip_vocab=64, clip_max_pos=77)
    enc._rel_bias = torch.zeros(32, 4, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(L.RFError, match="missing text-encoder weights"):
        enc.t5_encode(torch.zeros(1, 32, dtype=torch.long))


def _clip_models(layers, seed):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=layers,
                         num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu",
                         eos_token_id=2, bos_token_id=0, pad_token_id=1)
    cfg._attn_implementation = "eager"
    torch.manual_seed(seed)
    m32 = CLIPTextModel(cfg).eval()
    with torch.no_grad():
        for n, p in m32.named_parameters():
            if "layer_norm" in n and n.endswith("weight"):
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif n.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
            elif "embedding" in n:
                p.copy_(torch.randn_like(p) * 0.5)
            else:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
            p.copy_(p.to(torch.bfloat16).float())
    import copy
    m16 = copy.deepcopy(m32).to(torch.bfloat16)
    return cfg, m32, m16


@pytest.mark.parametrize("layers,B,S", [(12, 3, 77), (2, 1, 77), (3, 2, 20)])
def test_clip_text_model_matches_transformers(layers, B, S):
    from reflectionflow_b200.text import B200TextEncoders
    cfg, m32, m16 = _clip_models(layers, seed=layers + S)
    g = torch.Generator().manual_seed(B * 100 + S)
    ids = torch.randint(3, 49000, (B, S), generator=g)
    ids[:, 0] = 49406
    for b in range(B):  # EOS (the largest id) somewhere in the row, padding after it
        e = int(torch.randint(1, S, (1,), generator=g))
        ids[b, e] = 49407
        ids[b, e + 1:] = 1
    with torch.no_grad():
        r32 = m32(input_ids=ids)
        r16 = m16(input_ids=ids)
    enc = B200TextEncoders(t5_layers=1, t5_d_model=256, t5_d_ff=512, t5_heads=4, t5_vocab=64, clip_layers=layers)
    enc.load_clip_state_dict(m16.state_dict())
    pooled, hidden = enc.clip_encode(ids, return_hidden=True)
    torch.cuda.synchronize()
    e_ref, e_ours = _rel(r16.last_hidden_state, r32.last_hidden_state), _rel(hidden, r32.last_hidden_state)
    p_ref, p_ours = _rel(r16.pooler_output, r32.pooler_output), _rel(pooled, r32.pooler_output)
    e_cuda, same = _vs_cuda_bf16(m16, ids, hidden, lambda r: r.last_hidden_state)
    print(f"clip L{layers} S{S}: hidden ref {e_ref:.3e} ours {e_ours:.3e}; pooled ref {p_ref:.3e} ours {p_ours:.3e}; "
          f"hidden ours vs CUDA bf16 {e_cuda:.3e} (bit-identical {same:.4f})")
    assert e_ours <= 1.25 * e_ref + 1e-4
    assert p_ours <= 1.5 * p_ref + 1e-4       # B x 768 values only: noisier statistic
    # pooled is the hidden state at the EOS position, bit for bit
    pos = ids.argmax(-1)
    assert torch.equal(pooled.cpu(), hidden.cpu()[torch.arange(B), pos])


def test_pipeline_text_hook_end_to_end():
    """ids -> (T5, CLIP) -> DiT denoise -> latents through B200FluxPipeline's encode_prompt hook"""
    from reflectionflow_b200.pipeline import B200FluxPipeline
    from reflectionflow_b200.config import FluxDiTConfig
    from reflectionflow_b200.text import B200TextEncoders
    cfg = FluxDiTConfig(num_layers=1, num_single_layers=1)
    pipe = B200FluxPipeline.from_synthetic(cfg, seed=0)
    enc = B200TextEncoders(t5_layers=1, t5_vocab=512, clip_layers=1).init_synthetic_weights(seed=1)

    def tok(vocab, eos):
        def f(prompts, max_len):
            out = torch.ones(len(prompts), max_len, dtype=torch.long)
            for i, p in enumerate(prompts):
                b = [3 + (ord(c) % (vocab - 4)) for c in p][: max_len - 1]
                out[i, : len(b)] = torch.tensor(b)
                out[i, len(b)] = eos
            return out
        return f

    pipe.text_encoder_hook = enc.as_hook(tok(49408, 49407), tok(512, 1))
    lat = pipe(prompt="a red cube on a blue sphere", height=256, width=256, num_inference_steps=2,
               guidance_scale=3.5, max_sequence_length=128, output_type="latent",
               generator=torch.Generator("cpu").manual_seed(0)).images
    lat2 = pipe(prompt="a red cube on a blue sphere", height=256, width=256, num_inference_steps=2,
                guidance_scale=3.5, max_sequence_length=128, output_type="latent",
                generator=torch.Generator("cpu").manual_seed(0)).images
    assert torch.isfinite(lat.float()).all() and torch.equal(lat, lat2)
