"""GPU parity of the text / vision conditioning front-end (SURVEY.md section 8(f) row 1) against the fp32 CPU oracle
(oracle/ladi_oracle/clip.py, itself pinned against transformers' CLIP classes and the reference's encode_text_word_embedding).
Tolerances (relative L2, engine bf16 vs oracle fp32): kernels with exact semantics (gather, im2col, token assembly) are compared
bit-exactly against the same bf16 arithmetic in torch; attention <= 1e-2; whole towers <= 2e-2.
"""
import pytest
import torch

from kernel_check import rel_l2
from model_pairs import text_pair

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,heads,hd,nq,causal", [(2, 16, 80, 257, False), (3, 16, 64, 77, True), (1, 2, 8, 5, True), (2, 3, 128, 130, False),
                                                  (1, 1, 40, 1, False), (2, 4, 64, 300, True)])
def test_attention_small(cuda, B, heads, hd, nq, causal):
    from ladi_vton_b200 import ops
    g = torch.Generator().manual_seed(nq * 7 + hd)
    C = heads * hd
    qkv = torch.randn((B, nq, 3 * C), generator=g).to(cuda, torch.bfloat16)  # strided q/k/v views of one fused projection
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    out = ops.attention_small(q, k, v, heads, hd ** -0.5, causal=causal)
    sp = lambda t: t.float().cpu().view(B, nq, heads, hd).transpose(1, 2)
    ref = torch.nn.functional.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=causal).transpose(1, 2).reshape(B, nq, C)
    err = rel_l2(out, ref)
    assert err < 1e-2, err


def test_attention_small_errors(cuda):
    from ladi_vton_b200 import ops
    x = torch.zeros((1, 4, 36), device=cuda, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.attention_small(x, x, x, 3, 1.0)  # head_dim 12
    q = torch.zeros((1, 4, 64), device=cuda, dtype=torch.bfloat16)
    k = torch.zeros((1, 6, 64), device=cuda, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="nq == nkv"):
        ops.attention_small(q, k, k, 1, 1.0, causal=True)


def test_embed_patchify_assemble_exact(cuda):
    from ladi_vton_b200 import ops
    g = torch.Generator().manual_seed(3)
    V, C, T, B, R = 50, 64, 7, 3, 4
    tok = torch.randn((V, C), generator=g).to(cuda, torch.bfloat16)
    pos = torch.randn((T, C), generator=g).to(cuda, torch.bfloat16)
    we = torch.randn((R, C), generator=g).to(cuda, torch.bfloat16)
    src = torch.randint(0, V, (B * T,), generator=g).to(torch.int32)
    src[2], src[9], src[10] = -1, -3, -4
    out = ops.clip_embed(src.to(cuda), tok, we, pos, T)
    rows = torch.stack([tok[s] if s >= 0 else we[-s - 1] for s in src.tolist()]).float()
    ref = (rows + pos.float().repeat(B, 1)).to(torch.bfloat16)
    assert torch.equal(out, ref)
    px = torch.randn((2, 3, 28, 42), generator=g).to(cuda)
    cols = ops.patchify(px, 14, 640)
    ref = torch.nn.functional.unfold(px, kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588).to(torch.bfloat16)
    assert torch.equal(cols[:, :588], ref) and float(cols[:, 588:].abs().max()) == 0.0
    patch = torch.randn((2 * 6, C), generator=g).to(cuda, torch.bfloat16)
    cls = torch.randn((C,), generator=g).to(cuda, torch.bfloat16)
    pos = torch.randn((7, C), generator=g).to(cuda, torch.bfloat16)
    x = ops.vit_assemble(patch, cls, pos, 2)
    ref = (torch.cat([cls.float().expand(2, 1, C), patch.float().view(2, 6, C)], dim=1) + pos.float()[None]).to(torch.bfloat16)
    assert torch.equal(x, ref)


def _ids(B, T, vocab, g, dollars=()):
    ids = torch.randint(1, min(vocab, 250), (B, T), generator=g)
    ids[:, 0] = vocab - 2
    for b in range(B):
        ids[b, 10 + 3 * b:] = vocab - 1  # EOT = highest id, then padding with EOT (SD-2 tokenizer pads with the EOT id... argmax = first)
    for b, f, n in dollars:
        ids[b, f:f + n] = 259
    return ids


@pytest.mark.parametrize("full", [False, True])
def test_encode_text_word_embedding(cuda, full):
    """src/utils/encode_text_word_embedding.py: '$' substitution (rows 0 and 2 carry pseudo-words, row 1 none), causal text tower."""
    from ladi_vton_b200 import encode_text_word_embedding
    from ladi_oracle.clip import encode_text_word_embedding as oracle_fn
    cfg = {} if full else dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=3, num_attention_heads=2)
    eng, o = text_pair(cuda, 77, **cfg)
    g = torch.Generator().manual_seed(11)
    nv = 16 if full else 4
    ids = _ids(3, 77, eng.config.vocab_size, g, dollars=[(0, 5, nv), (2, 8, nv)])
    we = torch.randn((3, nv, eng.config.hidden_size), generator=g)
    with torch.no_grad():
        ref = oracle_fn(o, ids.clone(), we.clone(), nv)
    out = encode_text_word_embedding(eng, ids.clone(), we.clone(), nv)
    assert out.last_hidden_state.shape == ref.last_hidden_state.shape
    e1, e2 = rel_l2(out.last_hidden_state, ref.last_hidden_state), rel_l2(out.pooler_output, ref.pooler_output)
    print("text tower rel-L2 last/pooled:", e1, e2)
    assert e1 < 2e-2 and e2 < 2e-2
    # plain call (the pipeline's text_encoder(ids)[0]) == encode without pseudo-words
    plain = eng(ids)[0]
    with torch.no_grad():
        ref_plain = o(ids).last_hidden_state
    assert rel_l2(plain, ref_plain) < 2e-2
    # the substitution must matter and must be confined to rows with '$' (row 1 unchanged)
    assert torch.equal(plain[1], out.last_hidden_state[1]) and not torch.equal(plain[0], out.last_hidden_state[0])


def test_text_encoder_errors(cuda):
    from ladi_vton_b200 import CLIPTextModel, encode_text_word_embedding
    eng, _ = text_pair(cuda, 5, vocab_size=1000, hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1)
    ids = torch.randint(1, 200, (2, 77))
    ids[0, 75] = 259
    with pytest.raises(IndexError):
        encode_text_word_embedding(eng, ids, torch.zeros((2, 4, 64)), 4)  # 4 pseudo-words do not fit after token 75
    with pytest.raises(ValueError):
        eng(torch.full((1, 77), 5000))
    with pytest.raises(RuntimeError):
        CLIPTextModel().to("cpu")


@pytest.mark.parametrize("full", [False, True])
def test_vision_tower(cuda, full):
    """src/inference.py:269-273: vision_encoder(pixel_values).last_hidden_state (ViT-H/14: [B, 257, 1280])."""
    from ladi_vton_b200 import CLIPVisionModelWithProjection, synthetic as S
    from ladi_oracle.clip import ClipVisionEncoder
    cfg = {} if full else dict(hidden_size=160, intermediate_size=320, num_hidden_layers=2, num_attention_heads=2, image_size=56)
    eng = CLIPVisionModelWithProjection(**cfg)
    c = eng.config
    sd = S.random_state_dict(eng.param_shapes(), 99)
    for k in sd:
        if "embedding" in k and "patch" not in k:
            sd[k] = torch.randn(sd[k].shape, generator=torch.Generator().manual_seed(len(k)))
    o = ClipVisionEncoder(dim=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers, mlp=c.intermediate_size,
                          image=c.image_size, patch=c.patch_size).eval()
    o.load_state_dict(sd)
    B = 1 if full else 2
    px = torch.randn((B, 3, c.image_size, c.image_size), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        ref = o(px)
    out = eng.load_state_dict(sd).to(cuda)(px)
    assert out.last_hidden_state.shape == ref.last_hidden_state.shape == (B, (c.image_size // 14) ** 2 + 1, c.hidden_size)
    e1, e2 = rel_l2(out.last_hidden_state, ref.last_hidden_state), rel_l2(out.pooler_output, ref.pooler_output)
    print("vision tower rel-L2 last/pooled:", e1, e2)
    assert e1 < 2e-2 and e2 < 2e-2


def test_pipeline_with_native_text_encoder(cuda):
    """tryon_pipe.py:284-301: with guidance and no negative_prompt_embeds the pipeline encodes the '' prompt itself through
    tokenizer + text_encoder; the engine text tower plugs into that slot."""
    from ladi_vton_b200 import synthetic as S
    pipe, _ = S.build_pipeline(cuda, S.SMALL_UNET, S.SMALL_VAE)
    eng, _ = text_pair(cuda, 8, vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2)

    class Tok:
        model_max_length = 77

        def __call__(self, texts, padding=None, max_length=77, truncation=True, return_tensors="pt"):
            ids = torch.full((len(texts), max_length), 999)
            ids[:, 0] = 998
            return type("Enc", (), {"input_ids": ids})()

    pipe.tokenizer, pipe.text_encoder = Tok(), eng
    inp = S.synthetic_inputs(2, 128, 64, ctx_dim=128)
    neg = eng(Tok()([""] * 2).input_ids)[0].float()
    kw = dict(image=inp["image"], mask_image=inp["mask_image"], pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"], height=128,
              width=64, num_inference_steps=3, guidance_scale=7.5, output_type="pt")
    a = pipe(prompt_embeds=inp["prompt_embeds"], generator=torch.Generator().manual_seed(1), **{k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}).images
    b = pipe(prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=neg, generator=torch.Generator().manual_seed(1),
             **{k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}).images
    assert torch.equal(a, b)
