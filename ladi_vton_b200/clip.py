"""H100-native CLIP towers of the text/vision conditioning front-end (SURVEY.md section 8(f) row 1).

  * `CLIPTextModel` + `encode_text_word_embedding(text_encoder, input_ids, word_embeddings, num_vstar)`: drop-in for
    src/utils/encode_text_word_embedding.py:6-72 -- token embeddings with every prompt's first-'$' window replaced by
    its pseudo-word embeddings, the causal CLIP text transformer (SD-2 text encoder: 23 pre-LN layers, 1024 wide, 16 heads of 64,
    MLP 4096 GELU(erf)), final LayerNorm, pooled row at argmax(input_ids).  Also the `text_encoder(ids)[0]` call of the pipeline's
    own `_encode_prompt` (tryon_pipe.py:230-240, 284-301: the '' negative prompt of classifier-free guidance).
  * `CLIPVisionModelWithProjection`: `vision_encoder(pixel_values).last_hidden_state` of src/inference.py:269-273 (ViT-H/14: 32 layers,
    1280 wide, 16 heads of 80, MLP 5120; `last_hidden_state` is the encoder output BEFORE post_layernorm, 257 tokens).

State-dict keys are the transformers ones (`text_model.embeddings.token_embedding.weight`, `text_model.encoder.layers.N.self_attn.
{q,k,v,out}_proj.*`, `...layer_norm1/2.*`, `...mlp.fc1/fc2.*`, `text_model.final_layer_norm.*`; `vision_model.embeddings.{class_embedding,
patch_embedding.weight, position_embedding.weight}`, `vision_model.pre_layrnorm.*`, `vision_model.post_layernorm.*`).  All GEMMs run on
the wgmma kernel of the hot path (fused QKV, GELU / residual epilogues), LayerNorm on the hot-path kernel, attention on
`ladi_attention_small` (fp32 softmax; 80-wide heads do not fit the 64-wide tensor-core attention).  No CPU path.
"""
import torch

from . import ops
from .module import PackedModule, _Cfg
from .weights import f32, pack_linear

DOLLAR_ID = 259  # '$' (encode_text_word_embedding.py:13)


class CLIPOutput:
    """last_hidden_state / pooler_output with tuple-style indexing, like transformers' BaseModelOutputWithPooling."""

    def __init__(self, last_hidden_state, pooler_output, hidden_states=None, attentions=None):
        self.last_hidden_state, self.pooler_output = last_hidden_state, pooler_output
        self.hidden_states, self.attentions = hidden_states, attentions
        self.image_embeds = None

    def __getitem__(self, i):
        return (self.last_hidden_state, self.pooler_output)[i]


class _Tower(PackedModule):
    """Shared: layer packing, the pre-LN transformer stack."""
    prefix = ""

    def __init__(self, **config):
        self.config = _Cfg(config)
        self.dtype = torch.bfloat16

    def ignorable(self, key):  # transformers checkpoints also hold these; the path here never reads them
        return key.endswith("position_ids") or key.startswith(("visual_projection", "text_projection"))

    def _pack_layers(self, P):
        g = lambda k: self._sd[k].to(self.device, torch.float32)
        for i in range(self.config.num_hidden_layers):
            p = f"{self.prefix}.encoder.layers.{i}."
            pack_encoder_layer(P, p, g, p)

    def _stack(self, x, B, T, causal):
        """x [B*T, C] bf16 -> [B*T, C] bf16 through all encoder layers (transformers CLIPEncoderLayer: pre-LN, residual adds)."""
        cfg = self.config
        for i in range(cfg.num_hidden_layers):
            x = encoder_layer(self.P, f"{self.prefix}.encoder.layers.{i}.", x, B, T, cfg.num_attention_heads, cfg.intermediate_size,
                              cfg.layer_norm_eps, causal)
        return x


# ---- one CLIP encoder layer: shared by both towers and by the inversion adapter's full-sequence layers -----------------------------
def encoder_layer_shapes(S, p, d, mlp):
    """transformers CLIPEncoderLayer state-dict entries under prefix `p`."""
    for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
        S[p + f"self_attn.{n}.weight"], S[p + f"self_attn.{n}.bias"] = (d, d), (d,)
    for n in ("layer_norm1", "layer_norm2"):
        S[p + n + ".weight"], S[p + n + ".bias"] = (d,), (d,)
    S[p + "mlp.fc1.weight"], S[p + "mlp.fc1.bias"] = (mlp, d), (mlp,)
    S[p + "mlp.fc2.weight"], S[p + "mlp.fc2.bias"] = (d, mlp), (d,)


def pack_encoder_layer(P, dst, g, src):
    """State-dict entries under `src` (read through g(key) -> fp32 device tensor) -> packed entries P[dst + {ln1, ln2, qkv.*, o.*, fc1.*, fc2.*}]."""
    P[dst + "ln1"] = (f32(g(src + "layer_norm1.weight")), f32(g(src + "layer_norm1.bias")))
    P[dst + "ln2"] = (f32(g(src + "layer_norm2.weight")), f32(g(src + "layer_norm2.bias")))
    P[dst + "qkv.w"] = pack_linear(torch.cat([g(src + f"self_attn.{n}_proj.weight") for n in "qkv"]))
    P[dst + "qkv.b"] = f32(torch.cat([g(src + f"self_attn.{n}_proj.bias") for n in "qkv"]))
    for n, k in (("o", "self_attn.out_proj"), ("fc1", "mlp.fc1"), ("fc2", "mlp.fc2")):
        P[dst + n + ".w"], P[dst + n + ".b"] = pack_linear(g(src + k + ".weight")), f32(g(src + k + ".bias"))


def encoder_layer(P, p, x, B, T, heads, mlp, eps, causal=False):
    """x [B*T, C] bf16 -> [B*T, C] bf16 through the packed layer P[p + ...] (transformers CLIPEncoderLayer: pre-LN, residual adds)."""
    C = x.shape[1]
    qkv = ops.gemm(ops.layernorm(x, *P[p + "ln1"], eps=eps), P[p + "qkv.w"], 3 * C, bias=P[p + "qkv.b"]).view(B, T, 3 * C)
    a = ops.attention_small(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, (C // heads) ** -0.5, causal=causal)
    x = ops.gemm(a.view(B * T, C), P[p + "o.w"], C, bias=P[p + "o.b"], residual=x)
    h = ops.gemm(ops.layernorm(x, *P[p + "ln2"], eps=eps), P[p + "fc1.w"], mlp, bias=P[p + "fc1.b"], act=ops.ACT_GELU)
    return ops.gemm(h, P[p + "fc2.w"], C, bias=P[p + "fc2.b"], residual=x)


SD2_TEXT_ENCODER = dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
                        max_position_embeddings=77, layer_norm_eps=1e-5, hidden_act="gelu")
VIT_H_14 = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16, image_size=224, patch_size=14,
                num_channels=3, layer_norm_eps=1e-5, hidden_act="gelu")


class CLIPTextModel(_Tower):
    prefix = "text_model"

    def __init__(self, **config):
        cfg = dict(SD2_TEXT_ENCODER)
        cfg.update(config)
        if cfg["hidden_act"] != "gelu":
            raise NotImplementedError("only the GELU(erf) activation of the SD-2 text encoder is built")
        super().__init__(**cfg)

    def param_shapes(self):
        c, S = self.config, {}
        d = c.hidden_size
        S["text_model.embeddings.token_embedding.weight"] = (c.vocab_size, d)
        S["text_model.embeddings.position_embedding.weight"] = (c.max_position_embeddings, d)
        for i in range(c.num_hidden_layers):
            encoder_layer_shapes(S, f"text_model.encoder.layers.{i}.", d, c.intermediate_size)
        S["text_model.final_layer_norm.weight"], S["text_model.final_layer_norm.bias"] = (d,), (d,)
        return S

    def _pack_weights(self):
        g = lambda k: self._sd[k].to(self.device, torch.float32)
        P = {}
        P["tok"] = g("text_model.embeddings.token_embedding.weight").to(torch.bfloat16).contiguous()
        P["pos"] = g("text_model.embeddings.position_embedding.weight").to(torch.bfloat16).contiguous()
        P["lnf"] = (f32(g("text_model.final_layer_norm.weight")), f32(g("text_model.final_layer_norm.bias")))
        self._pack_layers(P)
        self.P = P

    def encode(self, input_ids, word_embeddings=None, num_vstar=1):
        """input_ids [B, T] int; word_embeddings [B, num_vstar, C] (or [B, C]) or None -> CLIPOutput (bf16 device tensors)."""
        if self.P is None:
            raise RuntimeError("CLIPTextModel: load_state_dict(...) and .to('cuda') first")
        cfg = self.config
        ids = input_ids.view(-1, input_ids.shape[-1])
        B, T = ids.shape
        if T > cfg.max_position_embeddings:
            raise ValueError(f"sequence length {T} exceeds max_position_embeddings {cfg.max_position_embeddings}")
        ids_h = ids.detach().cpu().to(torch.int64)
        if int(ids_h.min()) < 0 or int(ids_h.max()) >= cfg.vocab_size:
            raise ValueError("input_ids outside the vocabulary")
        src = ids_h.to(torch.int32).clone()
        we = None
        rows_with = (ids_h == DOLLAR_ID).any(dim=1)
        if word_embeddings is not None and bool(rows_with.any()):  # encode_text_word_embedding.py:13-38
            we = word_embeddings
            if we.dim() == 2:
                we = we.unsqueeze(1)
            if we.shape[0] != B:
                raise AssertionError("word_embeddings.shape[0] must equal the batch size")  # :32
            if we.shape[1] < num_vstar or we.shape[2] != cfg.hidden_size:
                raise ValueError(f"word_embeddings must be [B, >= num_vstar, {cfg.hidden_size}], got {tuple(we.shape)}")
            we = we[:, :num_vstar].to(self.device, torch.bfloat16).contiguous()
            for b in range(B):
                if bool(rows_with[b]):
                    f = int((ids_h[b] == DOLLAR_ID).nonzero()[0])
                    if f + num_vstar > T:
                        raise IndexError(f"prompt {b}: {num_vstar} pseudo-words starting at token {f} do not fit {T} tokens")
                    src[b, f:f + num_vstar] = -(b * num_vstar + torch.arange(num_vstar, dtype=torch.int32)) - 1
            we = we.view(B * num_vstar, cfg.hidden_size)
        x = ops.clip_embed(src.to(self.device).view(-1), self.P["tok"], we, self.P["pos"], T)
        x = self._stack(x, B, T, causal=True)
        last = ops.layernorm(x, *self.P["lnf"], eps=cfg.layer_norm_eps).view(B, T, cfg.hidden_size)
        eot = ids_h.to(torch.int).argmax(dim=-1).to(self.device)  # :60-63
        return CLIPOutput(last, last[torch.arange(B, device=self.device), eot])

    def __call__(self, input_ids, attention_mask=None, **kw):
        return self.encode(input_ids)


def encode_text_word_embedding(text_encoder, input_ids, word_embeddings, num_vstar=1):
    """Same arguments and return fields as the reference function (src/utils/encode_text_word_embedding.py:6-7)."""
    return text_encoder.encode(input_ids, word_embeddings, num_vstar)


class CLIPVisionModelWithProjection(_Tower):
    """Only the path the reference uses is built: `.last_hidden_state` (+ `pooler_output`); the visual projection is accepted in the
    state dict and ignored (`image_embeds` is never read on this path, src/inference.py:272-273)."""
    prefix = "vision_model"

    def __init__(self, **config):
        cfg = dict(VIT_H_14)
        cfg.update(config)
        if cfg["hidden_act"] != "gelu":
            raise NotImplementedError("only the GELU(erf) activation of CLIP ViT-H-14 (laion2B) is built")
        super().__init__(**cfg)

    def param_shapes(self):
        c, S = self.config, {}
        d, ps = c.hidden_size, c.patch_size
        S["vision_model.embeddings.class_embedding"] = (d,)
        S["vision_model.embeddings.patch_embedding.weight"] = (d, c.num_channels, ps, ps)
        S["vision_model.embeddings.position_embedding.weight"] = ((c.image_size // ps) ** 2 + 1, d)
        for n in ("pre_layrnorm", "post_layernorm"):
            S[f"vision_model.{n}.weight"], S[f"vision_model.{n}.bias"] = (d,), (d,)
        for i in range(c.num_hidden_layers):
            encoder_layer_shapes(S, f"vision_model.encoder.layers.{i}.", d, c.intermediate_size)
        return S

    def _pack_weights(self):
        g = lambda k: self._sd[k].to(self.device, torch.float32)
        P = {}
        P["cls"] = g("vision_model.embeddings.class_embedding").to(torch.bfloat16).contiguous()
        P["pos"] = g("vision_model.embeddings.position_embedding.weight").to(torch.bfloat16).contiguous()
        w = g("vision_model.embeddings.patch_embedding.weight")
        P["patch.w"] = pack_linear(w.reshape(w.shape[0], -1))  # [C, 3*14*14 = 588 -> 640]
        P["pre"] = (f32(g("vision_model.pre_layrnorm.weight")), f32(g("vision_model.pre_layrnorm.bias")))
        P["post"] = (f32(g("vision_model.post_layernorm.weight")), f32(g("vision_model.post_layernorm.bias")))
        self._pack_layers(P)
        self.P = P

    def __call__(self, pixel_values, **kw):
        if self.P is None:
            raise RuntimeError("CLIPVisionModelWithProjection: load_state_dict(...) and .to('cuda') first")
        cfg = self.config
        B, ch, H, W = pixel_values.shape
        if ch != cfg.num_channels or H != cfg.image_size or W != cfg.image_size:
            raise ValueError(f"pixel_values must be [B, {cfg.num_channels}, {cfg.image_size}, {cfg.image_size}], got {tuple(pixel_values.shape)}")
        px = pixel_values.to(self.device, torch.float32).contiguous()
        C = cfg.hidden_size
        cols = ops.patchify(px, cfg.patch_size, self.P["patch.w"].shape[1])
        patches = ops.gemm(cols, self.P["patch.w"], C)
        x = ops.vit_assemble(patches, self.P["cls"], self.P["pos"], B)
        T = x.shape[1]
        x = ops.layernorm(x.view(B * T, C), *self.P["pre"], eps=cfg.layer_norm_eps)
        x = self._stack(x, B, T, causal=False)
        pooled = ops.layernorm(x.view(B, T, C)[:, 0], *self.P["post"], eps=cfg.layer_norm_eps)
        return CLIPOutput(x.view(B, T, C), pooled)


CLIPVisionModel = CLIPVisionModelWithProjection
