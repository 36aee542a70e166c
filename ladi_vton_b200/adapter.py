"""H100-native InversionAdapter -- drop-in for the reference's src/models/inversion_adapter.py:5-28 built with the dims of
hubconf.py:16-27 (CLIP ViT-H vision hidden 1280, 16 heads of 80, MLP 5120; projection 1280 -> 5120 -> 5120 -> 16384) and called at
src/inference.py:276-277.  State-dict keys: encoder_layers.{l}.{self_attn.{q,k,v,out}_proj, layer_norm1, mlp.fc1, mlp.fc2, layer_norm2}
for l < num_encoder_layers, post_layernorm, layers.{0,3,6}.

The release checkpoints have one encoder layer; the training scripts (train_inversion_adapter.py, train_vto.py `--num_encoder_layers`)
can make more.  Layers 0..L-2 are full CLIP encoder layers over all 257 tokens (the arithmetic of clip.encoder_layer).  Only the CLS
row of the last layer's output is consumed (inversion_adapter.py:26), so after its LayerNorm-1 and the K/V projection of all tokens,
everything (query, attention, out-proj, MLP, projection head) runs on one row per image: 136 M weights are read once per call -- an
HBM-bound chain of GEMMs on the wgmma kernel with GELU(erf) / residual epilogues.
"""
import torch

from . import engine as eng, lib, ops
from .clip import encoder_layer, encoder_layer_shapes, pack_encoder_layer
from .module import PackedModule
from .weights import f32, pack_linear


class InversionAdapter(PackedModule):
    def __init__(self, input_dim=1280, hidden_dim=5120, output_dim=16384, config=None, num_encoder_layers=1, dropout=0.5, heads=16, mlp_dim=5120):
        if config is not None:  # accept the reference's `config=config.vision_config`
            heads = getattr(config, "num_attention_heads", heads)
            mlp_dim = getattr(config, "intermediate_size", mlp_dim)
        if int(num_encoder_layers) < 1:
            raise ValueError(f"num_encoder_layers must be >= 1, got {num_encoder_layers}")
        self.num_encoder_layers = int(num_encoder_layers)
        self.dim, self.hidden, self.out_dim, self.heads, self.mlp_dim = input_dim, hidden_dim, output_dim, heads, mlp_dim

    def param_shapes(self):
        d, S = self.dim, {}
        for l in range(self.num_encoder_layers):
            encoder_layer_shapes(S, f"encoder_layers.{l}.", d, self.mlp_dim)
        S["post_layernorm.weight"], S["post_layernorm.bias"] = (d,), (d,)
        S["layers.0.weight"], S["layers.0.bias"] = (self.hidden, d), (self.hidden,)
        S["layers.3.weight"], S["layers.3.bias"] = (self.hidden, self.hidden), (self.hidden,)
        S["layers.6.weight"], S["layers.6.bias"] = (self.out_dim, self.hidden), (self.out_dim,)
        return S

    def _pack_weights(self):
        g = lambda k: self._sd[k].to(self.device, torch.float32)
        L = self.num_encoder_layers
        e = f"encoder_layers.{L - 1}."
        P = {}
        for l in range(L - 1):  # full-sequence layers; the last one is packed below for its CLS-row form
            pack_encoder_layer(P, f"enc{l}.", g, f"encoder_layers.{l}.")
        P["ln1"] = (f32(g(e + "layer_norm1.weight")), f32(g(e + "layer_norm1.bias")))
        P["ln2"] = (f32(g(e + "layer_norm2.weight")), f32(g(e + "layer_norm2.bias")))
        P["lnp"] = (f32(g("post_layernorm.weight")), f32(g("post_layernorm.bias")))
        P["kv.w"] = pack_linear(torch.cat([g(e + "self_attn.k_proj.weight"), g(e + "self_attn.v_proj.weight")]))
        P["kv.b"] = f32(torch.cat([g(e + "self_attn.k_proj.bias"), g(e + "self_attn.v_proj.bias")]))
        for n, k in (("q", e + "self_attn.q_proj"), ("o", e + "self_attn.out_proj"), ("fc1", e + "mlp.fc1"), ("fc2", e + "mlp.fc2"),
                     ("l0", "layers.0"), ("l3", "layers.3"), ("l6", "layers.6")):
            P[n + ".w"], P[n + ".b"] = pack_linear(g(k + ".weight")), f32(g(k + ".bias"))
        self.P = P

    def _make_engine(self):
        return eng.Engine(eng.flatten(self.P, "adapter."), adapter_dim=self.dim, adapter_heads=self.heads, adapter_mlp=self.mlp_dim,
                          adapter_hidden=self.hidden, adapter_out=self.out_dim)

    def __call__(self, x):
        """x [B, 257, 1280] (CLIP vision last_hidden_state, any float dtype) -> [B, 16384] bf16."""
        P, d = self.P, self.dim
        B, T, _ = x.shape
        hd = d // self.heads
        xb = x.to(self.device, torch.bfloat16).contiguous()
        if self.use_engine():  # one ABI call (csrc/engine.cu adapter_forward)
            out = torch.empty((B, self.out_dim), dtype=torch.bfloat16, device=self.device)
            ws = self.engine.workspace(eng.MODULE_ADAPTER, B, T, 0)
            lib.call("ladi_inversion_adapter_forward", self.engine.h, ops._ptr(xb), B, T, ops._ptr(out), ops._ptr(ws), ws.numel(), ops._stream())
            return out
        if self.num_encoder_layers > 1:
            xt = xb.view(B * T, d)
            for l in range(self.num_encoder_layers - 1):
                xt = encoder_layer(P, f"enc{l}.", xt, B, T, self.heads, self.mlp_dim, 1e-5)
            xb = xt.view(B, T, d)
        y = ops.layernorm(xb.view(B * T, d), *P["ln1"])                                  # pre-LN over all tokens
        kv = ops.gemm(y, P["kv.w"], 2 * d, bias=P["kv.b"]).view(B, T, 2 * d)
        y0 = y.view(B, T, d)[:, 0]                                                      # CLS rows, pitch T*d
        q0 = ops.gemm(y0, P["q.w"], d, bias=P["q.b"])
        a = ops.cls_attention(q0, kv, self.heads, hd, hd ** -0.5)
        x0 = ops.gemm(a, P["o.w"], d, bias=P["o.b"], residual=xb[:, 0])                 # x + attn
        h = ops.gemm(ops.layernorm(x0, *P["ln2"]), P["fc1.w"], self.mlp_dim, bias=P["fc1.b"], act=ops.ACT_GELU)
        x0 = ops.gemm(h, P["fc2.w"], d, bias=P["fc2.b"], residual=x0)                   # x + mlp
        z = ops.layernorm(x0, *P["lnp"])
        z = ops.gemm(z, P["l0.w"], self.hidden, bias=P["l0.b"], act=ops.ACT_GELU)        # Dropout inactive in eval
        z = ops.gemm(z, P["l3.w"], self.hidden, bias=P["l3.b"], act=ops.ACT_GELU)
        return ops.gemm(z, P["l6.w"], self.out_dim, bias=P["l6.b"])
