"""The try-on models block by block against float64, with normalisation parameters that are not the identity.

Weights.  `varied_norms` draws a state dict as `synthetic.random_state_dict` does, then redraws every GroupNorm / LayerNorm weight as
1 + 0.5 U(-1, 1) and every norm bias as 0.2 N(0, 1), per channel, from a seed.  It selects the norm keys with the predicate
random_state_dict itself uses (`synthetic.is_norm_key`).  With all-ones weights and all-zeros biases a gamma <-> beta swap, an
ln1 <-> ln3 mix-up, a norm1 <-> norm2 exchange or a dropped affine changes nothing; with these weights each of them does.

Block gate.  The float64 oracle (oracle/ladi_oracle) runs the whole model on the GPU, with hooks that capture each block's input.
Each block then runs three ways on that input rounded to bf16, so errors do not compound from block to block:
  engine     the engine's Python sequencing of the block (bit-identical to csrc/engine.cu: test_engine_abi_bit_identity_varied_norms);
  reference  the oracle block in float64;
  port       the oracle block cast to bf16 and run by stock PyTorch (cuDNN / cuBLAS / SDPA): what a straight bf16 port gets.
A block passes when  rel-L2(engine, reference) <= R * rel-L2(port, reference),  rel-L2(engine, reference) <= CAP[kind]  and every
output element of the engine is finite.  R and CAP come from the H100 measurement recorded in DESIGN.md section 4, with headroom.

Step table and context K/V, per element.  `plan_steps` is a sinusoid and three GEMMs.  A worst-case bound carried through three GEMMs
of width 1280 grows past the values themselves, so each stage is checked on its own bf16 input, the previous stage's output, which
the test obtains by running the same kernels on the packed weights; the engine call must return that table bit for bit.
  stage 0  the device kernel evaluates f_k = expf(-x_k), x_k = ln(1e4) k / half, and cosf / sinf(t f_k) in fp32 (no fast math).  The
           argument's error is at most |arg| 2^-21 (1 + x_k): expf's 2 ulp and the product's rounding, plus the rounding of x_k
           (three fp32 operations, 2^-22 |x_k| relative) that expf turns into a relative error of the output.  cosf / sinf add 2^-22
           and the (hi, lo) bf16 pair misses the fp32 value by at most 2^-16 |e| (hi rounds to 2^-8 |e|, lo to 2^-8 of that).  So
           |hi + lo - e| <= |arg| 2^-21 (1 + x_k) + 2^-22 + 2^-16 |e| against the float64 sinusoid e.
  stage k  linear_1 + SiLU (reading the hi and lo columns against the same weights, K = 2 c0), linear_2 + SiLU, and every resnet's
           time_emb_proj + conv1.bias at once with an fp32 output: with a the stage's bf16 input, W_k the state-dict weights rounded
           to bf16 (what the pack holds) and b the fp32 bias, the bound is conv_expect(a W_k^T + b, |a| |W_k|^T + |b|, K, act).
`plan_context` is one GEMM of the bf16 context with the bf16 [to_k; to_v] rows of all cross-attention layers, bound
conv_expect(ctx W^T, |ctx| |W|^T, D, 0).  Both references are assembled from the state dict in module order, independently of the
engine's offset tables.

Faults.  test_injected_faults_are_rejected edits the packed parameters or the offset tables of a dedicated model instance and
requires the block check to reject each fault; it prints whether the end-to-end 2e-2 gate of the whole UNet / VAE encoder would
have seen it.
"""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import conv_expect, ratio, rel_l2

R = 1.25  # engine error / port error, per block (worst measured 0.95, a full CLIP encoder layer of the adapter)
CAP = dict(conv_in=5e-3, resnet=6e-3, transformer=6e-3, down=5e-3, up=5e-3, out=6e-3, attention=5e-3, moments=4e-3, norm_out=4e-3,
           emasc=7e-3, clip_layer=5e-3, adapter=1e-2)  # about twice the worst engine error measured per kind (DESIGN.md section 4)
E2E = 2e-2  # the end-to-end gate of the whole UNet forward and the VAE moments (tests/test_gpu_models.py)


# ================================================================================================================ weights
def varied_norms(shapes, seed):
    """random_state_dict(shapes, seed) with every norm weight redrawn as 1 + 0.5 U(-1, 1) and every norm bias as 0.2 N(0, 1)."""
    from ladi_vton_b200 import synthetic as S
    sd = S.random_state_dict(shapes, seed)
    g = torch.Generator().manual_seed(seed + 7919)
    for k, shp in shapes.items():
        if S.is_norm_key(k):
            sd[k] = 1.0 + 0.5 * (torch.rand(shp, generator=g) * 2 - 1) if k.endswith("weight") else 0.2 * torch.randn(shp, generator=g)
    return sd


def _shapes(model):
    from ladi_vton_b200 import CLIPTextModel, CLIPVisionModelWithProjection, InversionAdapter, synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes
    return {"unet": lambda full: unet_param_shapes({} if full else S.SMALL_UNET),
            "vae": lambda full: vae_param_shapes({} if full else S.SMALL_VAE),
            "adapter": lambda full: InversionAdapter(**({} if full else dict(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256)),
                                                     num_encoder_layers=2).param_shapes(),
            "text": lambda full: CLIPTextModel(**({} if full else dict(vocab_size=1000, hidden_size=64, intermediate_size=128,
                                                                       num_hidden_layers=2, num_attention_heads=1))).param_shapes(),
            "vision": lambda full: CLIPVisionModelWithProjection(**({} if full else dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                                                         num_attention_heads=1, image_size=28))).param_shapes()}[model]


# norms per full-size model: UNet 22 resnets x 2 + 16 transformers x 4 + conv_norm_out; VAE 24 resnets x 2 + 2 attentions + 2 norm_out;
# two-layer adapter 2 x 2 + post_layernorm; text 23 x 2 + final_layer_norm; vision 32 x 2 + pre_layrnorm + post_layernorm
NORMS = dict(unet=109, vae=52, adapter=5, text=47, vision=66)


@pytest.mark.parametrize("model", sorted(NORMS))
def test_varied_norms_redraw_every_norm(model):
    """The redraw reaches every key random_state_dict fills with ones or zeros and no other key (CPU, reduced widths; the full-size
    key sets are only counted)."""
    from ladi_vton_b200 import synthetic as S
    full = _shapes(model)(True)
    assert sum(S.is_norm_key(k) for k in full) == 2 * NORMS[model]
    shapes = _shapes(model)(False)
    plain, varied = S.random_state_dict(shapes, 5), varied_norms(shapes, 5)
    identity = {k for k, v in plain.items() if bool((v == (1.0 if k.endswith("weight") else 0.0)).all())}
    norms = {k for k in shapes if S.is_norm_key(k)}
    assert identity == norms and len(norms) > 0
    for k in shapes:
        v = varied[k]
        if k not in norms:
            assert torch.equal(v, plain[k]), k
        elif k.endswith("weight"):
            assert not bool((v == 1).all()) and float(v.min()) >= 0.5 and float(v.max()) <= 1.5 and v.numel() > 1 and float(v.std()) > 0.1, k
        else:
            assert not bool((v == 0).all()) and float(v.std()) > 0.05, k


# ================================================================================================================ the block harness
def _nhwc(x):
    return x.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous()


def _nchw(y):
    return y.permute(0, 3, 1, 2)


def _rel(y, ref):
    return float((y.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _row(kind, name, y, ref, port):
    return dict(kind=kind, name=name, e=_rel(y, ref), ep=_rel(port, ref), finite=bool(torch.isfinite(y).all()))


def _passes(r):
    return r["finite"] and r["e"] <= R * r["ep"] and r["e"] <= CAP[r["kind"]]


def _print(title, rows):
    print(f"\n{title}: block, engine rel-L2, port rel-L2, ratio (gate: ratio <= {R}, engine <= cap of the kind)")
    for r in rows:
        flag = "" if _passes(r) else "   <-- rejected"
        print(f"  {r['name']:52s} {r['kind']:11s} engine {r['e']:.3e}  port {r['ep']:.3e}  ratio {r['e'] / max(r['ep'], 1e-300):.3f}{flag}")
    worst = {}
    for r in rows:
        q = r["e"] / max(r["ep"], 1e-300)
        if q > worst.get(r["kind"], (0.0, 0.0))[0]:
            worst[r["kind"]] = (q, r["e"])
    print("  worst per kind: " + ", ".join(f"{k} ratio {q:.3f} (engine {e:.2e})" for k, (q, e) in worst.items()))


def _gate(title, rows):
    _print(title, rows)
    bad = [r["name"] for r in rows if not _passes(r)]
    assert not bad, f"{title}: blocks outside the gate: {bad}"


def _hooks(model, pre=(), post=()):
    """Capture the positional inputs of the modules in `pre` and the outputs of those in `post` during the next forward."""
    got, hs = {}, []
    for n in pre:
        hs.append(model.get_submodule(n).register_forward_pre_hook(lambda m, a, n=n: got.__setitem__(n, a)))
    for n in post:
        hs.append(model.get_submodule(n).register_forward_hook(lambda m, a, o, n=n: got.__setitem__("out:" + n, o)))
    return got, hs


def _oracle64(cls, sd, cuda, **cfg):
    with torch.device("meta"):
        o = cls(**cfg).eval()
    o.load_state_dict(sd, assign=True)
    return o.to(cuda, torch.float64)


def _bf16_input(t, cuda):
    """A float64 tensor on the device holding bf16 values: the oracle and the engine read the same numbers."""
    return t.to(torch.bfloat16).to(cuda, torch.float64)


class _Models:
    pass


# ================================================================================================================ UNet
def _unet_blocks(cfg):
    """(oracle module name, kind, channels of the current tensor in an up-block resnet's [x, skip] input) in the engine's packing order."""
    from ladi_vton_b200.unet import SD2_INPAINT_UNET
    cfg = {**SD2_INPAINT_UNET, **cfg}
    ch, L = cfg["block_out_channels"], cfg["layers_per_block"]
    out = [("conv_in", "conv_in", None)]
    for i, t in enumerate(cfg["down_block_types"]):
        for l in range(L):
            out.append((f"down_blocks.{i}.resnets.{l}", "resnet", None))
            if t.startswith("CrossAttn"):
                out.append((f"down_blocks.{i}.attentions.{l}", "transformer", None))
        if i < len(ch) - 1:
            out.append((f"down_blocks.{i}.downsamplers.0", "down", None))
    out += [("mid_block.resnets.0", "resnet", None), ("mid_block.attentions.0", "transformer", None), ("mid_block.resnets.1", "resnet", None)]
    rch = list(reversed(ch))
    c = rch[0]
    for i, t in enumerate(cfg["up_block_types"]):
        prev, c = c, rch[i]
        for l in range(L + 1):
            out.append((f"up_blocks.{i}.resnets.{l}", "resnet", prev if l == 0 else c))
            if t.startswith("CrossAttn"):
                out.append((f"up_blocks.{i}.attentions.{l}", "transformer", None))
        if i < len(ch) - 1:
            out.append((f"up_blocks.{i}.upsamplers.0", "up", None))
    out.append(("conv_norm_out", "out", None))
    return out


def _unet_models(cuda, cfg, seed, hw):
    from ladi_vton_b200 import UNet2DConditionModel, unet_param_shapes
    from ladi_oracle.unet import UNet2DConditionModel as OU
    M = _Models()
    M.cfg, M.dev, M.cache = cfg, cuda, {}
    M.sd = varied_norms(unet_param_shapes(cfg), seed)
    M.blocks = _unet_blocks(cfg)
    M.unet = UNet2DConditionModel(**cfg).load_state_dict(M.sd).to(cuda)
    M.o64 = _oracle64(OU, M.sd, cuda, **cfg)
    M.port = copy.deepcopy(M.o64).to(torch.bfloat16)
    g = torch.Generator().manual_seed(0)
    M.x = _bf16_input(torch.randn((2, 31) + hw, generator=g), cuda)  # batch 2: the CFG layout
    M.ctx = _bf16_input(torch.randn((2, 77, M.unet.config.cross_attention_dim), generator=g), cuda)
    assert sum(k == "resnet" for _, k, _ in M.blocks) == 22 and sum(k == "transformer" for _, k, _ in M.blocks) == 16
    return M


@pytest.fixture(scope="module")
def unet_full(cuda):
    return _unet_models(cuda, {}, 1234, (64, 48))


@pytest.fixture(scope="module")
def unet_small(cuda):
    from ladi_vton_b200 import synthetic as S
    return _unet_models(cuda, S.SMALL_UNET, 1234, (32, 24))


def _unet_capture(M, t):
    if t not in M.cache:
        got, hs = _hooks(M.o64, pre=[n for n, _, _ in M.blocks])
        try:
            with torch.no_grad():
                out = M.o64(M.x, torch.tensor(t, device=M.dev), M.ctx).sample
        finally:
            for h in hs:
                h.remove()
        M.cache[t] = (got, out)
    return M.cache[t]


def _unet_block(M, unet, blk, args, temb_port, step):
    from ladi_vton_b200 import ops
    name, kind, split = blk
    P, cfg = unet.P, unet.config
    x = args[0].to(torch.bfloat16)
    x64 = x.double()
    m, mp = M.o64.get_submodule(name), M.port.get_submodule(name)
    if kind == "resnet":
        ref, port = m(x64, args[1]), mp(x, temb_port)
        srcs = [_nhwc(x)] if split is None else [_nhwc(x[:, :split]), _nhwc(x[:, split:])]  # the up blocks' [x, skip] stays two tensors
        y = unet._resnet(name, srcs, m.conv1.out_channels, step)
    elif kind == "transformer":
        ref, port = m(x64, args[1]), mp(x, args[1].to(torch.bfloat16))
        y = unet._transformer(name, _nhwc(x), m.transformer_blocks[0].attn1.heads)
    elif kind == "conv_in":
        ref, port = m(x64), mp(x)
        B, c, h, w = x.shape
        xin = torch.zeros((B, h, w, unet.in_pitch), dtype=torch.bfloat16, device=M.dev)
        xin[..., :c] = _nhwc(x)
        y = ops.conv2d([xin[..., :c]], P["conv_in.w"], m.out_channels, bias=P["conv_in.b"])
    elif kind == "down":
        ref, port = m(x64), mp(x)
        y = ops.conv2d([_nhwc(x)], P[name + ".conv.w"], m.conv.out_channels, bias=P[name + ".conv.b"], stride=2, pad_lo=1)
    elif kind == "up":
        ref, port = m(x64), mp(x)
        w, b, c = P[name + ".conv.w"], P[name + ".conv.b"], m.conv.out_channels
        y = (ops.conv2d([_nhwc(x)], w, c, bias=b, up2x=True) if unet.fuse_up else ops.conv2d([ops.upsample2x(_nhwc(x))], w, c, bias=b))
    else:  # conv_norm_out + SiLU + conv_out
        o, op = M.o64, M.port
        ref, port = o.conv_out(F.silu(o.conv_norm_out(x64))), op.conv_out(F.silu(op.conv_norm_out(x)))
        hn = ops.groupnorm([_nhwc(x)], *P["conv_norm_out"], cfg.norm_num_groups, cfg.norm_eps, unet.ws, silu=True)
        B, _, h, w = x.shape
        y = torch.empty((B, h, w, cfg.out_channels), dtype=torch.float32, device=M.dev)
        ops.conv2d([hn], P["conv_out.w"], cfg.out_channels, bias=P["conv_out.b"], out=y, out_fp32=True)
    return _nchw(y), ref, port


def _unet_rows(M, unet, t, only=None, plan_t=None):
    got, _ = _unet_capture(M, t)
    unet.plan_steps([t if plan_t is None else plan_t])
    unet.plan_context(M.ctx)
    step = torch.zeros(2, dtype=torch.int32, device=M.dev)
    rows = []
    with torch.no_grad():
        temb_port = M.port.time_emb(torch.tensor(t, device=M.dev), M.x.shape[0])
        for blk in M.blocks:
            if only is None or blk[0] in only:
                rows.append(_row(blk[1], blk[0], *_unet_block(M, unet, blk, got[blk[0]], temb_port, step)))
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unet_full", "unet_small"])
@pytest.mark.parametrize("t", [981, 21])
def test_unet_blocks(cuda, request, which, t):
    """conv_in, 22 resnets (each with its time-embedding slice; the up blocks with their two-tensor [x, skip] input), 16 transformers (each
    with its text K/V), 3 downsamplers, 3 sub-pixel upsamplers and conv_norm_out + SiLU + conv_out, at 64x48 latents (full config) or
    32x24 (SMALL_UNET), batch 2, near both ends of the schedule."""
    M = request.getfixturevalue(which)
    _gate(f"{which} t={t}", _unet_rows(M, M.unet, t))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unet_full", "unet_small"])
def test_unet_forward_vs_float64(cuda, request, which):
    """The whole forward (one engine call) with these weights, against the float64 oracle, at the end-to-end gate."""
    M = request.getfixturevalue(which)
    for t in (981, 21):
        y = M.unet(M.x.float(), torch.tensor(t), M.ctx.float()).sample
        err = rel_l2(y, _unet_capture(M, t)[1])
        print(f"{which} forward t={t}: rel-L2 vs float64 oracle {err:.4f}")
        assert err < E2E


def _stage(a, w, bias, K, act, out_fp32=False):
    """conv_expect of one GEMM stage on its actual (bf16) input `a`, as float64."""
    a = a.double()
    return conv_expect(a @ w.T + bias, a.abs() @ w.abs().T + bias.abs(), K, act, out_fp32=out_fp32)


def _steps_stages(M, ts):
    """The step table stage by stage: the device sinusoid kernel, then the three GEMMs of plan_steps on the packed weights, each on the
    previous stage's bf16 output.  Returns [(what, y, r, bound)] with r and bound from the state dict in float64, and the final table."""
    from ladi_vton_b200 import lib, ops
    sd, dev, unet = M.sd, M.dev, M.unet
    P, c0 = unet.P, unet.config.block_out_channels[0]
    half, kp, n = c0 // 2, P["te1.w"].shape[1] // 2, len(ts)
    w = lambda k: sd[k].to(dev).to(torch.bfloat16).double()
    b = lambda k: sd[k].to(dev).float().double()
    tdev = torch.tensor([float(v) for v in ts], dtype=torch.float32, device=dev)
    pair = torch.empty((n, 2 * kp), dtype=torch.bfloat16, device=dev)
    lib.call("ladi_timestep_embedding", ops._ptr(tdev), n, c0, kp, ops._ptr(pair), ops._stream())
    x = math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=dev) / half
    arg = tdev.double()[:, None] * torch.exp(-x)[None]
    e = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1)
    e_arg = arg.abs() * 2.0 ** -21 * (1.0 + x)[None]
    out = [("sinusoid (hi + lo)", pair[:, :c0].double() + pair[:, kp:kp + c0].double(), e,
            torch.cat([e_arg, e_arg], dim=-1) + 2.0 ** -22 + 2.0 ** -16 * e.abs())]
    w1 = torch.zeros((4 * c0, 2 * kp), dtype=torch.float64, device=dev)
    w1[:, :c0] = w1[:, kp:kp + c0] = w("time_embedding.linear_1.weight")
    e1 = ops.gemm(pair, P["te1.w"], P["te1.w"].shape[0], bias=P["te1.b"], act=ops.ACT_SILU)
    out.append(("linear_1 + SiLU", e1, *_stage(pair, w1, b("time_embedding.linear_1.bias"), 2 * c0, 1)))
    e2 = ops.gemm(e1, P["te2.w"], P["te2.w"].shape[0], bias=P["te2.b"], act=ops.ACT_SILU)
    out.append(("linear_2 + SiLU", e2, *_stage(e1, w("time_embedding.linear_2.weight"), b("time_embedding.linear_2.bias"), 4 * c0, 1)))
    res = [nm for nm, k, _ in M.blocks if k == "resnet"]
    W = torch.cat([w(p + ".time_emb_proj.weight") for p in res])
    bias = torch.cat([(sd[p + ".time_emb_proj.bias"].float() + sd[p + ".conv1.bias"].float()).to(dev).double() for p in res])
    table = ops.gemm(e2, P["temb_all.w"], unet.temb_total, bias=P["temb_all.b"], out_fp32=True)
    r, bound = _stage(e2, W, bias, 4 * c0, 0, out_fp32=True)
    return out, (table, r, bound, res, [sd[p + ".conv1.bias"].shape[0] for p in res])


def _context_expect(M):
    sd, dev = M.sd, M.dev
    w = lambda k: sd[k].to(dev).to(torch.bfloat16).double()
    tr = [n for n, k, _ in M.blocks if k == "transformer"]
    W = torch.cat([torch.cat([w(p + ".transformer_blocks.0.attn2.to_k.weight"), w(p + ".transformer_blocks.0.attn2.to_v.weight")]) for p in tr])
    a = M.ctx.reshape(-1, M.ctx.shape[-1])
    r, bound = conv_expect(a @ W.T, a.abs() @ W.abs().T, a.shape[1], 0)
    return r, bound, tr, [2 * sd[p + ".proj_in.bias"].shape[0] for p in tr]


def _per_part(q, names, cols, what):
    o, worst = 0, 0.0
    for n, c in zip(names, cols):
        v = float(q[:, o:o + c].max())
        worst = max(worst, v)
        print(f"  {what} {n:44s} max err/bound {v:.3f}")
        o += c
    assert o == q.shape[1]
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unet_full", "unet_small"])
def test_plan_steps_and_context_per_element(cuda, request, which):
    """The 50-step table conv1.bias + time_emb_proj(silu(time_embedding(t))) of every resnet, and the K/V of every cross-attention layer,
    element by element against float64 within the bounds of the module docstring."""
    from ladi_vton_b200 import DDIMScheduler
    M = request.getfixturevalue(which)
    unet = M.unet
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    ts = [int(v) for v in sch.timesteps]
    assert len(ts) == 50 and ts[0] == 981 and ts[-1] == 1
    unet._steps = unet._steps_key = None
    y = unet.plan_steps(ts)  # one engine call
    stages, (table, r, bound, res, cols) = _steps_stages(M, ts)
    assert torch.equal(y, table)  # the engine call runs the same kernels on the same operands
    for what, ys, rs, bs in stages:
        q = float(ratio(ys, rs, bs).max())
        print(f"  plan_steps {what:44s} max err/bound {q:.3f}")
        assert q <= 1.0, what
    ws = _per_part(ratio(table, r, bound), res, cols, "plan_steps")
    kv = unet.plan_context(M.ctx)
    rc, bc, tr, ccols = _context_expect(M)
    wc = _per_part(ratio(kv.reshape(rc.shape), rc, bc), tr, ccols, "plan_context")
    print(f"{which}: plan_steps worst err/bound {ws:.3f}, plan_context {wc:.3f}")
    assert ws <= 1.0 and wc <= 1.0


# ================================================================================================================ VAE
FEAT_C = lambda ch, cout: {0: cout, 1: ch[0], 2: ch[1], 3: ch[2], 4: ch[3], 5: ch[3]}  # EMASC output widths per encoder layer
FEAT_F = {0: 1, 1: 1, 2: 1, 3: 2, 4: 4, 5: 8}


def _vae_blocks(cfg):
    ch, L = cfg["block_out_channels"], cfg["layers_per_block"]
    enc = [("encoder.conv_in", "conv_in", None)]
    for i in range(len(ch)):
        enc += [(f"encoder.down_blocks.{i}.resnets.{l}", "resnet", None) for l in range(L)]
        if i < len(ch) - 1:
            enc.append((f"encoder.down_blocks.{i}.downsamplers.0", "down", None))
    mid = lambda p: [(p + ".resnets.0", "resnet", None), (p + ".attentions.0", "attention", None), (p + ".resnets.1", "resnet", None)]
    enc += mid("encoder.mid_block") + [("encoder.conv_norm_out", "moments", None)]
    dec = [("post_quant_conv", "conv_in", None)] + mid("decoder.mid_block")
    for i in range(len(ch)):
        # the first resnet of up block i reads the previous stage's output plus EMASC feature i (in reversed list order)
        dec += [(f"decoder.up_blocks.{i}.resnets.{l}", "resnet", ("decoder.mid_block" if i == 0 else f"decoder.up_blocks.{i - 1}", i) if l == 0 else None)
                for l in range(L + 1)]
        if i < len(ch) - 1:
            dec.append((f"decoder.up_blocks.{i}.upsamplers.0", "up", None))
    dec += [("decoder.conv_norm_out", "norm_out", None), ("decoder.conv_out", "out", None)]
    return enc, dec


@pytest.fixture(scope="module")
def vae_full(cuda):
    from ladi_vton_b200 import AutoencoderKL
    from ladi_vton_b200.vae import SD2_VAE, vae_param_shapes
    from ladi_oracle.vae import AutoencoderKL as OV
    V = _Models()
    V.dev, V.cfg = cuda, dict(SD2_VAE)
    V.sd = varied_norms(vae_param_shapes({}), 1235)
    V.vae = AutoencoderKL().load_state_dict(V.sd).to(cuda)
    V.o64 = _oracle64(OV, V.sd, cuda)
    V.port = copy.deepcopy(V.o64).to(torch.bfloat16)
    V.enc, V.dec = _vae_blocks(V.cfg)
    g = torch.Generator().manual_seed(1)
    H, W = 512, 384
    V.x = _bf16_input(torch.rand((1, 3, H, W), generator=g) * 2 - 1, cuda)
    V.z = _bf16_input(torch.randn((1, 4, H // 8, W // 8), generator=g), cuda)
    fc = FEAT_C(V.cfg["block_out_channels"], V.cfg["out_channels"])
    V.feats = [_bf16_input(0.5 * torch.randn((1, fc[i], H // FEAT_F[i], W // FEAT_F[i]), generator=g), cuda) for i in range(6)]
    with torch.no_grad():
        got, hs = _hooks(V.o64, pre=[n for n, _, _ in V.enc])
        try:
            enc, feats = V.o64.encode(V.x)
        finally:
            for h in hs:
                h.remove()
        V.enc_got, V.moments, V.skips = got, enc.latent_dist.parameters, feats
        got, hs = _hooks(V.o64, pre=[n for n, _, _ in V.dec], post=["decoder.mid_block"] + [f"decoder.up_blocks.{i}" for i in range(3)])
        try:
            V.image = V.o64.decode(V.z, list(V.feats), [0, 1, 2, 3, 4, 5]).sample
        finally:
            for h in hs:
                h.remove()
        V.dec_got = got
    return V


def _padded(x):
    """NHWC bf16 with the pitch rounded up to 8 channels (the layout of the EMASC features), as a view of the first C channels."""
    B, c, h, w = x.shape
    p = torch.zeros((B, h, w, (c + 7) // 8 * 8), dtype=torch.bfloat16, device=x.device)
    p[..., :c] = _nhwc(x)
    return p[..., :c]


def _vae_block(V, vae, blk, got, residual0=True):
    from ladi_vton_b200 import ops
    name, kind, extra = blk
    P, cfg, G = vae.P, vae.config, vae.config.norm_num_groups
    o, op = V.o64, V.port
    args = got[name] if extra is None else (got["out:" + extra[0]],)
    x = args[0].to(torch.bfloat16)
    x64 = x.double()
    m, mp = o.get_submodule(name), op.get_submodule(name)
    B, c, h, w = x.shape
    if kind == "resnet" and extra is not None:
        f = V.feats[::-1][extra[1]]  # decoder.forward reverses the feature list
        ref, port = m(x64 + f), mp(x + f.to(torch.bfloat16))
        y = vae._resnet(name, ops.add(_nhwc(x), _nhwc(f)), m.conv1.out_channels)
    elif kind == "resnet":
        ref, port = m(x64), mp(x)
        y = vae._resnet(name, _nhwc(x), m.conv1.out_channels)
    elif kind == "attention":
        ref, port = m(x64), mp(x)
        y = vae._attn(name, _nhwc(x))
    elif kind == "conv_in" and name == "encoder.conv_in":
        ref, port = m(x64), mp(x)
        xin = _padded(x)
        y = ops.conv2d([xin], P["encoder.conv_in.w"], m.out_channels, bias=P["encoder.conv_in.b"])
    elif kind == "conv_in":  # post_quant_conv (a 1x1 GEMM) + decoder.conv_in
        ref, port = o.decoder.conv_in(m(x64)), op.decoder.conv_in(mp(x))
        cz = cfg.latent_channels
        zin = torch.zeros((B, h, w, 8), dtype=torch.bfloat16, device=V.dev)
        zin[..., :cz] = _nhwc(x)
        zq = torch.zeros((B, h, w, 8), dtype=torch.bfloat16, device=V.dev)
        ops.gemm(zin.view(B * h * w, 8)[:, :cz], P["post_quant.w"], cz, bias=P["post_quant.b"], out=zq.view(B * h * w, 8))
        y = ops.conv2d([zq[..., :cz]], P["decoder.conv_in.w"], o.decoder.conv_in.out_channels, bias=P["decoder.conv_in.b"])
    elif kind == "down":
        ref, port = m(x64), mp(x)
        y = ops.conv2d([_nhwc(x)], P[name + ".conv.w"], c, bias=P[name + ".conv.b"], stride=2, pad_lo=0)
    elif kind == "up":
        ref, port = m(x64), mp(x)
        wt, b = P[name + ".conv.w"], P[name + ".conv.b"]
        y = (ops.conv2d([_nhwc(x)], wt, c, bias=b, up2x=True) if vae.fuse_up else ops.conv2d([ops.upsample2x(_nhwc(x))], wt, c, bias=b))
    elif kind == "moments":  # encoder conv_norm_out + SiLU + conv_out with quant_conv folded in, fp32 out
        e, ep = o.encoder, op.encoder
        ref, port = o.quant_conv(e.conv_out(F.silu(e.conv_norm_out(x64)))), op.quant_conv(ep.conv_out(F.silu(ep.conv_norm_out(x))))
        hn = ops.groupnorm([_nhwc(x)], *P["encoder.conv_norm_out"], G, 1e-6, vae.ws, silu=True)
        y = torch.empty((B, h, w, 2 * cfg.latent_channels), dtype=torch.float32, device=V.dev)
        ops.conv2d([hn], P["enc_out.w"], 2 * cfg.latent_channels, bias=P["enc_out.b"], out=y, out_fp32=True)
    elif kind == "norm_out":  # decoder conv_norm_out + SiLU, then the layer-1 feature
        f1 = V.feats[1]
        ref, port = F.silu(m(x64)) + f1, F.silu(mp(x)) + f1.to(torch.bfloat16)
        y = ops.groupnorm([_nhwc(x)], *P["decoder.conv_norm_out"], G, 1e-6, vae.ws, silu=True, add=_nhwc(f1))
    else:  # decoder conv_out, fp32 out, with the layer-0 (image-space) feature as its residual when int_layers holds 0
        f0 = V.feats[0] if residual0 else None
        ref, port = m(x64), mp(x)
        if f0 is not None:
            ref, port = ref + f0, port + f0.to(torch.bfloat16)
        img = torch.empty((B, h, w, 4), dtype=torch.float32, device=V.dev)
        ops.conv2d([_nhwc(x)], P["decoder.conv_out.w"], cfg.out_channels, bias=P["decoder.conv_out.b"], out=img, out_fp32=True,
                   residual=None if f0 is None else _padded(f0))
        y = img[..., :cfg.out_channels]
    return _nchw(y), ref, port


def _vae_rows(V, vae, blocks, got, only=None):
    rows = []
    with torch.no_grad():
        for blk in blocks:
            if only is not None and blk[0] not in only:
                continue
            if blk[1] == "out":
                for r0, tag in ((True, " int_layers [0..5]"), (False, " int_layers [1..5]")):
                    rows.append(_row(blk[1], blk[0] + tag, *_vae_block(V, vae, blk, got, r0)))
            else:
                rows.append(_row(blk[1], blk[0], *_vae_block(V, vae, blk, got)))
    return rows


@pytest.mark.gpu
def test_vae_encoder_blocks(cuda, vae_full):
    """conv_in, the 8 resnets, the 3 downsamplers (asymmetric padding), the mid block (resnet, d = 512 attention, resnet) and
    conv_norm_out + SiLU + conv_out (quant_conv folded) to the moments, at 512x384."""
    V = vae_full
    _gate("VAE encoder 1x512x384", _vae_rows(V, V.vae, V.enc, V.enc_got))


@pytest.mark.gpu
def test_vae_decoder_blocks(cuda, vae_full):
    """post_quant_conv + conv_in, the mid block, the 12 up-block resnets (the first of each after its EMASC feature is added), the 3
    sub-pixel upsamplers, conv_norm_out + SiLU + the layer-1 feature, and conv_out with and without the layer-0 residual."""
    V = vae_full
    _gate("VAE decoder 1x512x384", _vae_rows(V, V.vae, V.dec, V.dec_got))


@pytest.mark.gpu
def test_vae_encode_decode_vs_float64(cuda, vae_full):
    """The whole encode (moments and skips) and decode (int_layers [1..5] and [0..5]) with these weights, one engine call each, at the
    gates of tests/test_gpu_models.py."""
    V = vae_full
    mom, f = V.vae.encode_nhwc(V.x.float())
    e = rel_l2(_nchw(mom), V.moments)
    print(f"VAE moments rel-L2 vs float64 {e:.4f}")
    assert e < E2E
    for i in (1, 3, 4, 5):
        assert rel_l2(_nchw(f[i]), V.skips[i]) < E2E
    for layers in ([1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5]):
        fl = [V.feats[i] for i in layers]
        with torch.no_grad():
            ref = V.image if 0 in layers else V.o64.decode(V.z, list(fl), layers).sample
            port = V.port.decode(V.z.to(torch.bfloat16), [t.to(torch.bfloat16) for t in fl], layers).sample
        img = V.vae.decode(V.z.float(), [_padded(t) for t in fl], layers).sample
        e, ep = rel_l2(img, ref), rel_l2(port, ref)
        print(f"VAE decode int_layers {layers}: rel-L2 vs float64 engine {e:.4f}, bf16 port {ep:.4f}")
        assert e < min(5e-2, 1.5 * ep)


# ================================================================================================================ EMASC, inversion adapter
@pytest.mark.gpu
@pytest.mark.parametrize("form", [("nonlinear", 3), ("nonlinear", 1), ("linear", 3)])
def test_emasc_layers(cuda, form):
    """Every layer of each EMASC form the engine runs, with (1 - mask) fused as a row scale, at the 512x384 pyramid (one engine call)."""
    from ladi_vton_b200 import EMASC, ops, synthetic as S
    from ladi_oracle.emasc_forms import EMASC as OE
    from ladi_oracle.parts import mask_features
    typ, k = form
    ein, eout = S.EMASC_IN, S.EMASC_OUT
    em = EMASC(ein, eout, kernel_size=k, padding=(k - 1) // 2, type=typ)
    sd = S.random_state_dict(em.param_shapes(), 2 + k)
    o64 = _oracle64(OE, sd, cuda, in_channels=ein, out_channels=eout, kernel_size=k, padding=(k - 1) // 2, type=typ)
    port = copy.deepcopy(o64).to(torch.bfloat16)
    em.load_state_dict(sd).to(cuda)
    g = torch.Generator().manual_seed(3)
    H, W, strides = 512, 384, [1, 1, 2, 4, 8]
    feats = [_bf16_input(torch.randn((2, c, H // s, W // s), generator=g), cuda) for c, s in zip(ein, strides)]
    mask = torch.zeros((2, 1, H, W), device=cuda)
    mask[0, :, 100:400, 80:300] = 1
    mask[1, :, 40:500, 8:200] = 1
    out = em([_nhwc(f) for f in feats], [ops.inv_mask_rows(mask, s) for s in strides])
    with torch.no_grad():
        ref = mask_features(o64(feats), mask.double())
        prt = mask_features(port([f.to(torch.bfloat16) for f in feats]), mask.bfloat16())
    _gate(f"EMASC {typ} {k}x{k}", [_row("emasc", f"conv.{i} ({ein[i]} -> {eout[i]}, /{strides[i]})", _nchw(y), r, p)
                                   for i, (y, r, p) in enumerate(zip(out, ref, prt))])


@pytest.mark.gpu
@pytest.mark.parametrize("layers", [1, 2])
def test_inversion_adapter_blocks(cuda, layers):
    """hubconf.py dims (1280 -> 5120 -> 5120 -> 16384, 16 heads, MLP 5120) with 1 and 2 encoder layers.  Blocks: each full-sequence CLIP
    encoder layer (Python sequencing), and the tail -- the last layer on the CLS row, post_layernorm and the projection head -- as a
    one-layer adapter packed from the same weights (one engine call).  Then the whole adapter against float64 at the 2e-2 gate."""
    from ladi_vton_b200 import InversionAdapter
    from ladi_vton_b200.clip import encoder_layer
    from ladi_oracle.parts import InversionAdapter as OA
    ad = InversionAdapter(num_encoder_layers=layers)
    sd = varied_norms(ad.param_shapes(), 4321 + layers)
    o64 = _oracle64(OA, sd, cuda, num_encoder_layers=layers)
    port = copy.deepcopy(o64).to(torch.bfloat16)
    ad.load_state_dict(sd).to(cuda)
    x = _bf16_input(torch.randn((2, 257, 1280), generator=torch.Generator().manual_seed(5)), cuda)
    B, T, d = x.shape
    got, hs = _hooks(o64, pre=[f"encoder_layers.{l}" for l in range(layers)])
    try:
        with torch.no_grad():
            whole_ref = o64(x)
    finally:
        for h in hs:
            h.remove()
    rows = []
    with torch.no_grad():
        for l in range(layers - 1):
            xi = got[f"encoder_layers.{l}"][0].to(torch.bfloat16)
            y = encoder_layer(ad.P, f"enc{l}.", xi.reshape(B * T, d), B, T, ad.heads, ad.mlp_dim, 1e-5).view(B, T, d)
            rows.append(_row("clip_layer", f"encoder_layers.{l}", y, o64.encoder_layers[l](xi.double()), port.encoder_layers[l](xi)))
        last = f"encoder_layers.{layers - 1}."
        tail = ad if layers == 1 else InversionAdapter(num_encoder_layers=1).load_state_dict(
            {k.replace(last, "encoder_layers.0."): v for k, v in sd.items() if not k.startswith("encoder_layers.") or k.startswith(last)}).to(cuda)
        xt = got[last[:-1]][0].to(torch.bfloat16)
        tail_of = lambda o, v: o.layers(o.post_layernorm(o.encoder_layers[-1](v)[:, 0]))
        rows.append(_row("adapter", f"{last}CLS row + post_layernorm + layers", tail(xt), tail_of(o64, xt.double()), tail_of(port, xt)))
    _gate(f"inversion adapter, {layers} encoder layer(s)", rows)
    err = rel_l2(ad(x), whole_ref)
    print(f"inversion adapter ({layers} layers) rel-L2 vs float64 {err:.4f}")
    assert err < E2E


# ================================================================================================================ whole models again
@pytest.mark.gpu
def test_engine_abi_bit_identity_varied_norms(cuda, unet_full, vae_full):
    """ladi_unet_forward, ladi_vae_encode, ladi_emasc_forward, ladi_vae_decode_emasc and ladi_inversion_adapter_forward (1 and 2 encoder
    layers) at full size with these weights: bit-identical to the Python sequencing the block tests run."""
    from ladi_vton_b200 import EMASC, InversionAdapter, ops, synthetic as S
    M, V = unet_full, vae_full
    unet = M.unet
    unet.plan_steps([981, 21])
    unet.plan_context(M.ctx)
    xin = torch.zeros((2, 64, 48, unet.in_pitch), dtype=torch.bfloat16, device=cuda)
    xin[..., :31] = _nhwc(M.x)
    step = torch.tensor([1, 0], dtype=torch.int32, device=cuda)
    em = EMASC(S.EMASC_IN, S.EMASC_OUT).load_state_dict(S.random_state_dict(S.emasc_param_shapes(S.EMASC_IN, S.EMASC_OUT), 9)).to(cuda)
    ads = []
    for layers in (1, 2):
        ad = InversionAdapter(num_encoder_layers=layers)
        ads.append(ad.load_state_dict(varied_norms(ad.param_shapes(), 4321 + layers)).to(cuda))
    feats = torch.randn((2, 257, 1280), generator=torch.Generator().manual_seed(5))
    mask = torch.zeros((1, 1, 512, 384), device=cuda)
    mask[:, :, 100:400, 80:300] = 1
    assert unet.engine is not None and V.vae.engine is not None and em.engine is not None and all(a.engine is not None for a in ads)

    def run():
        eps = unet.forward_nhwc(xin, step)
        mom, f = V.vae.encode_nhwc(V.x.float())
        sel = [f[i] for i in range(1, 6)]
        inter = em(sel, [ops.inv_mask_rows(mask, 512 // t.shape[1]) for t in sel])
        img = V.vae.decode_nhwc(V.z.float(), inter, [1, 2, 3, 4, 5])
        return ([eps.clone(), mom.clone()] + [t.clone() for t in f[1:]] + [t.clone() for t in inter] + [img[..., :3].clone()]
                + [a(feats).clone() for a in ads])
    a = run()
    ops.PROFILE = []  # the Python sequencing of the same kernels
    try:
        b = run()
    finally:
        ops.PROFILE = None
    for i, (s, t) in enumerate(zip(a, b)):
        assert torch.equal(s, t), f"output {i} of the C++ sequence differs from the Python sequencing"


@pytest.mark.gpu
def test_pipeline_small_varied_norms(cuda):
    """The small try-on pipeline (5 DDIM steps, CFG 7.5, graph replay) with these weights against the fp32 oracle: mean |diff| <= 2/255,
    and the replayed call bit-identical to the first."""
    import numpy as np
    from ladi_vton_b200 import synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes
    from ladi_oracle.parts import DDIMScheduler, EMASC as OE
    from ladi_oracle.pipeline import OracleTryOnPipeline
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    sds = S.build_state_dicts(S.SMALL_UNET, S.SMALL_VAE, seed=1234)
    sds["unet"], sds["vae"] = varied_norms(unet_param_shapes(S.SMALL_UNET), 1234), varied_norms(vae_param_shapes(S.SMALL_VAE), 1235)
    pipe, _ = S.build_pipeline(cuda, S.SMALL_UNET, S.SMALL_VAE, sds=sds)
    ou = OU(**S.SMALL_UNET).eval(); ou.load_state_dict(sds["unet"])
    ov = OV(**S.SMALL_VAE).eval(); ov.load_state_dict(sds["vae"])
    oe = OE(*sds["emasc_channels"]).eval(); oe.load_state_dict(sds["emasc"])
    inp = S.synthetic_inputs(2, 128, 64, ctx_dim=128)
    kw = dict(height=128, width=64, num_inference_steps=5, guidance_scale=7.5)
    ref = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])(
        inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
        inp["negative_prompt_embeds"], generator=torch.Generator().manual_seed(7), **kw)
    pipe.use_cuda_graph = True
    call = lambda: pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"],
                        warped_cloth=inp["warped_cloth"], prompt_embeds=inp["prompt_embeds"],
                        negative_prompt_embeds=inp["negative_prompt_embeds"], generator=torch.Generator().manual_seed(7), output_type="np",
                        **kw).images
    out = call()
    mad = float(np.abs(out - ref).mean()) * 255
    print(f"small pipeline, varied norms: mean|engine-oracle| = {mad:.3f}/255")
    assert out.shape == ref.shape and mad < 2.0
    assert np.array_equal(call(), out)


@pytest.mark.gpu
@pytest.mark.parametrize("full", [False, True])
def test_clip_text_tower_varied_norms(cuda, full):
    """The text tower (layer_norm1 / layer_norm2 of every layer, final_layer_norm) with non-identity norms against the fp32 oracle at
    the gate of tests/test_gpu_frontend.py."""
    from ladi_vton_b200 import CLIPTextModel
    from ladi_oracle.clip import ClipTextEncoder
    cfg = {} if full else dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=3, num_attention_heads=2)
    eng = CLIPTextModel(**cfg)
    c = eng.config
    sd = varied_norms(eng.param_shapes(), 77)
    for k in sd:
        if "embedding" in k:
            sd[k] = torch.randn(sd[k].shape, generator=torch.Generator().manual_seed(77 + len(k)))
    o = ClipTextEncoder(vocab=c.vocab_size, dim=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers,
                        mlp=c.intermediate_size, max_pos=c.max_position_embeddings).eval()
    o.load_state_dict(sd)
    eng.load_state_dict(sd).to(cuda)
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(1, 250, (3, 77), generator=g)
    ids[:, 0] = c.vocab_size - 2
    for b in range(3):
        ids[b, 10 + 3 * b:] = c.vocab_size - 1
    out = eng(ids)
    with torch.no_grad():
        ref = o(ids)
    e1, e2 = rel_l2(out.last_hidden_state, ref.last_hidden_state), rel_l2(out.pooler_output, ref.pooler_output)
    print(f"text tower (full={full}), varied norms: rel-L2 last {e1:.4f}, pooled {e2:.4f}")
    assert e1 < 2e-2 and e2 < 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("full", [False, True])
def test_clip_vision_tower_varied_norms(cuda, full):
    """The vision tower (pre_layrnorm, layer_norm1 / layer_norm2 of every layer, post_layernorm on the pooled row) with non-identity norms
    against the fp32 oracle at the gate of tests/test_gpu_frontend.py."""
    from ladi_vton_b200 import CLIPVisionModelWithProjection
    from ladi_oracle.clip import ClipVisionEncoder
    cfg = {} if full else dict(hidden_size=160, intermediate_size=320, num_hidden_layers=2, num_attention_heads=2, image_size=56)
    eng = CLIPVisionModelWithProjection(**cfg)
    c = eng.config
    sd = varied_norms(eng.param_shapes(), 99)
    for k in sd:
        if "embedding" in k and "patch" not in k:
            sd[k] = torch.randn(sd[k].shape, generator=torch.Generator().manual_seed(len(k)))
    o = ClipVisionEncoder(dim=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers, mlp=c.intermediate_size,
                          image=c.image_size, patch=c.patch_size).eval()
    o.load_state_dict(sd)
    px = torch.randn((1 if full else 2, 3, c.image_size, c.image_size), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        ref = o(px)
    out = eng.load_state_dict(sd).to(cuda)(px)
    e1, e2 = rel_l2(out.last_hidden_state, ref.last_hidden_state), rel_l2(out.pooler_output, ref.pooler_output)
    print(f"vision tower (full={full}), varied norms: rel-L2 last {e1:.4f}, pooled {e2:.4f}")
    assert e1 < 2e-2 and e2 < 2e-2


# ================================================================================================================ injected faults
@pytest.mark.gpu
def test_injected_faults_are_rejected(cuda, unet_full, vae_full):
    """Each fault is injected into a dedicated model instance that runs the Python sequencing (it reads the packed dict P and the offset
    tables the test edits); the block check must reject it.  The end-to-end error of the whole UNet forward / VAE moments is printed
    beside it: the faults that stay under 2e-2 there are the ones only the block check sees."""
    from ladi_vton_b200 import AutoencoderKL, UNet2DConditionModel
    M, V, t = unet_full, vae_full, 981
    u = UNet2DConditionModel().load_state_dict(M.sd).to(cuda)
    u.engine = None
    P, B = u.P, M.x.shape[0]
    xin = torch.zeros((B,) + tuple(M.x.shape[2:]) + (u.in_pitch,), dtype=torch.bfloat16, device=cuda)
    xin[..., :M.x.shape[1]] = _nhwc(M.x)
    ref_out = _unet_capture(M, t)[1]

    def unet_case(edit, blocks, plan_t=None):
        saved = dict(P), dict(u.temb_off), dict(u.kv_off)
        try:
            edit()
            rows = _unet_rows(M, u, t, only=blocks, plan_t=plan_t)
            e2e = rel_l2(_nchw(u.forward_nhwc(xin, torch.zeros(2, dtype=torch.int32, device=cuda))), ref_out)
        finally:
            P.clear(); P.update(saved[0]); u.temb_off.update(saved[1]); u.kv_off.update(saved[2])
            u._steps = u._steps_key = None
        return rows, e2e

    def swap(a, b):
        P[a], P[b] = P[b], P[a]

    r, tr, tb = "down_blocks.1.resnets.1", "down_blocks.1.attentions.0", "down_blocks.1.attentions.0.transformer_blocks.0"
    r0, r1 = "down_blocks.0.resnets.0", "down_blocks.0.resnets.1"
    a0, a1 = "down_blocks.0.attentions.0", "down_blocks.0.attentions.1"
    res = [n for n, k, _ in M.blocks if k == "resnet"]
    cases = [
        ("resnet norm1 <-> norm2 (640 -> 640)", lambda: swap(r + ".n1", r + ".n2"), [r], None),
        ("transformer ln2 gamma <-> beta", lambda: P.__setitem__(tb + ".ln2", P[tb + ".ln2"][::-1]), [tr], None),
        ("transformer ln1 <-> ln3", lambda: swap(tb + ".ln1", tb + ".ln3"), [tr], None),
        ("resnet reads its neighbour's temb_off", lambda: u.temb_off.__setitem__(r1, u.temb_off[r0]), [r1], None),
        ("transformer reads its neighbour's kv_off", lambda: u.kv_off.__setitem__(a1, u.kv_off[a0]), [a1], None),
        ("step table planned for t + 20", lambda: None, res, t + 20),
    ]
    clean, e2e_clean = unet_case(lambda: None, [r, tr, r1, a1] + res)
    _gate("dedicated UNet instance, no fault", clean)
    summary = [("none (UNet)", True, e2e_clean)]
    for what, edit, blocks, plan_t in cases:
        rows, e2e = unet_case(edit, blocks, plan_t)
        _print(f"fault: {what}", rows)
        assert not all(_passes(x) for x in rows), f"the block check missed: {what}"
        summary.append((what, False, e2e))

    v = AutoencoderKL().load_state_dict(V.sd).to(cuda)
    v.engine = None
    gn, n1 = "encoder.mid_block.attentions.0.group_norm", "encoder.mid_block.resnets.0.norm1"
    mid = ["encoder.mid_block.resnets.0", "encoder.mid_block.attentions.0"]
    for what, faulty in (("none (VAE)", False), ("VAE mid-block attention group_norm <-> resnets.0.norm1", True)):
        if faulty:
            v.P[gn], v.P[n1] = v.P[n1], v.P[gn]
        rows = _vae_rows(V, v, V.enc, V.enc_got, only=mid)
        e2e = rel_l2(_nchw(v.encode_nhwc(V.x.float())[0]), V.moments)
        if faulty:
            _print(f"fault: {what}", rows)
            assert not all(_passes(x) for x in rows), f"the block check missed: {what}"
        else:
            _gate("dedicated VAE instance, no fault", rows)
        summary.append((what, not faulty, e2e))
    print("\nfault, end-to-end rel-L2 (whole UNet forward at t=981 / VAE moments), caught by the end-to-end 2e-2 gate:")
    for what, is_clean, e2e in summary:
        print(f"  {what:56s} {e2e:.4f}  {'(no fault)' if is_clean else ('caught' if e2e >= E2E else 'MISSED end to end')}")
