"""Engine modules and their fp32 oracle twins on the same seeded weights, for the GPU parity tests of the front end, the inference CLI and
the evaluation CLI.  A plain module: pytest does not collect it."""
import torch

NV, CTX = 4, 128  # pseudo-words per prompt and text width of the reduced-width CLI models


def text_pair(cuda, seed, **cfg):
    from ladi_vton_b200 import CLIPTextModel, synthetic as S
    from ladi_oracle.clip import ClipTextEncoder
    eng = CLIPTextModel(**cfg)
    c = eng.config
    sd = S.random_state_dict(eng.param_shapes(), seed)
    for k in sd:  # unit-variance embeddings (library init scale is irrelevant behind the first LayerNorm, but keep the sum meaningful)
        if "embedding" in k:
            sd[k] = torch.randn(sd[k].shape, generator=torch.Generator().manual_seed(seed + len(k)))
    o = ClipTextEncoder(vocab=c.vocab_size, dim=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers,
                        mlp=c.intermediate_size, max_pos=c.max_position_embeddings).eval()
    o.load_state_dict(sd)
    return eng.load_state_dict(sd).to(cuda), o


def tps_pair(cuda):
    from ladi_oracle import warp as ow
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.warp import ConvNet_TPS, control_points
    eng = ConvNet_TPS(256, 192, 21, 3)
    sd = S.warp_state_dict(eng.param_shapes(), 11, ctrl_bias=torch.atanh(control_points()).view(-1))
    o = ow.ConvNet_TPS(256, 192, 21, 3).eval()
    o.load_state_dict(sd, strict=False)
    return eng.load_state_dict(sd).to(cuda), o


def unet_pair(cuda, widths=(64, 128, 256, 512, 1024)):
    from ladi_oracle import warp as ow
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.warp import UNetVanilla
    eng = UNetVanilla(24, 3, True, widths=widths)
    sd = S.warp_state_dict(eng.param_shapes(), 12)
    o = ow.UNetVanilla(24, 3, True, widths=widths).eval()
    o.load_state_dict(sd)
    return eng.load_state_dict(sd).to(cuda), o


def cli_models(cuda):
    """Engine modules + oracle twins on the same seeded weights."""
    from ladi_oracle.clip import ClipVisionEncoder
    from ladi_oracle.parts import DDIMScheduler as ODDIM, EMASC as OEMASC, InversionAdapter as OAdapter
    from ladi_oracle.pipeline import OracleTryOnPipeline
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    from ladi_vton_b200 import (EMASC, AutoencoderKL, CLIPVisionModelWithProjection, DDIMScheduler, InversionAdapter, UNet2DConditionModel,
                                synthetic as S)
    from ladi_vton_b200.inference import StandInTokenizer
    text, otext = text_pair(cuda, 21, vocab_size=49408, hidden_size=CTX, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2)
    vis = CLIPVisionModelWithProjection(hidden_size=160, intermediate_size=320, num_hidden_layers=2, num_attention_heads=2)
    c = vis.config
    vsd = S.random_state_dict(vis.param_shapes(), 31)
    for k in vsd:
        if "embedding" in k and "patch" not in k:
            vsd[k] = torch.randn(vsd[k].shape, generator=torch.Generator().manual_seed(len(k)))
    ovis = ClipVisionEncoder(dim=c.hidden_size, heads=c.num_attention_heads, layers=c.num_hidden_layers, mlp=c.intermediate_size,
                             image=c.image_size, patch=c.patch_size).eval()
    ovis.load_state_dict(vsd)
    ad = InversionAdapter(input_dim=160, hidden_dim=256, output_dim=CTX * NV, heads=2, mlp_dim=320)
    asd = S.random_state_dict(ad.param_shapes(), 41)
    oad = OAdapter(input_dim=160, hidden_dim=256, output_dim=CTX * NV, heads=2, mlp_dim=320).eval()
    oad.load_state_dict(asd)
    tps, otps = tps_pair(cuda)
    ref, oref = unet_pair(cuda)
    sds = S.build_state_dicts(S.SMALL_UNET, S.SMALL_VAE, seed=5)
    eng = dict(scheduler=DDIMScheduler(), text_encoder=text, vision_encoder=vis.load_state_dict(vsd).to(cuda),
               inversion_adapter=ad.load_state_dict(asd).to(cuda), tps=tps, refinement=ref, tokenizer=StandInTokenizer(),
               unet=UNet2DConditionModel(**S.SMALL_UNET).load_state_dict(sds["unet"]).to(cuda),
               vae=AutoencoderKL(**S.SMALL_VAE).load_state_dict(sds["vae"]).to(cuda),
               emasc=EMASC(*sds["emasc_channels"]).load_state_dict(sds["emasc"]).to(cuda))
    ou = OU(**S.SMALL_UNET).eval()
    ou.load_state_dict(sds["unet"])
    ov = OV(**S.SMALL_VAE).eval()
    ov.load_state_dict(sds["vae"])
    oe = OEMASC(*sds["emasc_channels"]).eval()
    oe.load_state_dict(sds["emasc"])
    orc = dict(tps=otps, refinement=oref, vision_encoder=ovis, inversion_adapter=oad, tokenizer=StandInTokenizer(), text_encoder=otext,
               pipe=OracleTryOnPipeline(ov, ou, ODDIM(), oe, [1, 2, 3, 4, 5]))
    return eng, orc
