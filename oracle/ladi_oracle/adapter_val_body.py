"""TEST INFRASTRUCTURE (CPU oracle) -- never imported by the product.

fp32 restatement of the per-batch body of `generate_images_inversion_adapter` (src/utils/image_from_pipe.py:139-218, the validation of
src/train_inversion_adapter.py), composed from the other oracle modules as eval_body.py does for `generate_images_from_tryon_pipe`:
the batch's `clip_cloth_features` when present, else CLIP pixel values -> vision tower last_hidden_state (:163-168); inversion adapter
-> [B, num_vstar, D] (:170-171); prompt template (:173-180); tokenizer (:183-185); encode_text_word_embedding(...).last_hidden_state
(:188-190) passed as `prompt_embeds=`; the '' negative prompt of classifier-free guidance through the same tokenizer + text encoder;
the inpainting pipeline at 512x384 with one image per prompt (:193-203).
"""
import torch

from .clip import encode_text_word_embedding
from .eval_body import _encode
from .inference_body import clip_pixel_values, prompts_for


@torch.no_grad()
def run_batch(batch, pipe, inversion_adapter, vision_encoder, tokenizer, text_encoder, num_vstar, guidance_scale, num_inference_steps,
              generator):
    feats = batch.get("clip_cloth_features")
    if feats is None:
        feats = vision_encoder(clip_pixel_values(batch["cloth"])).last_hidden_state
    word = inversion_adapter(feats.float())
    word = word.reshape((word.shape[0], num_vstar, -1))
    ids = tokenizer(prompts_for(batch["category"], num_vstar), max_length=tokenizer.model_max_length, padding="max_length",
                    truncation=True, return_tensors="pt").input_ids
    ctx = encode_text_word_embedding(text_encoder, ids, word, num_vstar).last_hidden_state
    neg = _encode(tokenizer, text_encoder, [""] * len(batch["category"]), ctx.shape[1]) if guidance_scale > 1.0 else None
    return pipe(batch["image"].float(), batch["inpaint_mask"].float(), ctx, neg, height=512, width=384, num_inference_steps=num_inference_steps,
                guidance_scale=guidance_scale, num_images_per_prompt=1, generator=generator)
