"""TEST INFRASTRUCTURE (CPU oracle) -- never imported by the product.

fp32 restatement of the per-batch body of `generate_images_from_tryon_pipe` (src/utils/image_from_pipe.py:42-117, the loop of src/eval.py
and of train_vto.py's validation), composed from the other oracle modules as inference_body.py does for src/inference.py:
  * text_usage 'noun_chunks': the batch's `captions`; 'none': one '' prompt per sample -- both go through the pipeline's tokenizer and
    text encoder (tryon_pipe.py:230-240, `prompt=`);
  * text_usage 'inversion_adapter': the batch's `clip_cloth_features` when present, else CLIP pixel values -> vision tower
    last_hidden_state (:62-70); inversion adapter -> [B, num_vstar, D] (:73-74); prompt template (:57-60); tokenizer (:77-79);
    encode_text_word_embedding(...).last_hidden_state (:82-83), passed as `prompt_embeds=`;
  * the '' negative prompt of classifier-free guidance through the same tokenizer + text encoder (tryon_pipe.py:284-301);
  * the dataset's `warped_cloth` (None with cloth_input_type 'none'), 512x384 output.

Not pinned against the reference's own function by a golden: that function tokenizes through `pipe.tokenizer` (a CLIPTokenizer, whose
vocabulary files are not available offline) and builds a CLIPProcessor from hub files, so it does not run here.  The pieces it is made
of are pinned individually (the pipeline and EMASC by tryon_small.npz, the text path by clip_text_small.npz, the linear and 1x1 EMASC
(emasc_forms.py) by emasc_forms.npz, tests/test_oracle_pins.py and tests/test_emasc_adapter_forms.py).
"""
import torch

from .clip import encode_text_word_embedding
from .inference_body import clip_pixel_values, prompts_for


def _encode(tokenizer, text_encoder, texts, max_length):
    ids = tokenizer(texts, max_length=max_length, padding="max_length", truncation=True, return_tensors="pt").input_ids
    return text_encoder(ids).last_hidden_state


@torch.no_grad()
def run_batch(batch, pipe, inversion_adapter, vision_encoder, tokenizer, text_encoder, text_usage, cloth_input_type, num_vstar,
              guidance_scale, num_inference_steps, generator, cloth_cond_rate=1.0):
    n = len(batch["category"])
    if text_usage == "inversion_adapter":
        feats = batch.get("clip_cloth_features")
        if feats is None:
            feats = vision_encoder(clip_pixel_values(batch["cloth"])).last_hidden_state
        word = inversion_adapter(feats.float())
        word = word.reshape((word.shape[0], num_vstar, -1))
        ids = tokenizer(prompts_for(batch["category"], num_vstar), max_length=tokenizer.model_max_length, padding="max_length",
                        truncation=True, return_tensors="pt").input_ids
        ctx = encode_text_word_embedding(text_encoder, ids, word, num_vstar).last_hidden_state
    elif text_usage in ("noun_chunks", "none"):
        prompts = list(batch["captions"]) if text_usage == "noun_chunks" else [""] * n
        ctx = _encode(tokenizer, text_encoder, prompts, tokenizer.model_max_length)
    else:
        raise ValueError(f"Unknown text usage {text_usage}")
    neg = _encode(tokenizer, text_encoder, [""] * n, ctx.shape[1]) if guidance_scale > 1.0 else None
    warped = batch["warped_cloth"].float() if cloth_input_type == "warped" else None
    return pipe(batch["image"].float(), batch["inpaint_mask"].float(), batch["pose_map"].float(), warped, ctx, neg, height=512, width=384,
                num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, generator=generator, cloth_cond_rate=cloth_cond_rate,
                cloth_input_type=cloth_input_type)
