"""ORACLE tooling — build-container only.  Golden vectors for the first chunk of an image-to-video request
(oracle/svd_pipeline_oracle.py, the restated StableVideoDiffusionPipeline) at a tiny configuration: arch.TINY UNet,
arch.CLIP_TINY tower, the full-width VAE, 8 frames at a 16 x 16 latent (128 x 128 image), 4 Karras steps.

The weights are synthetic (arch.synth_state_dict), written in the diffusers / transformers layouts and renamed back
through the package's maps, so the fixture also fixes what the maps produce.  The CLIP part is pinned against
transformers' CLIPVisionModelWithProjection on the same weights.  Fixtures keep outputs and seeds only; the decoded
frames (before the 8-bit round trip) are stored in fp16 to stay under 1 MB.    python oracle/make_golden_first_chunk.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_image_oracle as co  # noqa: E402
from oracle import make_golden_conditioner as mgc  # noqa: E402
from oracle import svd_pipeline_oracle as spo  # noqa: E402
from streamingt2v_b200 import arch  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
NAME = "first_chunk_tiny_t8_16x16"
T, H, W, STEPS, SEED = 8, 128, 128, 4, 71
W_SEEDS = dict(unet=72, clip=73, enc=74, dec=75)


def make_image(seed=SEED):
    rng = np.random.default_rng([seed, 77])
    return torch.from_numpy(rng.uniform(0, 1, size=(3, H, W)).astype(np.float32))


def weights():
    """SGM / open_clip named synthetic weights of the tiny first-chunk pipeline."""
    vcfg = arch.VaeConfig()
    return (arch.synth_state_dict(arch.plain_unet_param_shapes(arch.TINY), seed=W_SEEDS["unet"]),
            arch.synth_state_dict(arch.clip_visual_param_shapes(arch.CLIP_TINY), seed=W_SEEDS["clip"]),
            arch.synth_state_dict(arch.vae_encoder_param_shapes(vcfg), seed=W_SEEDS["enc"]),
            arch.synth_state_dict(arch.vae_decoder_param_shapes(vcfg), seed=W_SEEDS["dec"]))


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    vcfg = arch.VaeConfig()
    sd_u, sd_c, sd_e, sd_d = weights()
    # through the published layouts and back
    m = arch.sgm_to_diffusers_svd_keys(arch.TINY)
    sd_u = arch.from_diffusers_svd_state_dict({m[k]: v for k, v in sd_u.items()}, arch.TINY)
    hf = mgc.hf_tower(arch.CLIP_TINY, sd_c)
    sd_c2 = arch.from_hf_clip_vision_state_dict(hf.state_dict(), hf.config)
    assert all(torch.equal(sd_c2[k], sd_c[k]) for k in sd_c)
    me, md = arch.sgm_to_diffusers_vae_encoder_keys(vcfg), arch.sgm_to_diffusers_vae_decoder_keys(vcfg)
    sd_vae = {me[k]: (v.reshape(v.shape[:2]) if ".attentions." in me[k] and v.dim() == 4 else v) for k, v in sd_e.items()}
    sd_vae.update({md[k]: (v.reshape(v.shape[:2]) if ".attentions." in md[k] and v.dim() == 4 else v)
                   for k, v in sd_d.items()})
    sd_e2, sd_d2 = arch.from_diffusers_svd_vae_state_dict(sd_vae, vcfg)
    assert all(torch.equal(sd_e2[k], sd_e[k]) for k in sd_e) and all(torch.equal(sd_d2[k], sd_d[k]) for k in sd_d)

    image = make_image()
    with torch.no_grad():
        out = spo.pipeline(sd_u, arch.TINY, sd_c, arch.CLIP_TINY, sd_e, sd_d, vcfg, image, SEED, num_frames=T,
                           num_inference_steps=STEPS)
        # the pipeline's CLIP path: transformers' tower on the preprocessed clean image
        ref = hf(pixel_values=co.preprocess(image[None] * 2.0 - 1.0)).image_embeds
    clip_err = (out["crossattn"][:, 0] - ref).abs().max().item()
    print(f"[clip] oracle vs transformers: {clip_err:.3e} (max|ref| {ref.abs().max():.3f})")
    assert clip_err <= 1e-4 * ref.abs().max().item()
    f = out["frames"]
    print(f"[frames] {tuple(f.shape)} absmax {f.abs().max():.3f} std {f.std():.3f}; latents std {out['latents'].std():.3f}")
    np.savez_compressed(os.path.join(GOLDEN, f"{NAME}.npz"), crossattn=out["crossattn"].numpy(),
                        concat=out["concat"].numpy(), vector=out["vector"].numpy(), latents=out["latents"].numpy(),
                        frames=f.numpy().astype(np.float16),
                        meta=np.array([T, H, W, STEPS, SEED, *W_SEEDS.values()], np.int64),
                        clip_vs_transformers_maxerr=np.array([clip_err]))
    print("done")


if __name__ == "__main__":
    main()
