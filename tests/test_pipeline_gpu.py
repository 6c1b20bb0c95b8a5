"""GPU: one whole request through `pipeline.B200StreamingPipeline` on real components at full geometry (a 360x640
image, 576x1024 chunks, 720x1280 enhance and VFI frames; reduced UNet / CLIP configurations, 2 sampler steps, 8
frames per chunk, seeded synthetic EMA-VFI weights, an identity enhance) equals the same pieces composed by hand with
Pillow's resize, bit for bit: for a request the first chunk covers and for one with an autoregressive chunk."""
import dataclasses

import numpy as np
import pytest
import torch
from PIL import Image

from test_first_chunk_gpu import _pipeline

pytestmark = pytest.mark.gpu
TG, NCOND = 8, 3


@pytest.fixture(scope="module")
def parts(cuda_dev):
    from streamingt2v_b200 import arch
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.stage import B200StreamingSVDStage
    from streamingt2v_b200.vfi import B200VFI, seeded_state_dict
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    syn = arch.synth_state_dict_device
    vcfg = arch.VaeConfig()
    first = _pipeline(cuda_dev, arch.TINY, syn(arch.plain_unet_param_shapes(arch.TINY), cuda_dev, 11),
                      arch.CLIP_TINY, syn(arch.clip_visual_param_shapes(arch.CLIP_TINY), cuda_dev, 12),
                      vcfg, syn(arch.vae_encoder_param_shapes(vcfg), cuda_dev, 13),
                      syn(arch.vae_decoder_param_shapes(vcfg), cuda_dev, 14))
    cfg = dataclasses.replace(arch.TINY, num_frame_conditioning=NCOND)
    wrapper = B200StreamingWrapper(cfg, syn(arch.unet_param_shapes(cfg), cuda_dev, 15),
                                   syn(arch.controlnet_param_shapes(cfg), cuda_dev, 16), cuda_dev)
    stage = B200StreamingSVDStage(wrapper, B200EulerEDMSampler(num_steps=2, num_frames=TG), first.vae_decoder,
                                  first.conditioner, num_conditional_frames=NCOND, device=cuda_dev)

    def first_chunk(image, generator=None):
        return first(image, num_frames=TG, num_inference_steps=2, generator=generator)

    return stage, first_chunk, B200VFI(seeded_state_dict(0), cuda_dev)


@pytest.mark.parametrize("num_frames,n_gen", [(11, 0), (20, 1)])
def test_request_equals_hand_composition(parts, cuda_dev, num_frames, n_gen):
    from streamingt2v_b200.pipeline import B200StreamingPipeline
    from streamingt2v_b200.vfi import interpolate_video
    stage, first_chunk, net = parts
    seen = {}

    def identity_enhance(image, video, *, chunk_size, overlap_size, use_randomized_blending, generator):
        seen.update(image=image.cpu().numpy(), n=video.shape[0], chunk=(chunk_size, overlap_size),
                    on_device=image.is_cuda and video.is_cuda)
        return video

    image = np.random.default_rng(3).integers(0, 256, size=(360, 640, 3), dtype=np.uint8)
    p = B200StreamingPipeline(stage, first_chunk, net, identity_enhance)
    # the autoregressive chunks' conditioner draws its cond_aug noise from torch's global RNG, as the reference does
    torch.manual_seed(4)
    out = p(image, num_frames, generator=torch.Generator().manual_seed(2))
    torch.cuda.synchronize()
    half = (num_frames + 1) // 2
    assert out.shape == (num_frames, 720, 1280, 3) and out.dtype == torch.uint8 and out.is_cuda
    assert seen["n"] == half and seen["chunk"] == (half, 0) and seen["on_device"]
    assert np.array_equal(seen["image"], np.asarray(Image.fromarray(image).resize((1280, 720))))

    # by hand: the stage, uint8 frames, Pillow's resize on the host, VFI
    torch.manual_seed(4)
    video = stage.image_to_video(image, n_gen, first_chunk, generator=torch.Generator().manual_seed(2))
    assert video.shape[0] == TG + n_gen * (TG - NCOND) >= half
    u8 = stage.to_uint8_frames(video)[:half].cpu().numpy()
    frames = np.stack([np.asarray(Image.fromarray(f).resize((1280, 720))) for f in u8])
    want = interpolate_video(torch.from_numpy(frames).to(cuda_dev), num_frames, net)
    torch.cuda.synchronize()
    assert torch.equal(out, want), int((out.int() - want.int()).abs().max())
