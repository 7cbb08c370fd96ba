"""-m gpu: the whole request path on CUDA with synthetic tiny weights - what `editany_nogradio.py` does
(editany_nogradio.py:1-15): build `EditAnythingLoraModel`, replay an `input_data.pkl`, get (refined, output,
[segmask, mask], prompt) - with the SAM stand-in (`segment_anything` shim: H100 image encoder + PyTorch prompt
encoder / mask decoder / automatic mask generator), the UniPC scheduler and the shared-UNet tile pipeline."""
import pickle

import numpy as np
import pytest
import torch
from PIL import Image

from editanything_b200 import app
from editanything_b200.denoise import DenoiseEngine
from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline
from editanything_b200.sam_spec import SAM_TINY, make_sam_state_dict
from editanything_b200.schedulers import UniPCMultistepScheduler
from editanything_b200.segment_anything import (MaskDecoder, PromptEncoder, SamAutomaticMaskGenerator, SamPredictor,
                                                TwoWayTransformer, build_sam_from_state_dict)
from editanything_b200.unet_spec import TINY, make_state_dict
from editanything_b200.vae import VaeEngine, make_vae_state_dict
from editanything_b200.vae_spec import VaeConfig
from tests.test_app_cpu import _Enc, _Tok, _inputs

pytestmark = pytest.mark.gpu


def _sam(dev):
    torch.manual_seed(0)
    c = SAM_TINY.out_chans
    pe = PromptEncoder(embed_dim=c, image_embedding_size=(SAM_TINY.grid, SAM_TINY.grid),
                       input_image_size=(SAM_TINY.img_size, SAM_TINY.img_size))
    md = MaskDecoder(transformer_dim=c, transformer=TwoWayTransformer(2, c, 8, 2048))
    sd = {"image_encoder." + k: v for k, v in make_sam_state_dict(SAM_TINY, 5).items()}
    sd.update({"prompt_encoder." + k: v for k, v in pe.state_dict().items()})
    sd.update({"mask_decoder." + k: v for k, v in md.state_dict().items()})
    sam = build_sam_from_state_dict(SAM_TINY, sd)
    sam.to(device=dev)
    return sam


def test_sam_shim_on_the_b200_encoder():
    dev = torch.device("cuda:0")
    sam = _sam(dev)
    assert sam.image_encoder.engine is not None and sam.device.type == "cuda"
    img = np.random.RandomState(0).randint(0, 256, (120, 200, 3)).astype(np.uint8)
    pred = SamPredictor(sam)
    pred.set_image(img)
    assert tuple(pred.features.shape) == (1, SAM_TINY.out_chans, SAM_TINY.grid, SAM_TINY.grid)
    masks, scores, low = pred.predict(point_coords=np.array([[50, 60]]), point_labels=np.array([1]), multimask_output=False)
    assert masks.shape == (1, 120, 200) and masks.dtype == bool and np.isfinite(scores).all()
    gen = SamAutomaticMaskGenerator(sam, points_per_side=8, pred_iou_thresh=-1e9, stability_score_thresh=-1.0)
    anns = gen.generate(img)
    assert len(anns) >= 1 and all(a["segmentation"].shape == (120, 200) for a in anns)
    # the encoder feeding the decoder is the engine the parity tests pin (tests/test_gpu_sam.py): same features
    x = sam.preprocess(torch.as_tensor(pred.transform.apply_image(img), device=dev).permute(2, 0, 1)[None].float())
    assert torch.equal(sam.image_encoder(x), sam.image_encoder.engine(x))


def test_process_end_to_end_on_cuda(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    dev = torch.device("cuda:0")
    vcfg = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)
    vsd = dict(make_vae_state_dict(vcfg, 61, part="encoder"))
    vsd.update(make_vae_state_dict(vcfg, 62))
    vae = VaeEngine(vcfg, vsd, dev)
    main_eng = DenoiseEngine(TINY, make_state_dict(TINY, "unet", 51),
                             [make_state_dict(TINY, "controlnet", 52), make_state_dict(TINY, "controlnet", 53)], dev)
    tile_eng = DenoiseEngine(TINY, None, [make_state_dict(TINY, "controlnet", 54)], dev, unet_packed=main_eng.unet)
    tok, enc = _Tok(), _Enc(TINY.context_dim).to(dev)

    class _DevTok(_Tok):
        def __call__(self, *a, **k):
            r = super().__call__(*a, **k)
            r.input_ids = torch.as_tensor(r.input_ids.tolist())
            return r
    tok = _DevTok()

    def mk(eng):
        p = StableDiffusionControlNetInpaintPipeline(eng, vae=vae, text_encoder=enc, tokenizer=tok)
        p.scheduler = UniPCMultistepScheduler.from_config(p.scheduler.config)
        return p
    sam = _sam(dev)
    gen = SamAutomaticMaskGenerator(sam, points_per_side=8, pred_iou_thresh=-1e9, stability_score_thresh=-1.0)
    model = app.EditAnythingLoraModel(base_model_path="base", lora_model_path=None, use_blip=False, sam_generator=gen,
                                      mask_predictor=SamPredictor(sam), tile_model=mk(tile_eng), pipe=mk(main_eng))
    args, kwargs = _inputs()
    args = args[:8] + (128, 128, 20) + args[11:]       # image / detect resolution 128, 20 steps
    kwargs["refine_image_resolution"] = 256
    with open("input_data.pkl", "wb") as f:
        pickle.dump({"args": args, "kwargs": kwargs}, f)
    data = pickle.load(open("input_data.pkl", "rb"))
    refined, output, ref, text = model.process(*data["args"], **data["kwargs"])
    assert text == args[5] and len(output) == 2 and len(refined) == 2
    assert all(isinstance(i, Image.Image) and i.size == (192, 128) for i in output)        # 90x120 -> short side 128, /64
    assert all(isinstance(i, Image.Image) and i.size == (384, 256) for i in refined)
    assert all(np.isfinite(np.array(i)).all() and np.array(i).std() > 0 for i in output + refined)
    masks = model.get_click_mask(np.array(output[0]), [(30, 40, 1), (100, 20, 0)])
    assert masks.shape == (1, 128, 192)
