"""`EditAnythingLoraModel` - the orchestrator contract of the reference (SURVEY.md §8b row B1) on this backend.

Same constructor arguments, same `process(...)` argument list and return value as the reference class
(editany_lora.py:450-500, 609-938), so `editany_nogradio.py` and the Gradio front ends drive it unchanged:

    refined, output, [full_segmask, mask], prompt = model.process(*input_data["args"], **input_data["kwargs"])

What runs where:
    SAM control map          sam_generator.generate -> host.show_anns          (editany_lora.py:522-525, 426-449)
    pre-processing           host.HWC3 / resize_image / make_inpaint_condition  (:760-784, 822)
    prompt embeddings        host.get_pipeline_embeds                           (:791-793)
    generation + tile pass   editanything_b200.pipeline.StableDiffusionControlNetInpaintPipeline (:858-936)
The semantics (call order, RNG consumption, dtypes, un-normalised 0..255 control map, linear resize of the id map,
PIL mask round trip, one shared generator across the main and the tile pass) follow the reference line by line;
the code is this package's own.

Base models: SD1.5-style 4-channel UNets, and the 9-channel stabilityai/stable-diffusion-2-inpainting with the SD2.1
EditAnything ControlNets (sam2groundingdino_edit.py:36-44), e.g.

    EditAnythingLoraModel(base_model_path="stabilityai/stable-diffusion-2-inpainting",
                          controlmodel_name="LAION Pretrained(v0-4)-SD21", extra_inpaint=False, use_blip=False,
                          lora_model_path=None)

whose tile pass loads runwayml/stable-diffusion-v1-5 separately (editany_lora.py:395-405).

v-prediction base models run too: stabilityai/stable-diffusion-2-1 (768x768, the base of the reference's SD2.1
entry points, sam2image.py:28, sketch2image.py:68) predicts v, which its scheduler_config.json records as
`"prediction_type": "v_prediction"`; the loader carries that into the scheduler, the UniPC swap keeps it and the fused
step converts v to x0 and eps.  An SD2.1 base has no tile ControlNet of its own, so pass one, e.g.

    EditAnythingLoraModel(base_model_path="stabilityai/stable-diffusion-2-1",
                          controlmodel_name="LAION Pretrained(v0-4)-SD21", extra_inpaint=False, use_blip=False,
                          lora_model_path=None, tile_model=...)

and call `process(..., enable_tile=False)`.

Tile refinement: `refine_image_resolution` sets the short side of the tile pass's image as in the reference; the
VAE's attention runs on the fused kernel above 128 x 128 latents, so sizes up to 2048 x 2752 (256 x 344 latents) run
on one 80 GB H100 and are tested there.  Larger sizes are not verified.

LoRA: `lora_model_path` names a kohya `.safetensors` file merged at `lora_weight` into the UNet and the text
encoder of the generation and the tile pipeline before their weights are packed (editany_lora.py:378-381, 413-416;
editanything_b200.lora), e.g. the reference's "Beauty Edit" setup (editany_beauty.py:54-64)

    EditAnythingLoraModel(base_model_path=".../chilloutmix_NiPrunedFp32Fix",
                          lora_model_path=".../cuteGirlMix4_v10.safetensors", use_blip=True, extra_inpaint=True,
                          lora_weight=0.5)

Like the reference, a rebuild of the generation pipeline for another ControlNet (`condition_model`) merges the LoRA
at weight 1.0: it does not pass `lora_weight` on (editany_lora.py:660-666).  `load_lora_weights(pipe, path,
multiplier, device, dtype)` merges further files into a built pipeline.

All-region generation (`process(..., enable_all_generate=True)` with no `mask_image`, the demos' third tab) follows
editany_lora.py:658-676 and :796-812: the generation pipeline is rebuilt for the mode (sharing the packed UNet, VAE
and text encoder of the current one when the LoRA lists match), the mask is all white, and with `extra_inpaint` the
text-to-image `StableDiffusionControlNetPipeline` runs with the SAM ControlNet alone; without it the inpaint pipeline
repaints the whole image.  The tile pass then runs as usual.

Not supported here (raise NotImplementedError instead of diverging silently): reference-only mode (`ref_image`),
the alpha-mixing pipeline.
"""
import copy
import os
import random
from collections import OrderedDict

import numpy as np
import torch

from . import host
from .host import HWC3, get_pipeline_embeds, make_inpaint_condition, resize_image, show_anns

try:
    import cv2
except Exception:  # pragma: no cover
    cv2 = None
try:
    import PIL.Image
except Exception:  # pragma: no cover
    PIL = None

# controlmodel_name -> checkpoint id (editany_lora.py:72-79); ids resolve through EA_MODEL_ROOT (local directories:
# there is no network on the deployment boxes) - see pipeline.resolve_model_path
config_dict = OrderedDict(
    [
        ("LAION Pretrained(v0-4)-SD15", "shgao/edit-anything-v0-4-sd15"),
        ("LAION Pretrained(v0-4)-SD21", "shgao/edit-anything-v0-4-sd21"),
        ("LAION Pretrained(v0-3)-SD21", "shgao/edit-anything-v0-3"),
        ("SAM Pretrained(v0-1)-SD21", "shgao/edit-anything-v0-1-1"),
    ]
)
INPAINT_CONTROLNET = "lllyasviel/control_v11p_sd15_inpaint"
TILE_CONTROLNET = "lllyasviel/control_v11f1e_sd15_tile"
SAM_CHECKPOINT = "models/sam_vit_h_4b8939.pth"


def _device():
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def init_sam_model(sam_generator=None, mask_predictor=None):
    """editany_lora.py:82-95."""
    if sam_generator is not None and mask_predictor is not None:
        return sam_generator, mask_predictor
    from .segment_anything import SamAutomaticMaskGenerator, SamPredictor, sam_model_registry
    sam = sam_model_registry["default"](checkpoint=SAM_CHECKPOINT)
    sam.to(device=_device())
    return (SamAutomaticMaskGenerator(sam) if sam_generator is None else sam_generator,
            SamPredictor(sam) if mask_predictor is None else mask_predictor)


def _lora_list(lora_model_path, lora_weight):
    """The reference merges one LoRA file at `lora_weight` when a path is given (editany_lora.py:378-381, 413-416)."""
    return None if lora_model_path is None else [(lora_model_path, lora_weight)]


def load_lora_weights(pipeline, checkpoint_path, multiplier, device, dtype):
    """editany_lora.py:197-329 on an already built pipeline: merge one kohya `.safetensors` file, or a list of them
    in order, at `multiplier` into the UNet and the text encoder.  `device` and `dtype` are the reference's (it
    reads the file onto `device` and computes the delta in `dtype`, always "cpu" and torch.float32 at its call
    sites); here the delta is always fp32 on the CPU, added to the fp16 weights with one rounding.
    The packed UNet cannot take a delta, so the base UNet is re-read from `pipeline.base_model_dir`, the LoRA list
    the pipeline already carries and then the new files are merged, and the UNet is packed again on the engine's
    backend; the packed ControlNets are kept.  The text encoder is merged in place, or in a copy when another
    pipeline shares it (a tile pipeline built with `share_with`), so that one is not changed.  Every entry is
    checked before the pipeline changes.  Returns the pipeline."""
    from . import lora as L
    from .denoise import DenoiseEngine
    from .loading import load_weights
    from .weights import diffusers_to_ldm
    paths = [checkpoint_path] if isinstance(checkpoint_path, str) else list(checkpoint_path)
    new = L.normalize([(p, multiplier) for p in paths])
    eng = pipeline.engine
    usd = load_weights(os.path.join(pipeline.base_model_dir, "unet"))
    L.merge(pipeline.lora, unet_sd=usd)
    shared = pipeline.text_encoder_shared
    text_encoder = copy.deepcopy(pipeline.text_encoder) if shared else pipeline.text_encoder
    entries = L.plan(new, list(usd), {k: v.shape for k, v in usd.items()}, text_encoder)
    with torch.no_grad():
        L.apply([e for e in entries if e[0] == "unet"], usd)
        engine = DenoiseEngine(eng.cfg, diffusers_to_ldm(usd, "unet", eng.cfg), [], eng.dev, backend=eng.ops,
                               controlnets_packed=eng.cns)
        L.apply([e for e in entries if e[0] != "unet"])
    pipeline.engine, pipeline.text_encoder = engine, text_encoder
    pipeline.text_encoder_shared = False
    pipeline.lora = pipeline.lora + new
    return pipeline


def obtain_generation_model(base_model_path, lora_model_path, controlnet_path, generation_only=False,
                            extra_inpaint=True, lora_weight=1.0, share_with=None):
    """editany_lora.py:343-388: SAM-ControlNet (+ inpaint-ControlNet) pipeline with the UniPC scheduler; for
    all-region generation with `extra_inpaint` (generation_only=True) the text-to-image pipeline with the SAM
    ControlNet alone.  `share_with`: a pipeline of the same base model whose packed UNet, VAE and text encoder are
    reused (StableDiffusionControlNetInpaintPipeline.from_pretrained)."""
    from .pipeline import (ControlNetModel, ControlNetModel2, StableDiffusionControlNetInpaintPipeline,
                           StableDiffusionControlNetPipeline)
    from .schedulers import UniPCMultistepScheduler
    controlnet = [ControlNetModel2.from_pretrained(controlnet_path, torch_dtype=torch.float16)]
    if (not generation_only) and extra_inpaint:
        controlnet.append(ControlNetModel.from_pretrained(INPAINT_CONTROLNET, torch_dtype=torch.float16))
    cls = StableDiffusionControlNetPipeline if generation_only and extra_inpaint else \
        StableDiffusionControlNetInpaintPipeline
    pipe = cls.from_pretrained(base_model_path, controlnet=controlnet, torch_dtype=torch.float16, safety_checker=None,
                               share_with=share_with, lora=_lora_list(lora_model_path, lora_weight))
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    pipe.enable_xformers_memory_efficient_attention()
    pipe.enable_model_cpu_offload()
    return pipe


def obtain_tile_model(base_model_path, lora_model_path, lora_weight=1.0, share_with=None):
    """editany_lora.py:391-423.  `share_with`: a pipeline whose UNet / VAE / text encoder are reused when it was
    built from the same base model directory (the tile pass runs the same SD1.5 weights: 1.7 GB of HBM saved); the
    UNet and text encoder only when it also carries the same LoRA list, so nothing is merged twice.  An
    SD2-inpainting main pipeline is not shared: its tile pass runs on SD1.5 (editany_lora.py:395-405)."""
    from .loading import resolve_model_path
    from .pipeline import ControlNetModel2, StableDiffusionControlNetInpaintPipeline
    from .schedulers import UniPCMultistepScheduler
    controlnet = ControlNetModel2.from_pretrained(TILE_CONTROLNET, torch_dtype=torch.float16)
    if base_model_path in ("runwayml/stable-diffusion-v1-5", "stabilityai/stable-diffusion-2-inpainting"):
        base_model_path = "runwayml/stable-diffusion-v1-5"
    if share_with is not None and getattr(share_with, "base_model_dir", None) != \
            os.path.realpath(resolve_model_path(base_model_path)):
        share_with = None
    pipe = StableDiffusionControlNetInpaintPipeline.from_pretrained(base_model_path, controlnet=controlnet,
                                                                   torch_dtype=torch.float16, safety_checker=None,
                                                                   share_with=share_with,
                                                                   lora=_lora_list(lora_model_path, lora_weight))
    pipe.scheduler = UniPCMultistepScheduler.from_config(pipe.scheduler.config)
    pipe.enable_xformers_memory_efficient_attention()
    pipe.enable_model_cpu_offload()
    return pipe


def save_input_to_file(func):
    """annotator/util.py:75-93: the debug decorator that writes the call's (args, kwargs) to input_data.pkl - the
    file editany_nogradio.py replays.  Written BEFORE returning, after the call, like the reference."""
    import functools
    import pickle

    @functools.wraps(func)
    def wrapper(self, *args, **kwargs):
        result = func(self, *args, **kwargs)
        if os.environ.get("EA_SAVE_INPUT", "1") != "0":
            with open("input_data.pkl", "wb") as f:
                pickle.dump({"args": args, "kwargs": kwargs}, f)
        return result
    return wrapper


class EditAnythingLoraModel:
    def __init__(self, base_model_path="../chilloutmix_NiPrunedFp32Fix", lora_model_path="../40806/mix4",
                 use_blip=True, blip_processor=None, blip_model=None, sam_generator=None,
                 controlmodel_name="LAION Pretrained(v0-4)-SD15", extra_inpaint=True, tile_model=None,
                 lora_weight=1.0, alpha_mixing=None, mask_predictor=None, pipe=None):
        """Reference arguments (editany_lora.py:451-467) plus `pipe`: an already built generation pipeline
        (the reference always builds its own; tests and long-running servers inject one)."""
        if alpha_mixing is not None:
            raise NotImplementedError("alpha_mixing (StableDiffusionControlNetInpaintMixingPipeline)")
        self.device = _device()
        self.use_blip = use_blip
        self.default_controlnet_path = config_dict[controlmodel_name]
        self.base_model_path = base_model_path
        self.lora_model_path = lora_model_path
        self.defalut_enable_all_generate = False          # (sic) the reference's attribute name
        self.extra_inpaint = extra_inpaint
        self.last_ref_infer = False
        self.pipe = pipe if pipe is not None else obtain_generation_model(
            base_model_path, lora_model_path, self.default_controlnet_path, generation_only=False,
            extra_inpaint=extra_inpaint, lora_weight=lora_weight)
        self.sam_generator, self.mask_predictor = init_sam_model(sam_generator, mask_predictor)
        if use_blip:
            if blip_processor is None or blip_model is None:
                from transformers import AutoProcessor, Blip2ForConditionalGeneration
            self.blip_processor = blip_processor if blip_processor is not None else \
                AutoProcessor.from_pretrained("Salesforce/blip2-opt-2.7b")
            self.blip_model = blip_model if blip_model is not None else Blip2ForConditionalGeneration.from_pretrained(
                "Salesforce/blip2-opt-2.7b", torch_dtype=torch.float16, device_map="auto")
        self.tile_pipe = tile_model if tile_model is not None else obtain_tile_model(
            base_model_path, lora_model_path, lora_weight=lora_weight, share_with=self.pipe)

    # -------------------------------------------------------------------------------------------------
    def get_blip2_text(self, image):
        inputs = self.blip_processor(image, return_tensors="pt").to(self.device, torch.float16)
        ids = self.blip_model.generate(**inputs, max_new_tokens=50)
        return self.blip_processor.batch_decode(ids, skip_special_tokens=True)[0].strip()

    def get_sam_control(self, image):
        """editany_lora.py:522-525."""
        return show_anns(self.sam_generator.generate(image))

    def get_click_mask(self, image, clicked_points):
        """editany_lora.py:527-543."""
        self.mask_predictor.set_image(image)
        pts = np.array([p[:2] for p in clicked_points])
        labels = np.array([p[2] for p in clicked_points])
        masks, _, _ = self.mask_predictor.predict(point_coords=pts, point_labels=labels, multimask_output=False)
        return masks

    def _exec_device(self, pipe):
        return getattr(pipe, "_execution_device", self.device)

    # -------------------------------------------------------------------------------------------------
    @torch.inference_mode()
    @save_input_to_file
    def process(self, source_image, enable_all_generate, mask_image, control_scale, enable_auto_prompt, a_prompt,
                n_prompt, num_samples, image_resolution, detect_resolution, ddim_steps, guess_mode, scale, seed, eta,
                enable_tile=True, refine_alignment_ratio=None, refine_image_resolution=None, alpha_weight=0.5,
                use_scale_map=False, condition_model=None, ref_image=None, attention_auto_machine_weight=1.0,
                gn_auto_machine_weight=1.0, style_fidelity=0.5, reference_attn=True, reference_adain=True,
                ref_prompt=None, ref_sam_scale=None, ref_inpaint_scale=None, ref_auto_prompt=False, ref_textinv=True,
                ref_textinv_path=None, ref_scale=None):
        """editany_lora.py:609-938 -> (results_tile: list[PIL], results: list[PIL], [full_segmask, mask], prompt)."""
        if ref_image is not None:
            raise NotImplementedError("reference-only mode (utils/stable_diffusion_reference.py) is not implemented")
        this_controlnet_path = self.default_controlnet_path if condition_model in (None, "EditAnything") else condition_model
        input_image = source_image["image"] if isinstance(source_image, dict) else np.array(source_image, dtype=np.uint8)
        if mask_image is None:
            if enable_all_generate != self.defalut_enable_all_generate:     # :658-667 (lora_weight not passed, sic)
                self.pipe = obtain_generation_model(self.base_model_path, self.lora_model_path, this_controlnet_path,
                                                    enable_all_generate, self.extra_inpaint, share_with=self.pipe)
                self.defalut_enable_all_generate = enable_all_generate
            if enable_all_generate:
                mask_image = np.ones((input_image.shape[0], input_image.shape[1], 3)) * 255
            else:
                mask_image = source_image["mask"]
        else:
            mask_image = np.array(mask_image, dtype=np.uint8)
        if self.default_controlnet_path != this_controlnet_path:          # :679-696
            self.pipe = obtain_generation_model(self.base_model_path, self.lora_model_path, this_controlnet_path,
                                                enable_all_generate, self.extra_inpaint)
            self.default_controlnet_path = this_controlnet_path

        if self.use_blip and enable_auto_prompt:                           # :749-757
            blip2_prompt = self.get_blip2_text(input_image)
            a_prompt = blip2_prompt + "," + a_prompt if len(a_prompt) > 0 else blip2_prompt

        input_image = HWC3(input_image)
        img = resize_image(input_image, image_resolution)
        H, W, _ = img.shape
        # the default SAM model is trained with 1024 size (:765-769)
        full_segmask, detected_map = self.get_sam_control(resize_image(input_image, detect_resolution))
        # id map -> uint8 -> LINEAR resize (sic) -> un-normalised 0..255 float control (:771-778)
        detected_map = HWC3(detected_map.astype(np.uint8))
        detected_map = cv2.resize(detected_map, (W, H), interpolation=cv2.INTER_LINEAR)
        dev = self._exec_device(self.pipe)
        control = torch.from_numpy(detected_map.copy()).float().to(dev).unsqueeze(0).permute(0, 3, 1, 2).clone()

        mask_imag_ori = HWC3(mask_image.astype(np.uint8))
        mask_image_tmp = cv2.resize(mask_imag_ori, (W, H), interpolation=cv2.INTER_LINEAR)
        mask_image = PIL.Image.fromarray(mask_image_tmp)

        if seed == -1:
            seed = random.randint(0, 65535)
        host.seed_everything(seed)
        generator = torch.manual_seed(seed)
        postive_prompt, negative_prompt = a_prompt, n_prompt            # (sic)
        prompt_embeds, negative_prompt_embeds = get_pipeline_embeds(self.pipe, postive_prompt, negative_prompt, dev)

        if enable_all_generate and self.extra_inpaint:                    # :796-812, the text-to-image pipeline
            x_samples = self.pipe(prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                                  num_images_per_prompt=num_samples, num_inference_steps=ddim_steps,
                                  generator=generator, height=H, width=W, image=[control.type(torch.float16)],
                                  controlnet_conditioning_scale=[float(control_scale)], guidance_scale=scale,
                                  guess_mode=guess_mode).images
        else:
            multi_condition_image = [control.type(torch.float16)]
            multi_condition_scale = [float(control_scale)]
            if self.extra_inpaint:
                multi_condition_image.append(make_inpaint_condition(img, mask_image_tmp).type(torch.float16))
                multi_condition_scale.append(1.0)
            # use_scale_map: the reference builds the map (:838-848) but hands it only to the alpha-mixing pipeline
            x_samples = self.pipe(image=img, mask_image=mask_image, prompt_embeds=prompt_embeds,
                                  negative_prompt_embeds=negative_prompt_embeds, num_images_per_prompt=num_samples,
                                  num_inference_steps=ddim_steps, generator=generator,
                                  controlnet_conditioning_image=multi_condition_image, height=H, width=W,
                                  controlnet_conditioning_scale=multi_condition_scale, guidance_scale=scale,
                                  guess_mode=guess_mode).images
        results = [x_samples[i] for i in range(num_samples)]

        results_tile = []
        if enable_tile:                                                    # :885-936
            prompt_embeds, negative_prompt_embeds = get_pipeline_embeds(self.tile_pipe, postive_prompt, negative_prompt,
                                                                        self._exec_device(self.tile_pipe))
            mask_image_tile = None
            for i in range(num_samples):
                img_tile = PIL.Image.fromarray(resize_image(np.array(x_samples[i]), refine_image_resolution))
                if i == 0:
                    mask_image_tile = PIL.Image.fromarray(cv2.resize(mask_imag_ori, (img_tile.size[0], img_tile.size[1]),
                                                                     interpolation=cv2.INTER_LINEAR))
                results_tile += self.tile_pipe(
                    image=img_tile, mask_image=mask_image_tile, prompt_embeds=prompt_embeds,
                    negative_prompt_embeds=negative_prompt_embeds, num_images_per_prompt=1,
                    num_inference_steps=ddim_steps, generator=generator, controlnet_conditioning_image=img_tile,
                    height=img_tile.size[1], width=img_tile.size[0], controlnet_conditioning_scale=1.0,
                    alignment_ratio=refine_alignment_ratio, guidance_scale=scale, guess_mode=guess_mode).images
        return results_tile, results, [full_segmask, mask_image], postive_prompt
