"""`StableDiffusionControlNetInpaintPipeline` on the H100 denoise engine (SURVEY.md §8b B2).

Same call surface as the reference's diffusers-style pipeline
(`utils/stable_diffusion_controlnet_inpaint.py:391`, `__call__` `:1131-1703`), so
`EditAnythingLoraModel.process` (`editany_lora.py:858-882`) can call it unchanged: same keyword
arguments, same `check_inputs` errors (`:792-979`), same preparation arithmetic (`:142-388`,
`:981-1105`), same loop semantics (`:1540-1664`) — but the loop body (ControlNets -> UNet -> CFG ->
scheduler step -> inpaint blend) is ONE fused, CUDA-graph-replayed launch sequence of
`DenoiseEngine`.  Text encoder, tokenizer and VAE stay the caller's PyTorch modules (duck-typed, once
per image; SURVEY.md §8 R4/R6/R17 "keep in PyTorch").

Both branches of the reference are implemented, selected by `unet.config.in_channels` like there: 4 (any base
model; the source image is encoded and blended back into the kept region) and 9 (an inpainting base model such as
stabilityai/stable-diffusion-2-inpainting: the UNet also reads the mask and the latents of the masked image, the
ControlNets read the 4 latent channels, and there is no blend, so `alignment_ratio` is ignored, :1448-1468,
:1550-1560, :1647-1664).

Not supported (raises NotImplementedError rather than silently diverging): the reference-only mode
(`ref_image`, `utils/stable_diffusion_reference.py`), guess_mode.
"""
import math
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from .denoise import DenoiseEngine, ddim_schedule
from .loading import ControlNetModel, ControlNetModel2  # noqa: F401  (the names editany_lora.py imports)
from .schedulers import UniPCMultistepScheduler

try:  # PIL is only needed for PIL inputs / output_type="pil"
    import PIL.Image
except Exception:  # pragma: no cover
    PIL = None


@dataclass
class StableDiffusionPipelineOutput:
    images: Any
    nsfw_content_detected: Optional[List[bool]]


class DDIMScheduler:
    """DDIM (eta = 0) with the reference sampler's 'uniform' timestep table
    (cldm/ddim_hacked.py:23-52, ldm/modules/diffusionmodules/util.py:46-74) behind the scheduler
    surface the pipeline uses (`set_timesteps/timesteps/init_noise_sigma/scale_model_input/step/
    add_noise/order`, utils/...inpaint.py:1430-1431,1012,1547,1634,1651,1538)."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, linear_start=0.00085, linear_end=0.012, num_train_timesteps=1000):
        self.config = SimpleNamespace(beta_start=linear_start, beta_end=linear_end, beta_schedule="scaled_linear",
                                      num_train_timesteps=num_train_timesteps, prediction_type="epsilon")
        betas = np.linspace(linear_start ** 0.5, linear_end ** 0.5, num_train_timesteps, dtype=np.float64) ** 2
        self.alphas_cumprod = np.cumprod(1.0 - betas, axis=0)
        self.timesteps = None

    def set_timesteps(self, num_inference_steps, device=None):
        ts, a, ap = ddim_schedule(num_inference_steps, self.config.beta_start, self.config.beta_end,
                                  self.config.num_train_timesteps)
        self.timesteps = torch.as_tensor(ts.copy(), dtype=torch.long)
        self._a = {int(t): float(x) for t, x in zip(ts, a)}
        self._ap = {int(t): float(x) for t, x in zip(ts, ap)}

    def coefficients(self, t):
        return self._a[int(t)], self._ap[int(t)]

    def scale_model_input(self, sample, t):
        return sample

    def step(self, model_output, t, sample, **kw):
        a, ap = self.coefficients(t)
        x0 = (sample - math.sqrt(1.0 - a) * model_output) / math.sqrt(a)
        return SimpleNamespace(prev_sample=math.sqrt(ap) * x0 + math.sqrt(1.0 - ap) * model_output,
                               pred_original_sample=x0)

    def add_noise(self, original, noise, timesteps):
        t = int(timesteps.reshape(-1)[0]) if torch.is_tensor(timesteps) else int(timesteps)
        a = float(self.alphas_cumprod[t])
        return math.sqrt(a) * original + math.sqrt(1.0 - a) * noise


# --------------------------------------------------------------------------- input preparation
def prepare_image(image):
    """utils/...inpaint.py:142-163."""
    if isinstance(image, torch.Tensor):
        if image.ndim == 3:
            image = image.unsqueeze(0)
        return image.to(dtype=torch.float32)
    if PIL is not None and isinstance(image, PIL.Image.Image) or isinstance(image, np.ndarray):
        image = [image]
    if PIL is not None and isinstance(image[0], PIL.Image.Image):
        image = np.concatenate([np.array(i.convert("RGB"))[None, :] for i in image], axis=0)
    else:
        image = np.concatenate([i[None, :] for i in image], axis=0)
    image = image.transpose(0, 3, 1, 2)
    return torch.from_numpy(image).to(dtype=torch.float32) / 127.5 - 1.0


def prepare_mask_image(mask_image):
    """utils/...inpaint.py:290-325 (binarise at 0.5; 1 = repaint)."""
    if isinstance(mask_image, torch.Tensor):
        mask_image = mask_image.clone()
        if mask_image.ndim == 2:
            mask_image = mask_image.unsqueeze(0).unsqueeze(0)
        elif mask_image.ndim == 3 and mask_image.shape[0] == 1:
            mask_image = mask_image.unsqueeze(0)
        elif mask_image.ndim == 3:
            mask_image = mask_image.unsqueeze(1)
        mask_image[mask_image < 0.5] = 0
        mask_image[mask_image >= 0.5] = 1
        return mask_image
    if PIL is not None and isinstance(mask_image, PIL.Image.Image) or isinstance(mask_image, np.ndarray):
        mask_image = [mask_image]
    if PIL is not None and isinstance(mask_image[0], PIL.Image.Image):
        m = np.concatenate([np.array(x.convert("L"))[None, None, :] for x in mask_image], axis=0)
        m = m.astype(np.float32) / 255.0
    else:
        m = np.concatenate([x[None, None, :] for x in mask_image], axis=0).astype(np.float32)
    m[m < 0.5] = 0
    m[m >= 0.5] = 1
    return torch.from_numpy(m)


def prepare_controlnet_conditioning_image(cond, width, height, batch_size, num_images_per_prompt, dtype,
                                          do_classifier_free_guidance):
    """utils/...inpaint.py:328-388: tensors pass through UN-normalised (the SAM id map is 0..255,
    editany_lora.py:771-778); PIL images are lanczos-resized and scaled to [0,1]."""
    if not isinstance(cond, torch.Tensor):
        if PIL is not None and isinstance(cond, PIL.Image.Image):
            cond = [cond]
        if PIL is not None and isinstance(cond[0], PIL.Image.Image):
            arr = np.concatenate([np.array(i.resize((width, height), resample=PIL.Image.LANCZOS))[None, :]
                                  for i in cond], axis=0)
            cond = torch.from_numpy(arr.astype(np.float32) / 255.0).permute(0, 3, 1, 2)
        else:
            cond = torch.cat(list(cond), dim=0)
    repeat_by = batch_size if cond.shape[0] == 1 else num_images_per_prompt
    cond = cond.repeat_interleave(repeat_by, dim=0).to(dtype=dtype)
    if do_classifier_free_guidance:
        cond = torch.cat([cond] * 2)
    return cond


def randn_tensor(shape, generator=None, dtype=torch.float32):
    """diffusers' randn_tensor as the pipeline uses it: drawn on the generator's (CPU) device, one
    draw per generator when a list is given (utils/...inpaint.py:998-1008)."""
    if isinstance(generator, list):
        shp = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(shp, generator=g, dtype=dtype) for g in generator], dim=0)
    return torch.randn(tuple(shape), generator=generator, dtype=dtype)


class _NetStub:
    """What the reference reads off `pipe.unet` / `pipe.controlnet` (SURVEY.md §8b B3)."""

    def __init__(self, in_channels, dtype, nets=()):
        self.config = SimpleNamespace(in_channels=in_channels, sample_size=64)
        self.dtype = dtype
        self.nets = list(nets)


class StableDiffusionControlNetInpaintPipeline:
    def __init__(self, engine: DenoiseEngine, vae=None, text_encoder=None, tokenizer=None, scheduler=None,
                 safety_checker=None, feature_extractor=None):
        self.engine = engine
        self.vae, self.text_encoder, self.tokenizer = vae, text_encoder, tokenizer
        self.scheduler = scheduler if scheduler is not None else DDIMScheduler()
        self.safety_checker, self.feature_extractor = safety_checker, feature_extractor
        self.lora = []                     # [(path, multiplier), ...] merged into the UNet and text encoder
        self.text_encoder_shared = False   # another pipeline holds the same text encoder module (share_with)
        dt = engine.hdt
        self.unet = _NetStub(engine.cfg.in_channels, dt)
        self.controlnet = _NetStub(4, dt, nets=[_NetStub(4, dt) for _ in engine.cns])
        self.vae_scale_factor = 8 if vae is None else 2 ** (len(vae.config.block_out_channels) - 1)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, controlnet=None, torch_dtype=None, safety_checker=None,
                        feature_extractor=None, device=None, share_with=None, text_encoder=None, tokenizer=None,
                        vae=None, scheduler=None, lora=None, **_unused):
        """editany_lora.py:372-377: `from_pretrained(base_model_path, controlnet=[...], torch_dtype=torch.float16,
        safety_checker=None)`.  `controlnet`: one `ControlNetModel(2)` or a list (editanything_b200.loading);
        components may be passed in like diffusers allows (text_encoder=, tokenizer=, vae=, scheduler=).
        `lora`: kohya LoRA files [(path, multiplier), ...] merged into the UNet and the text encoder before packing,
        in order, like the reference's `load_lora_weights(pipe, [path], multiplier, "cpu", torch.float32)` right
        after loading (editany_lora.py:378-381, editanything_b200.lora); the ControlNets are not touched.  Recorded
        as `pipe.lora` with real paths.
        `share_with`: another pipeline of the same base model whose VAE and tokenizer are reused, and whose packed
        UNet and text encoder are reused too when it carries the same LoRA list (the tile-refinement pipeline,
        editany_lora.py:391-423); with a different list both are loaded and merged afresh."""
        from .lora import normalize
        from .loading import load_pipeline_parts, resolve_model_path, unet_config_from_diffusers, _read_json
        from .unet_spec import controlnet_config
        dev = torch.device(device) if device is not None else torch.device("cuda:0" if torch.cuda.is_available() else "cpu")
        cns = [] if controlnet is None else (list(controlnet) if isinstance(controlnet, (list, tuple)) else [controlnet])
        lora = normalize(lora)
        base_dir = os.path.realpath(resolve_model_path(pretrained_model_name_or_path))
        shared, shared_te = None, None
        if share_with is not None:
            ucfg = unet_config_from_diffusers(_read_json(os.path.join(base_dir, "unet", "config.json")))
            if share_with.engine.cfg != ucfg:
                raise ValueError(f"share_with runs a UNet {share_with.engine.cfg}, the base model "
                                 f"'{pretrained_model_name_or_path}' has {ucfg}: nothing can be shared")
            if getattr(share_with, "lora", []) == lora:
                shared, shared_te = share_with.engine.unet, share_with.text_encoder
                text_encoder = text_encoder or shared_te
            tokenizer = tokenizer or share_with.tokenizer
            vae = vae or share_with.vae
        ucfg, usd, vae, text_encoder, tokenizer, sched = load_pipeline_parts(
            base_dir, dev, text_encoder=text_encoder, tokenizer=tokenizer, vae=vae, scheduler=scheduler,
            unet_packed=shared, lora=lora, merge_text_encoder=text_encoder is None or text_encoder is not shared_te)
        for c in cns:
            # the ControlNets of a 9-channel inpainting UNet are 4-channel nets (models/cldm_v21.yaml:44)
            if c.cfg != controlnet_config(ucfg):
                raise ValueError(f"ControlNet topology {c.cfg} does not match the UNet {ucfg}")
        eng = DenoiseEngine(ucfg, usd, [c.state_dict_ldm for c in cns], dev, unet_packed=shared)
        pipe = cls(eng, vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, scheduler=sched,
                   safety_checker=safety_checker, feature_extractor=feature_extractor)
        pipe.base_model_dir = base_dir
        pipe.lora = lora
        if shared_te is not None and text_encoder is shared_te:
            share_with.text_encoder_shared = pipe.text_encoder_shared = True
        for stub, c in zip(pipe.controlnet.nets, cns):
            stub.config = c.config
        return pipe

    def load_textual_inversion(self, *a, **k):
        """editany_lora.py:734 calls this inside a try / except that tolerates failure; textual-inversion tokens need
        the diffusers loader mixin, which this backend does not carry."""
        raise NotImplementedError("textual inversion embeddings are not supported by this backend")

    # the reference toggles these; they are no-ops on this backend (nothing to offload or swap)
    def enable_xformers_memory_efficient_attention(self, *a, **k):
        pass

    def enable_model_cpu_offload(self, *a, **k):
        pass

    def enable_vae_slicing(self):
        pass

    def disable_vae_slicing(self):
        pass

    def to(self, *a, **k):
        return self

    @property
    def _execution_device(self):
        return self.engine.dev

    # ---------------------------------------------------------------------------------------
    def check_inputs(self, prompt, image, mask_image, controlnet_conditioning_image, height, width,
                     callback_steps, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                     controlnet_conditioning_scale=None):
        """utils/...inpaint.py:792-979 — same conditions, same exception types."""
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if callback_steps is None or not isinstance(callback_steps, int) or callback_steps <= 0:
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type"
                             f" {type(callback_steps)}.")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError("Cannot forward both `prompt` and `prompt_embeds`. Please make sure to only forward one"
                             " of the two.")
        if prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and"
                             " `prompt_embeds` undefined.")
        if prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError("Cannot forward both `negative_prompt` and `negative_prompt_embeds`.")
        if prompt_embeds is not None and negative_prompt_embeds is not None \
                and prompt_embeds.shape != negative_prompt_embeds.shape:
            raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape when passed"
                             f" directly, but got {prompt_embeds.shape} != {negative_prompt_embeds.shape}.")
        n_nets = len(self.controlnet.nets)
        if n_nets > 1 or isinstance(controlnet_conditioning_image, list):
            if not isinstance(controlnet_conditioning_image, list):
                raise TypeError("For multiple controlnets: `image` must be type `list`")
            if len(controlnet_conditioning_image) != n_nets:
                raise ValueError("For multiple controlnets: `image` must have the same length as the number of"
                                 " controlnets.")
            if isinstance(controlnet_conditioning_scale, list) and len(controlnet_conditioning_scale) != n_nets:
                raise ValueError("For multiple controlnets: When `controlnet_conditioning_scale` is specified as"
                                 " `list`, it must have the same length as the number of controlnets")
        elif not isinstance(controlnet_conditioning_scale, float):
            raise TypeError("For single controlnet: `controlnet_conditioning_scale` must be type `float`.")
        if isinstance(image, torch.Tensor) and not isinstance(mask_image, torch.Tensor):
            raise TypeError("if `image` is a tensor, `mask_image` must also be a tensor")
        if PIL is not None and isinstance(image, PIL.Image.Image) and not isinstance(mask_image, PIL.Image.Image):
            raise TypeError("if `image` is a PIL image, `mask_image` must also be a PIL image")
        if isinstance(image, torch.Tensor):
            if image.ndim not in (3, 4):
                raise ValueError("`image` must have 3 or 4 dimensions")
            if mask_image.ndim not in (2, 3, 4):
                raise ValueError("`mask_image` must have 2, 3, or 4 dimensions")
            ib, ic, ih, iw = (1,) + tuple(image.shape) if image.ndim == 3 else tuple(image.shape)
            if mask_image.ndim == 2:
                mb, mc, mh, mw = (1, 1) + tuple(mask_image.shape)
            elif mask_image.ndim == 3:
                mb, mc, (mh, mw) = mask_image.shape[0], 1, mask_image.shape[1:]
            else:
                mb, mc, mh, mw = mask_image.shape
            if ic != 3:
                raise ValueError("`image` must have 3 channels")
            if mc != 1:
                raise ValueError("`mask_image` must have 1 channel")
            if ib != mb:
                raise ValueError("`image` and `mask_image` mush have the same batch sizes")
            if ih != mh or iw != mw:
                raise ValueError("`image` and `mask_image` must have the same height and width dimensions")
            if image.min() < -1 or image.max() > 1:
                raise ValueError("`image` should be in range [-1, 1]")
            if mask_image.min() < 0 or mask_image.max() > 1:
                raise ValueError("`mask_image` should be in range [0, 1]")
        # :955-979 (a tensor mask has 1 channel, checked above; the reference's latent_channels is the VAE's 4)
        latent_channels = getattr(getattr(self.vae, "config", None), "latent_channels", 4)
        expected = latent_channels if self.unet.config.in_channels == 4 else 2 * latent_channels + 1
        if expected != self.unet.config.in_channels:
            raise ValueError(f"The config of `pipeline.unet` expects {self.unet.config.in_channels} but received"
                             f" non inpainting latent channels: {latent_channels}, mask channels: 1, and masked image"
                             f" channels: {latent_channels}. Please verify the config of `pipeline.unet` and the"
                             " `mask_image` and `image` inputs.")

    def _default_height_width(self, height, width, image):
        """utils/...inpaint.py:1107-1127 (including its shape[3]/shape[2] swap for tensors)."""
        if isinstance(image, list):
            image = image[0]
        if height is None:
            height = image.shape[3] if isinstance(image, torch.Tensor) else image.height
            height = (height // 8) * 8
        if width is None:
            width = image.shape[2] if isinstance(image, torch.Tensor) else image.width
            width = (width // 8) * 8
        return height, width

    def _encode_prompt(self, prompt, num_images_per_prompt, do_cfg, negative_prompt=None, prompt_embeds=None,
                       negative_prompt_embeds=None):
        """utils/...inpaint.py:551-703: with embeds given, repeat per image and stack [negative; positive]."""
        if prompt_embeds is None:
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError("no tokenizer/text_encoder attached: pass `prompt_embeds`")
            prompt = [prompt] if isinstance(prompt, str) else prompt
            ids = self.tokenizer(prompt, padding="max_length", max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors="pt").input_ids
            prompt_embeds = self.text_encoder(ids.to(self._execution_device))[0]
        bs, L, D = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, L, D)
        if do_cfg:
            if negative_prompt_embeds is None:
                if self.tokenizer is None or self.text_encoder is None:
                    raise ValueError("no tokenizer/text_encoder attached: pass `negative_prompt_embeds`")
                neg = [""] * bs if negative_prompt is None else (
                    [negative_prompt] if isinstance(negative_prompt, str) else negative_prompt)
                ids = self.tokenizer(neg, padding="max_length", max_length=L, truncation=True,
                                     return_tensors="pt").input_ids
                negative_prompt_embeds = self.text_encoder(ids.to(self._execution_device))[0]
            negative_prompt_embeds = negative_prompt_embeds.repeat(1, num_images_per_prompt, 1).view(
                bs * num_images_per_prompt, L, D)
            prompt_embeds = torch.cat([negative_prompt_embeds.to(prompt_embeds.device), prompt_embeds])
        return prompt_embeds

    def prepare_latents(self, batch_size, num_channels_latents, height, width, dtype, generator, latents=None):
        shape = (batch_size, num_channels_latents, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an"
                             f" effective batch size of {batch_size}.")
        if latents is None:
            latents = randn_tensor(shape, generator=generator, dtype=dtype)
        return latents * self.scheduler.init_noise_sigma

    def prepare_masked_image_latents(self, masked_image, batch_size, dtype, generator):
        """utils/...inpaint.py:1056-1105 (without the CFG duplication the caller immediately undoes)."""
        if self.vae is None:
            raise ValueError("a VAE is required to encode `image`")
        masked_image = masked_image.to(dtype=dtype)
        vdev = self._vae_device()
        if vdev is not None:
            masked_image = masked_image.to(vdev)          # the reference's `.to(device=device, dtype=dtype)` (:1068)
        if isinstance(generator, list):
            lat = torch.cat([self.vae.encode(masked_image[i:i + 1]).latent_dist.sample(generator=generator[i])
                             for i in range(batch_size)], dim=0)
        else:
            lat = self.vae.encode(masked_image).latent_dist.sample(generator=generator)
        lat = self.vae.config.scaling_factor * lat
        if lat.shape[0] < batch_size:
            if batch_size % lat.shape[0] != 0:
                raise ValueError("The passed images and the required batch size don't match.")
            lat = lat.repeat(batch_size // lat.shape[0], 1, 1, 1)
        return lat

    def _vae_device(self):
        v = self.vae
        for attr in ("device", "dev"):
            d = getattr(v, attr, None)
            if isinstance(d, (torch.device, str)):
                return torch.device(d)
        if hasattr(v, "parameters"):
            try:
                return next(iter(v.parameters())).device
            except StopIteration:
                return None
        return None

    def run_safety_checker(self, image, device, dtype):
        """utils/...inpaint.py:705-716."""
        if self.safety_checker is not None:
            safety_checker_input = self.feature_extractor(self.numpy_to_pil(image), return_tensors="pt").to(device)
            image, has_nsfw_concept = self.safety_checker(images=image,
                                                          clip_input=safety_checker_input.pixel_values.to(dtype))
        else:
            has_nsfw_concept = None
        return image, has_nsfw_concept

    def decode_latents(self, latents):
        """utils/...inpaint.py:718-724.  A `VaeDecoderEngine` (editanything_b200.vae) does the 1/scaling_factor,
        the decode and the (x / 2 + 0.5).clamp(0, 1) in its own kernels; any other object with the diffusers
        AutoencoderKL surface goes through the reference's three lines."""
        if hasattr(self.vae, "decode_latents"):
            image = self.vae.decode_latents(latents)
        else:
            image = self.vae.decode(latents / self.vae.config.scaling_factor).sample
            image = (image / 2 + 0.5).clamp(0, 1)
        return image.cpu().permute(0, 2, 3, 1).float().numpy()

    @staticmethod
    def numpy_to_pil(images):
        images = (images * 255).round().astype("uint8")
        return [PIL.Image.fromarray(i) for i in images]

    # ---------------------------------------------------------------------------------------
    @torch.no_grad()
    def __call__(self, prompt=None, image=None, mask_image=None, controlnet_conditioning_image=None, height=None,
                 width=None, num_inference_steps=50, guidance_scale=7.5, negative_prompt=None,
                 num_images_per_prompt=1, eta=0.0, generator=None, latents=None, prompt_embeds=None,
                 negative_prompt_embeds=None, output_type="pil", return_dict=True, callback=None, callback_steps=1,
                 cross_attention_kwargs=None, controlnet_conditioning_scale=1.0, alignment_ratio=None,
                 guess_mode=False, ref_image=None, ref_mask=None, ref_controlnet_conditioning_scale=1.0,
                 ref_prompt=None, attention_auto_machine_weight=1.0, gn_auto_machine_weight=1.0, style_fidelity=0.5,
                 reference_attn=True, reference_adain=True, ref_scale=1.0):
        if ref_image is not None:
            raise NotImplementedError("reference-only mode needs per-module hooks the fused UNet does not expose")
        if eta != 0.0:
            raise NotImplementedError("only deterministic sampling (eta = 0) is fused")
        height, width = self._default_height_width(height, width, controlnet_conditioning_image)
        self.check_inputs(prompt, image, mask_image, controlnet_conditioning_image, height, width, callback_steps,
                          negative_prompt, prompt_embeds, negative_prompt_embeds, controlnet_conditioning_scale)
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None:
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        N = batch_size * num_images_per_prompt
        do_cfg = guidance_scale > 1.0
        if not do_cfg:
            raise NotImplementedError("guidance_scale <= 1 (no classifier-free guidance) is not fused")
        n_nets = len(self.controlnet.nets)
        if isinstance(controlnet_conditioning_scale, float):
            controlnet_conditioning_scale = [controlnet_conditioning_scale] * n_nets
        if not isinstance(controlnet_conditioning_image, list):
            controlnet_conditioning_image = [controlnet_conditioning_image]

        prompt_embeds = self._encode_prompt(prompt, num_images_per_prompt, do_cfg, negative_prompt, prompt_embeds,
                                            negative_prompt_embeds)
        edt = prompt_embeds.dtype
        image = prepare_image(image)
        mask_image = prepare_mask_image(mask_image)
        conds = [prepare_controlnet_conditioning_image(c, width, height, N, num_images_per_prompt, torch.float32,
                                                       do_cfg) for c in controlnet_conditioning_image]

        self.scheduler.set_timesteps(num_inference_steps, device=self._execution_device)
        timesteps = self.scheduler.timesteps
        lat = self.prepare_latents(N, 4, height, width, edt, generator, latents)
        noise = lat
        eng = self.engine
        dev = eng.dev
        inpaint_unet = self.unet.config.in_channels != 4
        if inpaint_unet:
            # 9-channel branch (:1396, :1448-1468): the mask at latent size and the latents of the masked image are
            # extra UNet inputs; the unmasked image is not encoded and nothing is blended
            masked_image = image * (mask_image < 0.5)
            mask_lat = F.interpolate(mask_image, size=(height // self.vae_scale_factor, width // self.vae_scale_factor))
            mask_lat = mask_lat.to(edt)
            if mask_lat.shape[0] < N:
                if N % mask_lat.shape[0] != 0:
                    raise ValueError("The passed mask and the required batch size don't match.")
                mask_lat = mask_lat.repeat(N // mask_lat.shape[0], 1, 1, 1)
            masked_lat = self.prepare_masked_image_latents(masked_image, N, edt, generator)
            mask_lat, masked_lat = mask_lat.to(dev, torch.float32), masked_lat.to(dev, torch.float32)
            alignment_ratio = None
        else:
            init_lat = self.prepare_masked_image_latents(image, N, edt, generator)
            mh, mw = mask_image.shape[2], mask_image.shape[3]
            # NB the reference names these (w, h) but they are (H, W) of the NCHW mask (:1484-1489)
            m = F.interpolate(mask_image, (mh // 8, mw // 8), mode="nearest").to(lat.dtype)
            m = 1 - m                                       # 1 = keep the original image
            if m.shape[0] < N:
                m = m.repeat(N // m.shape[0], 1, 1, 1)

        eng.prepare(prompt_embeds, conds, controlnet_conditioning_scale, guess_mode=guess_mode, cfg_duplicated=do_cfg)
        # fused step: the built-in DDIM, and UniPC (what every reference entry point installs, editany_lora.py:383,418)
        # through its per-step coefficient rows; any other scheduler object runs eng.eps + scheduler.step
        unipc = isinstance(self.scheduler, UniPCMultistepScheduler) and self.scheduler.config.solver_order <= 2
        fused = isinstance(self.scheduler, DDIMScheduler) or unipc
        n_t = len(timesteps)
        blend_steps = 0 if alignment_ratio is None else sum(1 for i in range(n_t) if i < n_t * alignment_ratio)
        if blend_steps and blend_steps >= n_t:
            # the reference indexes timesteps[i + 1] (:1652): alignment_ratio = 1.0 raises there too
            raise IndexError("alignment_ratio covers the last step: timesteps[i + 1] is out of range")
        # everything below lives on the execution device (the noise was DRAWN on the generator's device above,
        # like diffusers' randn_tensor, then moved - utils/...inpaint.py:998-1012)
        lat = lat.to(dev, torch.float32)
        if inpaint_unet:
            noise_d = init_d = m_d = None
        else:
            noise_d, init_d, m_d = noise.to(dev, torch.float32), init_lat.to(dev, torch.float32), m.to(dev, torch.float32)
        if fused:
            acp = self.scheduler.alphas_cumprod
            coefs = [(float(acp[int(t)]), float(acp[int(t)])) for t in timesteps] if unipc else \
                [self.scheduler.coefficients(t) for t in timesteps]
            # the kept region of step i is add_noise(init, noise, timesteps[i + 1]) while i < len * alignment_ratio
            # (:1647-1656).  With a callback the blend runs on the host side AFTER the callback, like the reference
            # (:1640-1656 calls back with the un-blended latents); otherwise it is fused into the step's last kernel.
            host_blend = callback is not None and blend_steps > 0
            k_next = [(math.sqrt(float(acp[int(timesteps[i + 1])])), math.sqrt(1.0 - float(acp[int(timesteps[i + 1])])))
                      if i < blend_steps else (1.0, 0.0) for i in range(n_t)]
            on = [1.0 if (i < blend_steps and not host_blend) else 0.0 for i in range(n_t)]
            eng.set_schedule([int(t) for t in timesteps], [c[0] for c in coefs], [c[1] for c in coefs],
                             blend=([k[0] for k in k_next], [k[1] for k in k_next], on),
                             multistep=self.scheduler.coefficient_rows() if unipc else None)
            if inpaint_unet:
                eng.set_unet_condition(mask_lat, masked_lat)
            eng.begin(lat, guidance_scale, known_nchw=init_d if blend_steps else None,
                      mask_n1hw=m_d if blend_steps else None, noise_nchw=noise_d if blend_steps else None)
            for i, t in enumerate(timesteps):
                eng.step()
                if callback is not None and i % callback_steps == 0:
                    callback(i, t, eng.latents())
                if host_blend and i < blend_steps:
                    eng.blend_now(k_next[i][0], k_next[i][1])
            lat = eng.latents()
        else:
            if inpaint_unet:
                cond = torch.cat([torch.cat([mask_lat] * 2), torch.cat([masked_lat] * 2)], 1)
            for i, t in enumerate(timesteps):
                x_in = self.scheduler.scale_model_input(torch.cat([lat] * 2), t)
                if inpaint_unet:
                    x_in = torch.cat([x_in, cond], 1)                                  # :1550-1558
                eps = eng.eps(x_in, float(t))
                e = eps[:N] + guidance_scale * (eps[N:] - eps[:N])
                lat = self.scheduler.step(e, t, lat).prev_sample
                if callback is not None and i % callback_steps == 0:
                    callback(i, t, lat)
                if i < blend_steps:
                    lat = self.scheduler.add_noise(init_d, noise_d, timesteps[i + 1]) * m_d + lat * (1 - m_d)
        if not inpaint_unet and (alignment_ratio is None or alignment_ratio == 1.0):
            lat = init_d * m_d + lat * (1 - m_d)                                   # :1658-1664

        if output_type == "latent":
            images, nsfw = lat, None
        else:
            if self.vae is None:
                raise ValueError("a VAE is required unless output_type='latent'")
            images = self.decode_latents(lat.to(next(iter(self.vae.parameters())).dtype)
                                         if hasattr(self.vae, "parameters") else lat)
            images, nsfw = self.run_safety_checker(images, dev, edt)
            if output_type == "pil":
                images = self.numpy_to_pil(images)
        if not return_dict:
            return images, nsfw
        return StableDiffusionPipelineOutput(images=images, nsfw_content_detected=nsfw)
