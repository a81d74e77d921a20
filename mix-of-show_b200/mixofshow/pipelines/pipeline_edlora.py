"""Drop-in for the reference's `mixofshow/pipelines/pipeline_edlora.py`: `bind_concept_prompt` and `EDLoRAPipeline`
with the same constructor / `set_new_concept_cfg` / `set_controller` / `__call__` surface, and the diffusers
`StableDiffusionPipeline` the reference imports from the same module (test_edlora.py:16, train_edlora.py:18): the sampler
of vanilla LoRA checkpoints (`convert_edlora(pipe, ckpt, enable_edlora=False, alpha)`), prompts encoded unbound, one CLIP
pass per prompt, one [B, 77, 768] embedding for every cross-attention layer (the UNet's default processors).

The denoise loop (reference :271-301) runs on the GPU engine: per step one captured UNet graph (CFG batch 2) and
ONE fused kernel for CFG combine + DPM-Solver++(2M) update + re-duplication of the latents (`mos_cfg_dpmpp_step`).
With `cfg_group` two ranks share one call: each runs one CFG half at batch 1 and they exchange eps once per step
(`denoise_latents`, shared with the regional pipeline).
Prompt encoding and image decoding run on the GPU CLIP / VAE engines (mixofshow/models/clip_b200.py, vae_b200.py) when
`from_pretrained` finds `text_encoder/` and `vae/`; without them pass `prompt_embeds` and request `output_type='latent'`.
"""
from types import SimpleNamespace
from typing import List, Optional, Union

import torch

from mixofshow.models.edlora import (revise_edlora_unet_attention_controller_forward,
                                     revise_edlora_unet_attention_forward)
from mos_b200 import dp, ops
from mos_b200.scheduler import DPMSolverPP2M


def numpy_to_pil(images):
    """[N,H,W,3] floats in [0,1] -> list of PIL images (diffusers `DiffusionPipeline.numpy_to_pil`, reached from the
    reference at pipeline_edlora.py:313), so that `.images[0].save(...)` works as in the reference's scripts."""
    from PIL import Image
    if images.ndim == 3:
        images = images[None]
    return [Image.fromarray(im) for im in (images * 255).round().astype('uint8')]


def bind_concept_prompt(prompts, new_concept_cfg):
    """Each prompt becomes 16 layer-specific prompts; `concept_name` -> `concept_token_names[layer]`
    (reference :18-29). Output order: prompt-major, layer fastest."""
    if isinstance(prompts, str):
        prompts = [prompts]
    new_prompts = []
    for prompt in prompts:
        per_layer = [prompt] * 16
        for concept_name, new_token_cfg in new_concept_cfg.items():
            per_layer = [p.replace(concept_name, new_name)
                         for p, new_name in zip(per_layer, new_token_cfg['concept_token_names'])]
        new_prompts.extend(per_layer)
    return new_prompts


def denoise_latents(unet, scheduler, latents, guidance_scale, prompt_embeds, cross_attention_kwargs=None,
                    adapter_state=None, controller=None, callback=None, callback_steps=1, cfg_group=None):
    """The denoise loop of both pipelines (reference pipeline_edlora.py:271-301, pipeline_regionally_t2iadapter.py:548-580),
    over `scheduler.timesteps`; updates and returns `latents` [n, 4, h, w] (already scaled by init_noise_sigma).
    `prompt_embeds` and the region embeddings of `cross_attention_kwargs['region_list']` hold the CFG halves uncond | cond
    along the batch ([2n, ...] with guidance > 1); `adapter_state` holds the adapter residuals once ([n, C, h', w']).

    One prepared session: weights verified / packed and the step-invariant inputs uploaded ONCE; a step is then one graph
    replay + one fused CFG / DPM-Solver++ kernel, with no host synchronisation inside the loop.

    With `cfg_group` (two ranks, dp.check_cfg_group) group rank i runs only half i (0 = uncond, 1 = cond) as a batch-n
    session, and each step all-gathers the two eps halves into the [2n] layout the fused step reads (dp.CFGExchange).
    Both ranks then run the same fused step on the same inputs, so they hold the same latents bit for bit; the initial
    latents are those of group rank 0."""
    do_cfg = guidance_scale > 1.0
    timesteps = [int(t) for t in scheduler.timesteps]
    n, _, h, w = latents.shape
    device = latents.device
    exchange = None
    if cfg_group is None:
        nb = 2 * n if do_cfg else n
        if do_cfg and adapter_state is not None:
            adapter_state = [torch.cat([v] * 2, dim=0) for v in adapter_state]
    else:
        nb = n
        exchange = dp.CFGExchange(cfg_group, tuple(latents.shape), device)
        exchange.broadcast(latents)
        half = slice(exchange.half * n, (exchange.half + 1) * n)
        prompt_embeds = prompt_embeds[half]
        if cross_attention_kwargs and 'region_list' in cross_attention_kwargs:
            cross_attention_kwargs = dict(cross_attention_kwargs, region_list=[
                (emb[half], box) for emb, box in cross_attention_kwargs['region_list']])
    x0_prev = torch.zeros_like(latents)
    sess = unet.session(nb, h, w, device, prompt_embeds, cross_attention_kwargs, adapter_state)
    unet_in = sess.latents_in
    unet_in.copy_(torch.cat([latents] * 2) if nb > n else latents)
    sess.t_in.fill_(float(timesteps[0]))
    for i, t in enumerate(timesteps):
        noise_pred = sess.step()
        t_next = float(timesteps[i + 1]) if i + 1 < len(timesteps) else 0.0
        coef = scheduler.coefficients(i)
        if exchange is None:
            # CFG combine + scheduler.step + cat([latents]*2) + next timestep, one kernel (reference :285-290, :273)
            ops.cfg_dpmpp_step(noise_pred, latents, x0_prev, unet_in.view(-1), cfg=do_cfg,
                               guidance=float(guidance_scale), coef=coef, t_out=sess.t_in, t_next=t_next)
        else:
            # the batch-n session takes one copy of the next input, the kernel would write two
            ops.cfg_dpmpp_step(exchange.all_gather(noise_pred), latents, x0_prev, None, cfg=True,
                               guidance=float(guidance_scale), coef=coef, t_out=sess.t_in, t_next=t_next)
            unet_in.copy_(latents)
        if controller is not None and hasattr(controller, 'step_callback'):
            new_latents = controller.step_callback(latents)
            if new_latents is not latents:      # a controller may return edited latents (reference :293-295)
                latents.copy_(new_latents.to(latents.dtype))
                unet_in.copy_(torch.cat([latents] * 2) if do_cfg else latents)
        if callback is not None and i % callback_steps == 0:
            callback(i, t, latents)
    return latents


class _GPUPipeline:
    """What both pipelines share: the components, `from_pretrained`'s loading and the denoise loop."""

    def __init__(self, vae=None, text_encoder=None, tokenizer=None, unet=None, scheduler=None):
        assert unet is not None, f'{type(self).__name__} needs the GPU UNet'
        self.vae, self.text_encoder, self.tokenizer, self.unet = vae, text_encoder, tokenizer, unet
        self.scheduler = scheduler if scheduler is not None else DPMSolverPP2M()
        # diffusers: 2 ** (len(vae.config.block_out_channels) - 1); 8 for SD1.5 (and when no VAE is attached)
        self.vae_scale_factor = 2 ** (len(vae.config.block_out_channels) - 1) if vae is not None else 8
        self.device = torch.device('cuda')

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, scheduler=None, vae=None, tokenizer=None, device='cuda',
                        **unused):
        """diffusers call shape (`EDLoRAPipeline.from_pretrained(path, scheduler=..., torch_dtype=...)`, test_edlora.py /
        README.md:146): loads `unet/` and `text_encoder/` of a diffusers-layout directory into the GPU containers
        (mixofshow/utils/model_io.py), `vae/` (when present) into the GPU VAE and `tokenizer/` through transformers."""
        import os
        from mixofshow.utils import model_io
        unet = model_io.load_unet(pretrained_model_name_or_path)
        text_encoder = model_io.load_text_encoder(pretrained_model_name_or_path, device=device)
        if vae is None and os.path.isdir(os.path.join(pretrained_model_name_or_path, 'vae')):
            vae = model_io.load_vae(pretrained_model_name_or_path, device=device)
        if tokenizer is None:
            from transformers import CLIPTokenizer
            tokenizer = CLIPTokenizer.from_pretrained(pretrained_model_name_or_path, subfolder='tokenizer')
        pipe = cls(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, unet=unet, scheduler=scheduler)
        pipe._loaded_from(pretrained_model_name_or_path)
        return pipe.to(device)

    def _loaded_from(self, path):
        """after `from_pretrained` has loaded the components (EDLoRAPipeline reads a fused model's concept config)"""

    def to(self, device):
        self.device = torch.device(device)
        return self

    @staticmethod
    def _batch_size(prompt, prompt_embeds):
        if prompt is not None and isinstance(prompt, str):
            return 1
        if prompt is not None and isinstance(prompt, list):
            return len(prompt)
        return prompt_embeds.shape[0]

    def _uncond_tokens(self, prompt, negative_prompt, batch_size):
        """reference :161-181 (diffusers' checks on negative_prompt)"""
        if negative_prompt is None:
            return [''] * batch_size
        if type(prompt) is not type(negative_prompt):
            raise TypeError(f'`negative_prompt` should be the same type to `prompt`, but got '
                            f'{type(negative_prompt)} != {type(prompt)}.')
        if isinstance(negative_prompt, str):
            return [negative_prompt]
        if batch_size != len(negative_prompt):
            raise ValueError(f'`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but '
                             f'`prompt`: {prompt} has batch size {batch_size}.')
        return negative_prompt

    def _denoise(self, prompt_embeds, batch_size, height, width, num_inference_steps, guidance_scale, generator, latents,
                 output_type, return_dict, callback, callback_steps, cross_attention_kwargs, cfg_group):
        """reference :262-322 from the timesteps to the decoded images; `prompt_embeds` carries the CFG halves"""
        device = self.device
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        shape = (batch_size, self.unet.in_channels, h, w)
        if latents is None:
            latents = torch.randn(shape, generator=generator, device=generator.device if generator is not None
                                  else 'cpu').to(device)
        latents = (latents.to(device, torch.float32) * self.scheduler.init_noise_sigma).contiguous()
        assert tuple(latents.shape) == shape, f'latents shape {tuple(latents.shape)} != {shape}'

        denoise_latents(self.unet, self.scheduler, latents, guidance_scale, prompt_embeds, cross_attention_kwargs,
                        controller=getattr(self, 'controller', None), callback=callback, callback_steps=callback_steps,
                        cfg_group=cfg_group)
        if output_type == 'latent':
            image = latents
        else:
            if self.vae is None:
                raise ValueError("no VAE supplied: use output_type='latent'")
            image = self.vae.decode(latents / 0.18215).sample
            image = (image / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).float().numpy()
            if output_type == 'pil':
                image = numpy_to_pil(image)
        if not return_dict:
            return (image)
        return SimpleNamespace(images=image, nsfw_content_detected=None)


class EDLoRAPipeline(_GPUPipeline):
    def __init__(self, vae=None, text_encoder=None, tokenizer=None, unet=None, scheduler=None, safety_checker=None,
                 feature_extractor=None, requires_safety_checker: bool = False):
        assert unet is not None, 'EDLoRAPipeline needs the GPU UNet'
        revise_edlora_unet_attention_forward(unet)          # reference :93
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler)
        self.new_concept_cfg = None

    def _loaded_from(self, pretrained_model_name_or_path):
        import os
        from mixofshow.utils import model_io
        if os.path.exists(os.path.join(pretrained_model_name_or_path, 'new_concept_cfg.json')):   # a fused model
            cfg = model_io.load_new_concept_cfg(pretrained_model_name_or_path)
            model_io.ensure_concept_tokens(self.tokenizer, cfg)
            self.set_new_concept_cfg(cfg)

    def set_new_concept_cfg(self, new_concept_cfg=None):
        self.new_concept_cfg = new_concept_cfg

    def set_controller(self, controller):
        self.controller = controller
        revise_edlora_unet_attention_controller_forward(self.unet, controller)

    # reference :111-190
    def _encode_prompt(self, prompt, new_concept_cfg, device, num_images_per_prompt, do_classifier_free_guidance,
                       negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None):
        assert num_images_per_prompt == 1, 'only support num_images_per_prompt=1 now'
        batch_size = self._batch_size(prompt, prompt_embeds)
        if prompt_embeds is None:
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError('no tokenizer / text_encoder supplied: pass prompt_embeds [B,16,77,768]')
            prompt_extend = bind_concept_prompt(prompt, new_concept_cfg)
            ids = self.tokenizer(prompt_extend, padding='max_length', max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors='pt').input_ids
            prompt_embeds = self.text_encoder(ids.to(device))[0]
            prompt_embeds = prompt_embeds.reshape(batch_size, -1, *prompt_embeds.shape[1:])   # '(b n) m c -> b n m c'
        prompt_embeds = prompt_embeds.to(device)
        bs_embed, layer_num, seq_len, _ = prompt_embeds.shape
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError('classifier-free guidance needs negative_prompt_embeds [B,77,768] when no text '
                                 'encoder is supplied')
            uncond_tokens = self._uncond_tokens(prompt, negative_prompt, batch_size)
            ids = self.tokenizer(uncond_tokens, padding='max_length', max_length=seq_len, truncation=True,
                                 return_tensors='pt').input_ids
            negative_prompt_embeds = self.text_encoder(ids.to(device))[0]
        if do_classifier_free_guidance:
            seq_len = negative_prompt_embeds.shape[1]
            negative_prompt_embeds = negative_prompt_embeds.to(device)
            negative_prompt_embeds = negative_prompt_embeds.view(batch_size, 1, seq_len, -1).repeat(1, layer_num, 1, 1)
            prompt_embeds = torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 50, guidance_scale: float = 7.5,
                 negative_prompt=None, num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = 'pil',
                 return_dict: bool = True, callback=None, callback_steps: int = 1, cross_attention_kwargs=None,
                 cfg_group=None):
        """`cfg_group`: a torch.distributed group of two ranks that sample this one call together, rank 0 the uncond
        and rank 1 the cond half of every UNet call (`denoise_latents`); both return the same images."""
        dp.check_cfg_group(cfg_group, guidance_scale, getattr(self, 'controller', None))
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f'`height` and `width` have to be divisible by 8 but are {height} and {width}.')
        batch_size = self._batch_size(prompt, prompt_embeds)
        device = self.device
        do_cfg = guidance_scale > 1.0
        assert self.new_concept_cfg is not None
        prompt_embeds = self._encode_prompt(prompt, self.new_concept_cfg, device, num_images_per_prompt, do_cfg,
                                            negative_prompt, prompt_embeds=prompt_embeds,
                                            negative_prompt_embeds=negative_prompt_embeds)
        return self._denoise(prompt_embeds, batch_size, height, width, num_inference_steps, guidance_scale, generator,
                             latents, output_type, return_dict, callback, callback_steps, cross_attention_kwargs,
                             cfg_group)


class StableDiffusionPipeline(_GPUPipeline):
    """diffusers' StableDiffusionPipeline on the GPU engines, the sampler of vanilla LoRA: `from_pretrained` and `__call__`
    with EDLoRAPipeline's arguments; prompts are tokenized as written (no binding), CLIP runs once per prompt, and
    `prompt_embeds` / `negative_prompt_embeds` are [B, 77, 768].  The UNet keeps its default attention processors and
    reads that one embedding in all 16 cross-attention layers.  As in diffusers there is no `set_new_concept_cfg`: the
    concept tokens `<new{k}>` that `convert_edlora(pipe, ckpt, enable_edlora=False, alpha)` adds go into the prompt
    literally."""

    def __init__(self, vae=None, text_encoder=None, tokenizer=None, unet=None, scheduler=None, safety_checker=None,
                 feature_extractor=None, requires_safety_checker: bool = False):
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler)

    def _encode_prompt(self, prompt, device, num_images_per_prompt, do_classifier_free_guidance, negative_prompt=None,
                       prompt_embeds=None, negative_prompt_embeds=None):
        """diffusers StableDiffusionPipeline._encode_prompt: [uncond; cond] [2B, 77, 768] with CFG, [B, 77, 768] without"""
        assert num_images_per_prompt == 1, 'only support num_images_per_prompt=1 now'
        batch_size = self._batch_size(prompt, prompt_embeds)
        if prompt_embeds is None:
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError('no tokenizer / text_encoder supplied: pass prompt_embeds [B,77,768]')
            prompts = [prompt] if isinstance(prompt, str) else list(prompt)
            ids = self.tokenizer(prompts, padding='max_length', max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors='pt').input_ids
            prompt_embeds = self.text_encoder(ids.to(device))[0]
        prompt_embeds = prompt_embeds.to(device)
        if prompt_embeds.ndim != 3:
            raise ValueError(f'prompt_embeds must be [B, 77, 768], got {tuple(prompt_embeds.shape)}')
        if not do_classifier_free_guidance:
            return prompt_embeds
        if negative_prompt_embeds is None:
            if self.tokenizer is None or self.text_encoder is None:
                raise ValueError('classifier-free guidance needs negative_prompt_embeds [B,77,768] when no text '
                                 'encoder is supplied')
            uncond_tokens = self._uncond_tokens(prompt, negative_prompt, batch_size)
            ids = self.tokenizer(uncond_tokens, padding='max_length', max_length=prompt_embeds.shape[1], truncation=True,
                                 return_tensors='pt').input_ids
            negative_prompt_embeds = self.text_encoder(ids.to(device))[0]
        negative_prompt_embeds = negative_prompt_embeds.to(device).reshape(prompt_embeds.shape)
        return torch.cat([negative_prompt_embeds, prompt_embeds])

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 50, guidance_scale: float = 7.5,
                 negative_prompt=None, num_images_per_prompt: Optional[int] = 1, eta: float = 0.0, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, output_type: Optional[str] = 'pil',
                 return_dict: bool = True, callback=None, callback_steps: int = 1, cross_attention_kwargs=None,
                 cfg_group=None):
        """`cfg_group`: a torch.distributed group of two ranks that sample this one call together, rank 0 the uncond
        and rank 1 the cond half of every UNet call (`denoise_latents`); both return the same images."""
        dp.check_cfg_group(cfg_group, guidance_scale, getattr(self, 'controller', None))
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f'`height` and `width` have to be divisible by 8 but are {height} and {width}.')
        batch_size = self._batch_size(prompt, prompt_embeds)
        prompt_embeds = self._encode_prompt(prompt, self.device, num_images_per_prompt, guidance_scale > 1.0,
                                            negative_prompt, prompt_embeds=prompt_embeds,
                                            negative_prompt_embeds=negative_prompt_embeds)
        return self._denoise(prompt_embeds, batch_size, height, width, num_inference_steps, guidance_scale, generator,
                             latents, output_type, return_dict, callback, callback_steps, cross_attention_kwargs,
                             cfg_group)
