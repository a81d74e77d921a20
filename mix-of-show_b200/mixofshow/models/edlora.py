"""Drop-in for the reference's `mixofshow/models/edlora.py` (same names, argument meaning and error behaviour), with
the arithmetic executed by hand-written sm_90a kernels (libmos_sm100.so) instead of diffusers / xformers / cuBLAS.

  LoRALinearLayer                                   <- mixofshow/models/edlora.py:221-246
  EDLoRA_AttnProcessor                              <- :103-173
  EDLoRA_Control_AttnProcessor                      <- :22-100
  revise_edlora_unet_attention_forward              <- :176-190
  revise_edlora_unet_attention_controller_forward   <- :193-218
  remove_edlora_unet_attention_forward              <- :12-19

Two ways these objects are used:
  * operator level (exactly the reference protocol): `processor(attn, hidden_states, encoder_hidden_states=...)`
    and `module(x)` on a LoRA-patched module run the fused CUDA kernels on the tensors they are given;
  * whole-UNet level: the GPU UNet (`mixofshow.models.unet_b200.UNet2DConditionModel`) reads them as descriptors
    (which layer index, which controller, which LoRA pairs) and configures the captured denoise step.
"""
import math

import torch
import torch.nn as nn

from mos_b200 import functional as Fm


class AttnProcessor:
    """Default processor (plain attention, no layer-wise embedding pick) — what diffusers' AttnProcessor does."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        assert attention_mask is None, 'attention masks are not used by the ED-LoRA path'
        out, _ = Fm.attention_block(attn, hidden_states, encoder_hidden_states)
        return out


def remove_edlora_unet_attention_forward(unet):
    def change_forward(unet):
        for name, layer in unet.named_children():
            if layer.__class__.__name__ == 'Attention' and name == 'attn2':
                layer.set_processor(AttnProcessor())
            else:
                change_forward(layer)
    change_forward(unet)


def _prologue(attn, hidden_states, temb):
    """Shared shape handling of both processors (edlora.py:40-66 / 116-137)."""
    if getattr(attn, 'spatial_norm', None) is not None:
        raise ValueError('spatial_norm is not used by SD1.5 attention and is not supported')
    input_ndim = hidden_states.ndim
    shape4 = None
    if input_ndim == 4:
        batch_size, channel, height, width = hidden_states.shape
        shape4 = (batch_size, channel, height, width)
        hidden_states = hidden_states.view(batch_size, channel, height * width).transpose(1, 2)
    assert not getattr(attn, 'norm_cross', None)
    if getattr(attn, 'group_norm', None) is not None:
        raise ValueError('attn.group_norm is not used by SD1.5 attention and is not supported')
    return hidden_states, shape4


def _epilogue(attn, hidden_states, residual, shape4):
    if shape4 is not None:
        b, c, h, w = shape4
        hidden_states = hidden_states.transpose(-1, -2).reshape(b, c, h, w)
    if getattr(attn, 'residual_connection', False):
        hidden_states = hidden_states + residual
    f = getattr(attn, 'rescale_output_factor', 1.0)
    if f != 1.0:
        hidden_states = hidden_states / f
    return hidden_states


class EDLoRA_Control_AttnProcessor:
    r"""Cross-attention with the layer-wise embedding pick and an attention controller that sees the probability
    maps `[B*heads, N, 77]` (fp32, emitted by the flash kernel next to the output)."""

    def __init__(self, cross_attention_idx, place_in_unet, controller, attention_op=None):
        self.cross_attention_idx = cross_attention_idx
        self.place_in_unet = place_in_unet
        self.controller = controller
        self.attention_op = attention_op

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        residual = hidden_states
        hidden_states, shape4 = _prologue(attn, hidden_states, temb)
        if encoder_hidden_states is None:
            is_cross = False
        else:
            is_cross = True
            if len(encoder_hidden_states.shape) == 4:  # multi-layer embedding
                encoder_hidden_states = encoder_hidden_states[:, self.cross_attention_idx, ...]
        assert attention_mask is None, 'attention masks are not used by the ED-LoRA path'
        # the reference calls the controller for every layer that does not take the xformers branch; with
        # xformers installed that is cross-attention only (edlora.py:77-83) — which is the behaviour kept here.
        out, probs = Fm.attention_block(attn, hidden_states, encoder_hidden_states, want_probs=is_cross)
        if is_cross:
            ret = self.controller(probs, is_cross, self.place_in_unet)
            if ret is not probs and not torch.equal(ret, probs):
                raise NotImplementedError('controllers that edit the attention probabilities are not supported')
        return _epilogue(attn, out, residual, shape4)


class EDLoRA_AttnProcessor:
    def __init__(self, cross_attention_idx, attention_op=None):
        self.attention_op = attention_op
        self.cross_attention_idx = cross_attention_idx

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None):
        residual = hidden_states
        hidden_states, shape4 = _prologue(attn, hidden_states, temb)
        if encoder_hidden_states is not None and len(encoder_hidden_states.shape) == 4:  # multi-layer embedding
            encoder_hidden_states = encoder_hidden_states[:, self.cross_attention_idx, ...]
        assert attention_mask is None, 'attention masks are not used by the ED-LoRA path'
        out, _ = Fm.attention_block(attn, hidden_states, encoder_hidden_states)
        return _epilogue(attn, out, residual, shape4)


def revise_edlora_unet_attention_forward(unet):
    def change_forward(unet, count):
        for name, layer in unet.named_children():
            if layer.__class__.__name__ == 'Attention' and 'attn2' in name:
                layer.set_processor(EDLoRA_AttnProcessor(count))
                count += 1
            else:
                count = change_forward(layer, count)
        return count

    # use this to ensure the order
    cross_attention_idx = change_forward(unet.down_blocks, 0)
    cross_attention_idx = change_forward(unet.mid_block, cross_attention_idx)
    cross_attention_idx = change_forward(unet.up_blocks, cross_attention_idx)
    print(f'Number of attention layer registered {cross_attention_idx}')


def revise_edlora_unet_attention_controller_forward(unet, controller):
    class DummyController:
        def __call__(self, *args):
            return args[0]

        def __init__(self):
            self.num_att_layers = 0

    if controller is None:
        controller = DummyController()

    def change_forward(unet, count, place_in_unet):
        for name, layer in unet.named_children():
            if layer.__class__.__name__ == 'Attention' and 'attn2' in name:  # only cross-attention gets a controller
                layer.set_processor(EDLoRA_Control_AttnProcessor(count, place_in_unet, controller))
                count += 1
            else:
                count = change_forward(layer, count, place_in_unet)
        return count

    cross_attention_idx = change_forward(unet.down_blocks, 0, 'down')
    cross_attention_idx = change_forward(unet.mid_block, cross_attention_idx, 'mid')
    cross_attention_idx = change_forward(unet.up_blocks, cross_attention_idx, 'up')
    print(f'Number of attention layer registered {cross_attention_idx}')
    controller.num_att_layers = cross_attention_idx


class LoRALinearLayer(nn.Module):
    """y = original(x) + alpha * up(down(x)) on a Linear or 1x1 Conv2d, installed by overwriting the module's
    forward exactly as the reference does; the forward is one fused wgmma GEMM (K1)."""

    def __init__(self, name, original_module, rank=4, alpha=1):
        super().__init__()
        self.name = name
        if rank > 4:
            raise ValueError('the fused sm_90a epilogue supports LoRA rank <= 4 (the reference default is 4)')
        if original_module.__class__.__name__ == 'Conv2d':
            in_channels, out_channels = original_module.in_channels, original_module.out_channels
            self.lora_down = torch.nn.Conv2d(in_channels, rank, (1, 1), bias=False)
            self.lora_up = torch.nn.Conv2d(rank, out_channels, (1, 1), bias=False)
        else:
            in_features, out_features = original_module.in_features, original_module.out_features
            self.lora_down = nn.Linear(in_features, rank, bias=False)
            self.lora_up = nn.Linear(rank, out_features, bias=False)
        self.register_buffer('alpha', torch.tensor(alpha))
        torch.nn.init.kaiming_uniform_(self.lora_down.weight, a=math.sqrt(5))
        torch.nn.init.zeros_(self.lora_up.weight)
        object.__setattr__(self, '_orig', original_module)   # not a submodule: parameters stay where they are
        object.__setattr__(original_module, '_mos_lora', self)   # descriptor read by the packers (not a child module)
        self.original_forward = original_module.forward
        original_module.forward = self.forward

    def forward(self, hidden_states):
        return Fm.lora_linear(self._orig, hidden_states)
