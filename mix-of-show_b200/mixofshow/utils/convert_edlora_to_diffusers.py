"""Drop-in for the reference's `mixofshow/utils/convert_edlora_to_diffusers.py` (on-disk / checkpoint plumbing, SURVEY.md
§8f rank 3): loading an ED-LoRA delta checkpoint (`{'params': {'new_concept_embedding', 'text_encoder', 'unet'}}`,
written at train_edlora.py:168-171 from trainer_edlora.py:358-378) into a pipeline — new concept tokens and embedding
rows, LoRA folded into the UNet and text-encoder weights.  Pure host logic; works on the reference's diffusers objects
and on this repo's `UNet2DConditionModel` / `CLIPTextModel` containers alike (they expose the same `state_dict` /
`load_state_dict` / `get_input_embeddings` / `resize_token_embeddings` surface)."""
import copy

LORA_LEAVES = {
    'text_encoder': ('q_proj', 'k_proj', 'v_proj', 'out_proj', 'fc1', 'fc2'),
    'unet': ('to_q', 'to_k', 'to_v', 'to_out.0', 'ff.net.0.proj', 'ff.net.2', 'proj_out', 'proj_in'),
}


def load_new_concept(pipe, new_concept_embedding, enable_edlora=True):
    """reference :4-31.  Adds 16 tokens `<new{idx*16 + layer}>` per concept (1 without ED-LoRA), resizes the embedding
    table and writes the learned rows; returns (pipe, new_concept_cfg)."""
    new_concept_cfg = {}
    for idx, (concept_name, concept_embedding) in enumerate(new_concept_embedding.items()):
        num_new_embedding = 16 if enable_edlora else 1
        new_token_names = [f'<new{idx * num_new_embedding + layer_id}>' for layer_id in range(num_new_embedding)]
        num_added_tokens = pipe.tokenizer.add_tokens(new_token_names)
        assert num_added_tokens == len(new_token_names), 'some token is already in tokenizer'
        new_token_ids = [pipe.tokenizer.convert_tokens_to_ids(token_name) for token_name in new_token_names]
        pipe.text_encoder.resize_token_embeddings(len(pipe.tokenizer))
        token_embeds = pipe.text_encoder.get_input_embeddings().weight.data
        token_embeds[new_token_ids] = concept_embedding.clone().to(token_embeds.device, dtype=token_embeds.dtype)
        new_concept_cfg.update({concept_name: {'concept_token_ids': new_token_ids,
                                               'concept_token_names': new_token_names}})
    return pipe, new_concept_cfg


def lora_down_name(weight_name, model_type):
    """reference :34-51: '<module>.weight' -> '<module>.lora_down.weight' for the module leaves that may carry a LoRA."""
    name = weight_name
    for leaf in LORA_LEAVES[model_type]:
        name = name.replace(f'{leaf}.weight', f'{leaf}.lora_down.weight')
    return name


def merge_lora_into_weight(original_state_dict, lora_state_dict, model_type, alpha):
    """reference :33-76: W' = W + alpha * up @ down (1x1 conv weights via squeeze / unsqueeze) for every weight that has
    a LoRA pair in `lora_state_dict`; everything else is copied."""
    assert model_type in ['unet', 'text_encoder']
    new_state_dict = copy.deepcopy(original_state_dict)
    load_cnt = 0
    for k in new_state_dict.keys():
        down_name = lora_down_name(k, model_type)
        up_name = down_name.replace('lora_down', 'lora_up')
        if up_name in lora_state_dict:
            load_cnt += 1
            original_params = new_state_dict[k]
            down = lora_state_dict[down_name].to(original_params.device)
            up = lora_state_dict[up_name].to(original_params.device)
            if len(original_params.shape) == 4:
                # flatten, not the reference's squeeze: at rank 1 squeeze also drops the rank dimension, and up @ down
                # becomes the dot product of two vectors added to every element of the weight
                lora_param = (up.flatten(1) @ down.flatten(1)).unsqueeze(-1).unsqueeze(-1)
            else:
                lora_param = up @ down
            new_state_dict[k] = original_params + alpha * lora_param
    print(f'load {load_cnt} LoRAs of {model_type}')
    return new_state_dict


def convert_edlora(pipe, state_dict, enable_edlora, alpha=0.6):
    """reference :79-99."""
    state_dict = state_dict['params'] if 'params' in state_dict.keys() else state_dict
    new_concept_cfg = {}
    if 'new_concept_embedding' in state_dict and len(state_dict['new_concept_embedding']) != 0:
        pipe, new_concept_cfg = load_new_concept(pipe, state_dict['new_concept_embedding'], enable_edlora)
    unet_lora_state_dict = state_dict['unet']
    pretrained_unet_state_dict = pipe.unet.state_dict()
    updated_unet_state_dict = merge_lora_into_weight(pretrained_unet_state_dict, unet_lora_state_dict, model_type='unet',
                                                     alpha=alpha)
    pipe.unet.load_state_dict(updated_unet_state_dict)
    text_encoder_lora_state_dict = state_dict['text_encoder']
    pretrained_text_encoder_state_dict = pipe.text_encoder.state_dict()
    updated_text_encoder_state_dict = merge_lora_into_weight(pretrained_text_encoder_state_dict, text_encoder_lora_state_dict,
                                                             model_type='text_encoder', alpha=alpha)
    pipe.text_encoder.load_state_dict(updated_text_encoder_state_dict)
    return pipe, new_concept_cfg
