"""VILAForCausalLM — the HF-Hub-facing twin of LlavaLlamaModel (SURVEY §8 f1).

Reference: llava/remote_code/modeling_vila.py — `VILAForCausalLM` (:506), `forward` (:1024-1086, the
extra `pixel_values` argument), `generate` (:1089-1125: returns `input_ids ++ output_ids` unless
`return_output_ids_only`), `generate_content` (:1128-1244), `default_generation_config` (:1246-1258:
eos_token_id is the tokenizer's single id here, not `stop_token_ids`).  Released NVILA checkpoints
load through this class (`AutoModel.from_pretrained(..., trust_remote_code=True)`); here it is the
same module tree and the same sm_90a ops as LlavaLlamaModel, with the remote-code call semantics.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from .llava_llama import LlavaLlamaModel


class VILAForCausalLM(LlavaLlamaModel):
    def forward(self, input_ids=None, media=None, images=None, media_config=None, pixel_values=None,
                attention_mask=None, position_ids=None, past_key_values=None, inputs_embeds=None,
                labels=None, packing: bool = True, force_packing: bool = False, seqlens_in_batch=None,
                dpo_forward: bool = False, **kwargs):
        """modeling_vila.py:1024-1086 (pixel_values is accepted and unused there as well)."""
        return super().forward(input_ids=input_ids, media=media, images=images, media_config=media_config,
                               attention_mask=attention_mask, position_ids=position_ids,
                               past_key_values=past_key_values, inputs_embeds=inputs_embeds, labels=labels,
                               packing=packing, force_packing=force_packing,
                               seqlens_in_batch=seqlens_in_batch, dpo_forward=dpo_forward, **kwargs)

    __call__ = forward

    @torch.inference_mode()
    def generate(self, input_ids=None, media: Optional[Dict[str, List[torch.Tensor]]] = None,
                 media_config: Dict[str, Dict[str, Any]] = None, attention_mask=None,
                 return_output_ids_only: bool = False, **generation_kwargs) -> torch.LongTensor:
        """modeling_vila.py:1089-1125: the prompt ids are PREPENDED to the new ids (community-VLM
        convention) unless return_output_ids_only; with a generation_config carrying
        num_return_sequences the prompt rows are repeated accordingly."""
        output_ids = super().generate(input_ids=input_ids, media=media, media_config=media_config,
                                      attention_mask=attention_mask, **generation_kwargs)
        if return_output_ids_only:
            return output_ids
        gc = generation_kwargs.get("generation_config", None)
        prompt = input_ids.to(output_ids.device)
        if gc is not None:
            n = getattr(gc, "num_return_sequences", 1) or 1
            prompt = prompt.repeat_interleave(n, dim=0)
        return torch.cat([prompt, output_ids], dim=-1)

    @property
    def default_generation_config(self):
        """modeling_vila.py:1246-1258: as LlavaLlamaModel's, but eos = tokenizer.eos_token_id."""
        gc = super().default_generation_config
        if self.generation_config is None or getattr(self.generation_config, "eos_token_id", None) is None:
            gc.eos_token_id = self.tokenizer.eos_token_id
        return gc

    # generate_content (modeling_vila.py:1128-1244) is inherited: it is the same code as llava_arch.py:835-948
    # (media extraction, response_format -> xgrammar logits processor, greedy retry after a sampling failure) and
    # decodes `output_ids[0]` of THIS class's generate — i.e. prompt + answer ids; media and special tokens are
    # skipped by the tokenizer.
