"""Sequence packing (training-time path, SURVEY §8 a14) — host-side index plumbing on torch tensors.

Reference:
  LlavaMetaForCausalLM.repack_multimodal_data, non-SP branch   llava/model/llava_arch.py:744-800
  _get_unpad_data / set_seqlens_in_batch                        llava/model/utils/packing.py:12-36
The reference packs a padded batch into ONE row, appends a dummy token (attention_mask 0) so that HF's
flash-attention wrapper takes its unpad path, and lets the patched `_get_unpad_data` hand flash-attn
`cu_seqlens` built from `seqlens_in_batch`: attention is block-diagonal causal, position ids restart
per sequence.  Here the packed row goes to Qwen2ForCausalLM.forward(seqlens_in_batch=...), which runs
the GEMMs / norms once over all packed rows and the wgmma FMHA once per sequence segment.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn.functional as F

IGNORE_INDEX = -100


def repack_multimodal_data(inputs_embeds: torch.Tensor, attention_mask: torch.Tensor,
                           position_ids: Optional[torch.Tensor], labels: torch.Tensor,
                           pad_to_multiple_of: Optional[int] = None, pad_token_id: int = 0
                           ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """[B, L, H] padded batch -> ([1, T+1(+pad), H], mask [1, ..] int32, position_ids [1, ..] int32,
    labels [1, ..]) with T = sum of the sequence lengths.  Quirks kept from the reference: the dummy
    token at the end (mask 0, label IGNORE), the first label of every sequence masked to IGNORE, int32
    masks / positions, `pad_to_multiple_of` padding with position -1 and `pad_token_id`-valued rows."""
    device = inputs_embeds.device
    bsz = inputs_embeds.shape[0]
    mask = attention_mask.to(torch.bool)
    seqlens = [int(mask[k].sum()) for k in range(bsz)]
    emb_p = [inputs_embeds[k][mask[k]] for k in range(bsz)]
    mask_p = [torch.ones(n, dtype=torch.int, device=device) for n in seqlens]
    pos_p = [torch.arange(n, dtype=torch.int, device=device) for n in seqlens]
    lab_p = [labels[k][mask[k]].clone() for k in range(bsz)]
    emb_p.append(torch.zeros(1, inputs_embeds.shape[-1], dtype=inputs_embeds.dtype, device=device))
    mask_p.append(torch.tensor([0], dtype=torch.int, device=device))
    pos_p.append(torch.tensor([0], dtype=torch.int, device=device))
    lab_p.append(torch.tensor([IGNORE_INDEX], dtype=torch.int, device=device))
    for lab in lab_p:
        if lab.numel():
            lab[0] = IGNORE_INDEX
    emb = torch.cat(emb_p, dim=0).unsqueeze(0)
    am = torch.cat(mask_p, dim=0).unsqueeze(0)
    pos = torch.cat(pos_p, dim=0).unsqueeze(0)
    lab = torch.cat([l.to(lab_p[0].dtype) for l in lab_p], dim=0).unsqueeze(0)
    if pad_to_multiple_of:
        cur = lab.shape[1]
        if cur % pad_to_multiple_of != 0:
            tgt = (cur // pad_to_multiple_of + 1) * pad_to_multiple_of
            d = tgt - cur
            emb = torch.cat((emb, torch.full((1, d, emb.shape[-1]), pad_token_id).to(emb)), dim=1)
            lab = torch.cat((lab, torch.full((1, d), IGNORE_INDEX).to(lab)), dim=1)
            am = torch.cat((am, torch.zeros((1, d), dtype=torch.bool).to(am)), dim=1)
            pos = torch.cat((pos, torch.full((1, d), -1).to(pos)), dim=1)
    return emb, am, pos, lab


def get_unpad_data(attention_mask: torch.Tensor, seqlens_in_batch: Optional[torch.Tensor] = None
                   ) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """packing._get_unpad_data: (indices of real tokens, cu_seqlens int32 [n+1], max_seqlen)."""
    if seqlens_in_batch is None:
        seqlens_in_batch = torch.sum(attention_mask, dim=1)
    indices = torch.nonzero(attention_mask.flatten(), as_tuple=False).flatten()
    max_seqlen = int(seqlens_in_batch.max())
    cu = F.pad(torch.cumsum(seqlens_in_batch, dim=0, dtype=torch.int32), (1, 0))
    return indices, cu, max_seqlen
