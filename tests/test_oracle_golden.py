"""CPU: the oracle restatement against the committed golden fixtures, which were produced by the
REFERENCE's own modules (oracle/gen_golden.py).  No GPU, no reference checkout needed."""
from pathlib import Path

import torch
import torch.nn.functional as F

from oracle import vila_oracle as O

G = Path(__file__).resolve().parent / "golden"


def test_siglip_tower_matches_reference_fixture():
    fx = torch.load(G / "siglip_tiny.pt")
    cfg = O.SiglipCfg(**fx["cfg"])
    assert fx["n_hidden_states"] == cfg.num_hidden_layers + 1
    got = O.siglip_tower(fx["pixels"], fx["weights"], cfg, -2)
    assert (got - fx["hidden_m2"]).abs().max().item() < 2e-5
    got_last = O.siglip_tower(fx["pixels"], fx["weights"], cfg, -1)
    assert (got_last - fx["hidden_m1"]).abs().max().item() < 2e-5
    assert (got - got_last).abs().max().item() > 1e-3  # -2 really is a different tensor than -1


def test_projector_matches_reference_fixture():
    fx = torch.load(G / "projector.pt")
    for kind, d in fx.items():
        got = O.projector(d["x"], d["weights"], kind)
        assert got.shape == d["y"].shape
        assert (got - d["y"]).abs().max().item() < 1e-5, kind


def test_dynamic_s2_encode_images_matches_reference_fixture():
    fx = torch.load(G / "arch_glue.pt")
    proj = lambda f: F.linear(O.downsample(f, 2), fx["lin_w"], fx["lin_b"])
    for case in fx["s2"]:
        got = O.encode_images(case["feats"], lambda x: x, proj, dynamic_s2=True,
                              block_sizes=case["block_sizes"], scales=[4, 8, 12],
                              resize_output_to_scale_idx=case["idx"])
        assert len(got) == len(case["out"])
        for a, b in zip(got, case["out"]):
            assert a.shape == b.shape and (a - b).abs().max().item() < 1e-6


def test_embed_splice_matches_reference_fixture():
    fx = torch.load(G / "arch_glue.pt")["embed"]
    for side in ("right", "left"):
        a, b, c = O.embed_splice(fx["ids"], fx["table"], {"image": list(fx["m_img"]), "video": list(fx["m_vid"])},
                                 {"image": fx["IMG"], "video": fx["VID"]}, None, fx["mask"], side)
        w = fx["out"][side]
        assert torch.equal(a, w["inputs"]) and torch.equal(b, w["labels"]) and torch.equal(c, w["mask"])
    # unconsumed media must raise like the reference (llava_arch.py:484)
    import pytest
    with pytest.raises(ValueError):
        O.embed_splice(fx["ids"][:, :2], fx["table"], {"image": list(fx["m_img"])}, {"image": fx["IMG"]})


def test_qwen2_matches_transformers_fixture():
    fx = torch.load(G / "qwen2_tiny.pt")
    cfg = O.Qwen2Cfg(head_dim=fx["cfg"]["hidden_size"] // fx["cfg"]["num_attention_heads"], **fx["cfg"])
    logits, _ = O.qwen2_forward(fx["emb"][0], fx["weights"], cfg)
    assert (logits - fx["logits"]).abs().max().item() < 5e-5
    far, _ = O.qwen2_forward(fx["emb"][0], fx["weights"], cfg, position_ids=fx["pos_far"])
    assert (far - fx["logits_far"]).abs().max().item() < 5e-5
    ids, _ = O.greedy_generate(fx["emb"][0], fx["weights"], cfg, 10)
    assert ids == fx["greedy"]


def test_kv_cached_decode_equals_full_forward():
    fx = torch.load(G / "qwen2_tiny.pt")
    cfg = O.Qwen2Cfg(head_dim=16, **fx["cfg"])
    emb = fx["emb"][0]
    full, _ = O.qwen2_forward(emb, fx["weights"], cfg)
    _, past = O.qwen2_forward(emb[:15], fx["weights"], cfg)
    for t in range(15, 21):
        step, past = O.qwen2_forward(emb[t:t + 1], fx["weights"], cfg, past=past)
    assert (step[0] - full[-1]).abs().max().item() < 1e-4


def test_flat_square_edge_cases():
    x = torch.arange(2 * 3 * 5 * 2, dtype=torch.float32).view(2, 3, 5, 2)
    y = O.flat_square(x, 2)
    assert y.shape == (2, 2, 3, 8)
    # out[n, i, j, (q*2+p)*c + ch] = x[n, 2i+q, 2j+p, ch], zero beyond the border
    assert torch.equal(y[0, 0, 0], torch.cat([x[0, 0, 0], x[0, 0, 1], x[0, 1, 0], x[0, 1, 1]]))
    assert y[0, 1, 2, 2:].abs().sum() == 0 and torch.equal(y[0, 1, 2, :2], x[0, 2, 4])
    assert O.flat_square(torch.zeros(1, 4, 4, 2), 3).shape == (1, 2, 2, 18)


def test_oracle_attention_blocking_does_not_change_results():
    """the head / query-row blocking of the oracle's attention (a memory bound for 16K-66K token
    sequences) computes the same function: tiny budgets give the same logits up to fp32 BLAS summation
    order (1e-5), with and without a cache"""
    d = torch.load(G / "qwen2_tiny.pt")
    cfg = O.Qwen2Cfg(head_dim=16, **d["cfg"])
    p = d["weights"]
    emb = d["emb"][0]
    want, past = O.qwen2_forward(emb, p, cfg)
    step, _ = O.qwen2_forward(emb[-3:], p, cfg, past=[(k[:, :-3], v[:, :-3]) for k, v in past])
    old = O.SCORE_BUDGET
    try:
        for budget in (1, 7 * emb.shape[0], 3 * emb.shape[0] * emb.shape[0]):
            O.SCORE_BUDGET = budget
            got, _ = O.qwen2_forward(emb, p, cfg)
            assert (got - want).abs().max().item() < 1e-5, budget
            got2, _ = O.qwen2_forward(emb[-3:], p, cfg, past=[(k[:, :-3], v[:, :-3]) for k, v in past])
            assert (got2 - step).abs().max().item() < 1e-5, budget
    finally:
        O.SCORE_BUDGET = old
