"""End-to-end parity (GPU): vila_b200.model.LlavaLlamaModel through its public API against the CPU
oracle on identical random-init weights and synthetic inputs.  Tolerance model: tests/helpers.py
(check_close): CUDA error vs fp32 truth <= 2x the reference's own bf16 error + 1e-3 relative;
greedy ids exact up to the first bf16-level tie."""
import pytest
import torch

from tests.helpers import check_close, greedy_ids_match, oracle_from_state_dict

pytestmark = pytest.mark.gpu


def build(cfg, seed=0):
    from vila_b200.model import LlavaLlamaModel
    return LlavaLlamaModel(cfg, device="cuda").init_random(seed)


def synth_inputs(cfg, n_images=1, n_text=9, seed=1):
    g = torch.Generator().manual_seed(seed)
    S = cfg.vision_tower_cfg.image_size
    images = [torch.randn(3, S, S, generator=g).to(torch.bfloat16) for _ in range(n_images)]
    ids = torch.randint(3, 900, (n_text,), generator=g).tolist()
    for k in range(n_images):
        ids.insert(2 + 3 * k, cfg.image_token_id)
    return torch.tensor([ids]), images


@pytest.mark.parametrize("projector", ["mlp_downsample", "mlp_downsample_2x2_fix", "mlp_downsample_3x3_fix"])
def test_forward_logits_match_oracle(cuda, projector):
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(projector=projector)
    model = build(cfg)
    ids, images = synth_inputs(cfg, n_images=2)
    out = model(input_ids=ids, media={"image": [im.cuda() for im in images]})
    sd = model.state_dict()
    truth = oracle_from_state_dict(sd, cfg, torch.float32).forward_logits(
        ids, [im.float() for im in images])
    lowp = oracle_from_state_dict(sd, cfg, torch.bfloat16).forward_logits(ids, images)
    assert out.logits.shape[1] == truth.shape[0]
    check_close(f"logits[{projector}]", out.logits[0], truth, lowp)


def test_vision_tower_and_projector_stages(cuda):
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(vis_layers=4)
    model = build(cfg, seed=3)
    _, images = synth_inputs(cfg, n_images=3)
    px = torch.stack(images).cuda()
    sd = model.state_dict()
    o32 = oracle_from_state_dict(sd, cfg, torch.float32)
    o16 = oracle_from_state_dict(sd, cfg, torch.bfloat16)
    feats = model.vision_tower(px)
    t32 = o32.tower(torch.stack(images).float())
    check_close("vision_tower", feats, t32, o16.tower(torch.stack(images)))
    enc = model.encode_images(px)
    check_close("encode_images", enc, o32.project(t32), o16.encode_images(torch.stack(images)))
    # list input and fp16 input (reference calls .half() on pixels, llava_arch.py:864)
    lst = model.vision_tower([im.cuda() for im in images])
    assert torch.equal(torch.stack(lst), feats)
    assert model.vision_tower(px.half()).dtype == torch.float16


@pytest.mark.parametrize("idx", [-1, 0])
def test_encode_images_dynamic_s2(cuda, idx):
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(dynamic_s2=True, image_size=56, s2_resize_output_to_scale_idx=idx)
    model = build(cfg, seed=4)
    g = torch.Generator().manual_seed(5)
    block_sizes = [(2, 3), None, (1, 2)]
    n_tiles = (1 + 4 + 6) + 1 + (1 + 4 + 2)
    px = torch.randn(n_tiles, 3, 56, 56, generator=g).to(torch.bfloat16)
    got = model.encode_images(px.cuda(), block_sizes=block_sizes)
    sd = model.state_dict()
    t32 = oracle_from_state_dict(sd, cfg, torch.float32).encode_images(px.float(), block_sizes)
    t16 = oracle_from_state_dict(sd, cfg, torch.bfloat16).encode_images(px, block_sizes)
    assert len(got) == len(t32) == 3
    for i, (a, b, c) in enumerate(zip(got, t32, t16)):
        assert a.shape == b.shape
        check_close(f"dynamic_s2 image {i}", a, b, c)


def test_generate_greedy_matches_oracle(cuda):
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(llm_layers=3)
    model = build(cfg, seed=6)
    ids, images = synth_inputs(cfg, n_images=1, n_text=12)
    out = model.generate(input_ids=ids, media={"image": [images[0].cuda()]}, max_new_tokens=24,
                         eos_token_id=None)
    assert out.shape == (1, 24) and out.dtype == torch.long
    oracle = oracle_from_state_dict(model.state_dict(), cfg, torch.float32)
    want, logits = oracle.generate(ids, [images[0].float()], 24)
    # margin: 3 bf16 ulps at the logit scale
    margin = 3 * 2 ** -8 * logits.abs().max().item()
    greedy_ids_match(out[0].tolist(), want, logits, margin)
    # eos handling: stop right after the first generated token when it is declared EOS
    first = int(out[0, 0])
    out2 = model.generate(input_ids=ids, media={"image": [images[0].cuda()]}, max_new_tokens=24,
                          eos_token_id=[first])
    assert out2.tolist() == [[first]]
    # second call reuses the captured CUDA graph and must reproduce the same ids
    out3 = model.generate(input_ids=ids, media={"image": [images[0].cuda()]}, max_new_tokens=24,
                          eos_token_id=None)
    assert torch.equal(out, out3)


def test_decode_logits_match_prefill(cuda):
    """Incremental prefill (prefill_hidden with Sq=1, token by token on the KV cache) must agree with
    one prefill of the whole sequence.  No decode kernel runs here: the decode engines are compared
    with the oracle step by step in test_decode_engines_gpu.py."""
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(llm_layers=2)
    model = build(cfg, seed=7)
    llm = model.llm
    g = torch.Generator(device="cuda").manual_seed(8)
    emb = (torch.randn(150, cfg.hidden_size, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    cache = llm.new_cache(256)
    hid = llm.prefill_hidden(emb[:140], cache)
    lg_a = None
    for t in range(140, 150):  # extend token by token through the prefill path with Sq=1
        hid = llm.prefill_hidden(emb[t:t + 1], cache)
    lg_a = llm.logits_from_hidden(hid[-1:])
    cache2 = llm.new_cache(256)
    hid2 = llm.prefill_hidden(emb, cache2)
    lg_b = llm.logits_from_hidden(hid2[-1:])
    check_close("incremental vs full prefill", lg_a, lg_b.float())


def test_batch_padding_and_video_encoders(cuda):
    from vila_b200.model import tiny_test_config
    from oracle import vila_oracle as O
    cfg = tiny_test_config(projector="mlp_downsample_2x2_fix", video_encoder="tsp",
                           tsp_pool_sizes=((4, 1, 1), (2, 2, 2)))
    model = build(cfg, seed=9)
    g = torch.Generator().manual_seed(10)
    S = cfg.vision_tower_cfg.image_size
    video = torch.randn(8, 3, S, S, generator=g).to(torch.bfloat16)
    image = torch.randn(3, S, S, generator=g).to(torch.bfloat16)
    ids = torch.tensor([[5, cfg.video_token_id, 6, 7, cfg.image_token_id, 8],
                        [9, 10, 11, cfg.pad_token_id, cfg.pad_token_id, cfg.pad_token_id]])
    mask = torch.tensor([[1, 1, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0]], dtype=torch.bool)
    emb, labels, amask = model._embed(ids, {"video": [video.cuda()], "image": [image.cuda()]},
                                      {"video": {}, "image": {}}, None, mask)
    sd = model.state_dict()
    o32 = oracle_from_state_dict(sd, cfg, torch.float32)
    feats_v = o32.encode_images(video.float())
    feats_i = o32.encode_images(image.float()[None])
    end = o32.llm["model.embed_tokens.weight"][list(cfg.newline_token_ids)]
    vid = O.tsp_video_encoder(feats_v, cfg.tsp_pool_sizes, end)
    img = O.image_encoder(list(feats_i), end)
    want, wlab, wmask = O.embed_splice(ids, o32.llm["model.embed_tokens.weight"],
                                       {"video": [vid], "image": img},
                                       {"image": cfg.image_token_id, "video": cfg.video_token_id},
                                       None, mask, "right")
    assert emb.shape == want.shape
    assert torch.equal(amask.cpu(), wmask) and torch.equal(labels.cpu(), wlab)
    check_close("_embed (video TSP + image, padded batch)", emb, want)
    # forward over the padded batch returns zeros on padded positions
    out = model(input_ids=ids, media={"video": [video.cuda()], "image": [image.cuda()]}, attention_mask=mask)
    assert out.logits.shape[:2] == want.shape[:2]
    assert out.logits[1, 3:].abs().max().item() == 0
    with pytest.raises(ValueError):
        model._embed(ids[:1, :1], {"image": [image.cuda()]}, {"image": {}}, None, None)


def test_save_load_roundtrip(cuda, tmp_path):
    from vila_b200.model import tiny_test_config
    from vila_b200.model.loading import load_pretrained, save_pretrained
    cfg = tiny_test_config()
    model = build(cfg, seed=11)
    save_pretrained(model, str(tmp_path / "ckpt"))
    again = load_pretrained(str(tmp_path / "ckpt"))
    a, b = model.state_dict(), again.state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    ids, images = synth_inputs(cfg)
    la = model(input_ids=ids, media={"image": [images[0].cuda()]}).logits
    lb = again(input_ids=ids, media={"image": [images[0].cuda()]}).logits
    assert torch.equal(la, lb)


def test_no_cpu_fallback(cuda):
    """The product path must fail loudly on CPU tensors instead of silently computing elsewhere."""
    from vila_b200 import ops
    with pytest.raises(RuntimeError):
        ops.linear(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


def test_force_packing_matches_unpacked_and_oracle(cuda):
    """a14: forward(force_packing=True) packs the padded batch into one row (+ dummy token) and runs
    block-diagonal causal attention; every packed row must carry the logits the same token gets in the
    ordinary padded-batch forward, and the oracle's per-sequence logits."""
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(llm_layers=2)
    model = build(cfg, seed=12)
    g = torch.Generator().manual_seed(13)
    S = cfg.vision_tower_cfg.image_size
    image = torch.randn(3, S, S, generator=g).to(torch.bfloat16)
    ids = torch.tensor([[5, cfg.image_token_id, 6, 7, 8, 9, 10],
                        [11, 12, 13, cfg.pad_token_id, cfg.pad_token_id, cfg.pad_token_id, cfg.pad_token_id],
                        [14, 15, 16, 17, 18, cfg.pad_token_id, cfg.pad_token_id]])
    mask = torch.tensor([[1] * 7, [1, 1, 1, 0, 0, 0, 0], [1, 1, 1, 1, 1, 0, 0]], dtype=torch.bool)
    labels = torch.randint(3, 900, ids.shape, generator=g)
    plain = model(input_ids=ids, media={"image": [image.cuda()]}, attention_mask=mask, labels=labels)
    packed = model(input_ids=ids, media={"image": [image.cuda()]}, attention_mask=mask, labels=labels,
                   force_packing=True)
    lens = [7 - 1 + 17, 3, 5]
    assert packed.logits.shape[:2] == (1, sum(lens) + 1)
    sd = model.state_dict()
    o32 = oracle_from_state_dict(sd, cfg, torch.float32)
    off = 0
    for k, n in enumerate(lens):
        a = packed.logits[0, off:off + n].float()
        b = plain.logits[k, :n].float()
        assert (a - b).abs().max().item() <= 2 ** -6 * max(1.0, b.abs().max().item()), k
        if k > 0:  # text-only rows: the oracle forward of that sequence alone
            emb = o32.llm["model.embed_tokens.weight"][ids[k, :n]]
            from oracle import vila_oracle as O
            truth, _ = O.qwen2_forward(emb, o32.llm, o32.lcfg)
            check_close(f"packed row {k} vs oracle", a, truth)
        off += n
    assert packed.loss is not None and torch.isfinite(packed.loss)
    # dpo_forward returns (logits, repacked labels) with the first label of every sequence masked
    lg, lab = model(input_ids=ids, media={"image": [image.cuda()]}, attention_mask=mask, labels=labels,
                    force_packing=True, dpo_forward=True)
    assert lab.shape == (1, sum(lens) + 1) and int(lab[0, 0]) == -100 and int(lab[0, lens[0]]) == -100


def test_remote_code_class_stream_and_cli(cuda, tmp_path, capsys):
    """f1 / f3 / config #1 plumbing on the GPU path: VILAForCausalLM.generate prepends the prompt ids;
    generate_content(stream=True) yields the same text in chunks; `llava.cli.infer` runs end to end on
    a checkpoint directory in the reference's three-folder layout."""
    import numpy as np
    from PIL import Image as PILImage
    from vila_b200.model import VILAForCausalLM, tiny_test_config
    from vila_b200.model.loading import save_pretrained
    cfg = tiny_test_config(projector="mlp_downsample_3x3_fix", image_aspect_ratio="dynamic", model_max_length=64)
    model = VILAForCausalLM(cfg, device="cuda").init_random(14)
    ids, images = synth_inputs(cfg, n_images=1, n_text=8)
    full = model.generate(input_ids=ids, media={"image": [images[0].cuda()]}, max_new_tokens=6, eos_token_id=None)
    only = model.generate(input_ids=ids, media={"image": [images[0].cuda()]}, max_new_tokens=6, eos_token_id=None,
                          return_output_ids_only=True)
    assert full.shape == (1, ids.shape[1] + 6) and torch.equal(full[:, :ids.shape[1]].cpu(), ids)
    assert torch.equal(full[:, ids.shape[1]:], only)
    from types import SimpleNamespace
    gc = SimpleNamespace(max_new_tokens=12, do_sample=False, eos_token_id=None, pad_token_id=0, max_length=None)
    img = PILImage.fromarray(np.random.RandomState(3).randint(0, 256, (336, 336, 3), dtype=np.uint8))
    p_ids, p_media, p_cfg = model._prepare_content([img, "Describe."])
    new_ids = model.generate(input_ids=p_ids, media=p_media, media_config=p_cfg, generation_config=gc,
                             return_output_ids_only=True)
    text = model.tokenizer.decode(new_ids[0], skip_special_tokens=True)
    chunks = list(model.generate_content([img, "Describe."], generation_config=gc, stream=True))
    assert len(chunks) >= 2 and " ".join(chunks).split() == text.split()
    whole = model.generate_content([img, "Describe."], generation_config=gc)   # remote-code: prompt + answer
    assert whole.split()[-len(text.split()):] == text.split()
    # a logits processor (the xgrammar hook's interface) steers the eager path
    class Force:
        def __call__(self, input_ids, scores):
            scores = torch.full_like(scores, float("-inf"))
            scores[..., 42] = 0
            return scores
    forced = model.llm.generate(inputs_embeds=model._embed(ids, {"image": [images[0].cuda()]}, {"image": {}}, None, None)[0],
                                max_new_tokens=4, eos_token_id=None, logits_processor=[Force()])
    assert forced.tolist() == [[42, 42, 42, 42]]
    # CLI on a saved checkpoint
    save_pretrained(model, str(tmp_path / "NVILA-Lite-tiny"))
    p = tmp_path / "img.png"
    img.save(p)
    import llava.cli.infer as infer
    out = infer.main(["--model-path", str(tmp_path / "NVILA-Lite-tiny"), "--media", str(p), "--text", "Describe."])
    assert isinstance(out, str) and out in capsys.readouterr().out


def test_continuous_batching_matches_oracle(cuda):
    """f3: five requests of different lengths through three slots of the shared paged pool (batched
    skinny GEMMs + vila_decode_attention_batch in one CUDA graph; finished slots are refilled): every
    request's greedy ids against the oracle's, and the idle-slot / refill bookkeeping."""
    from vila_b200.model import tiny_test_config
    from vila_b200.serving import BatchedDecoder
    cfg = tiny_test_config(llm_layers=3)
    model = build(cfg, seed=15)
    reqs, wants = [], []
    oracle = oracle_from_state_dict(model.state_dict(), cfg, torch.float32)
    for i, n_text in enumerate([5, 12, 3, 9, 7]):
        ids, images = synth_inputs(cfg, n_images=1 if i % 2 == 0 else 0, n_text=n_text, seed=20 + i)
        reqs.append({"input_ids": ids, "media": {"image": [im.cuda() for im in images]} if images else None})
        wants.append(oracle.generate(ids, [im.float() for im in images], 10))
    got = model.generate_batch(reqs, max_new_tokens=10, slots=3, max_tokens_per_slot=256, eos_token_id=[])
    assert len(got) == 5 and all(len(g) == 10 for g in got)
    for g, (want, logits) in zip(got, wants):
        greedy_ids_match(g, want, logits, 3 * 2 ** -8 * logits.abs().max().item())
    # first tokens come from the ordinary prefill path: identical to single-request generate
    for r, g in zip(reqs, got):
        one = model.generate(input_ids=r["input_ids"], media=r["media"], max_new_tokens=2, eos_token_id=None)
        assert int(one[0, 0]) == g[0]
    # EOS frees a slot early; idle slots are skipped
    eos_tok = got[0][3]
    again = model.generate_batch(reqs[:2], max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[eos_tok])
    assert again[0] == got[0][:got[0].index(eos_tok) + 1]
    dec = BatchedDecoder(model.llm, slots=2, max_tokens_per_slot=256, max_new=8)
    dec.capture()
    dec.run(3)  # all idle: nothing happens
    assert int((dec.positions >= 0).sum()) == 0 and int(dec.step_idx.sum()) == 0
