"""llava/model/builder.py:27-156 — load_pretrained_model -> (tokenizer, model, image_processor, context_len)."""


def load_pretrained_model(model_path, model_name, model_base=None, load_8bit=False, load_4bit=False,
                          device_map="auto", device="cuda", **kwargs):
    if load_8bit or load_4bit:
        raise NotImplementedError("bitsandbytes quantised loading is out of scope (bf16 weights fit one H100)")
    from vila_b200.model.loading import load_pretrained
    # decode_weights="fp8" / "w4a16": the single-stream decoder streams e4m3 weights with per-row scales
    # (vila_gemv_fp8) / 4-bit weights with group-128 scales and zero points (vila_gemv_w4a16);
    # load_8bit / load_4bit keep their bitsandbytes meaning and are refused above
    model = load_pretrained(model_path, device=device, decode_weights=kwargs.pop("decode_weights", "bf16"))
    context_len = getattr(model.config, "model_max_length", 2048)
    return model.tokenizer, model, model.vision_tower.image_processor, context_len
