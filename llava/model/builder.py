"""llava/model/builder.py:27-156 — load_pretrained_model -> (tokenizer, model, image_processor, context_len)."""


def load_pretrained_model(model_path, model_name, model_base=None, load_8bit=False, load_4bit=False,
                          device_map="auto", device="cuda", **kwargs):
    if load_8bit or load_4bit:
        raise NotImplementedError("bitsandbytes quantised loading is out of scope (bf16 weights fit one H100)")
    from vila_b200.model.loading import load_pretrained
    model = load_pretrained(model_path, device=device)
    context_len = getattr(model.config, "model_max_length", 2048)
    return model.tokenizer, model, model.vision_tower.image_processor, context_len
