"""CPU: the C-ABI library loads and exports every symbol include/vila_b200.h declares (no compute
calls), fails loudly without a GPU, and the host-side glue behaves like the reference's."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def header_functions():
    text = (ROOT / "include" / "vila_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vila_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from vila_b200 import _lib
    lib = _lib.load()
    names = header_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/vila_b200.h but not exported"
    # and every ctypes signature corresponds to a declared function
    for n in _lib.SIGNATURES:
        assert n in names, f"{n} bound in _lib.py but not declared in the header"
    assert lib.vila_abi_version() == 3


# the ctypes class in vila_b200/_lib.py of every parameter struct the header declares
STRUCT_CLASSES = {
    "vila_fmha_params": "FmhaParams",
    "vila_gemv_params": "GemvParams",
    "vila_gemv_batch_params": "GemvBatchParams",
    "vila_decode_attn_params": "DecodeAttnParams",
    "vila_decode_attn_split_params": "DecodeAttnSplitParams",
    "vila_decode_attn_fp8_params": "DecodeAttnFp8Params",
    "vila_sample_params": "SampleParams",
    "vila_sample_finalize_params": "SampleFinalizeParams",
    "vila_logprobs_params": "LogprobsParams",
    "vila_logprobs_row_params": "LogprobsRowParams",
    "vila_penalty_params": "PenaltyParams",
    "vila_penalty_row_params": "PenaltyRowParams",
}
SCALAR_CTYPES = {"int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32, "float": ctypes.c_float}


def header_struct_fields(body):
    """(name, is_pointer, base type) of every field of a struct body of the header, in declaration order."""
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        first, *rest = decl.split(",")
        tokens = first.replace("*", " * ").split()
        base = " ".join(t for t in tokens[:-1] if t not in ("*", "const"))
        fields.append((tokens[-1], "*" in tokens, base))
        fields.extend((x.strip().lstrip("*"), x.strip().startswith("*"), base) for x in rest)
    return fields


def test_struct_layouts_match_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    structs = dict(re.findall(r"typedef struct (vila_\w+_params) \{(.*?)\} \1;", text, flags=re.S))
    assert sorted(structs) == sorted(STRUCT_CLASSES), "every parameter struct of the header needs a ctypes class"
    for cname, body in structs.items():
        cls = getattr(_lib, STRUCT_CLASSES[cname])
        fields = header_struct_fields(body)
        assert [f[0] for f in fields] == [f[0] for f in cls._fields_], (cname, fields)
        for (name, is_pointer, base), (_, ctype) in zip(fields, cls._fields_):
            if is_pointer:
                assert ctype is ctypes.c_void_p or issubclass(ctype, ctypes._Pointer), (cname, name, ctype)
            else:
                assert base in SCALAR_CTYPES, f"{cname}.{name}: {base} has no ctypes counterpart here"
                assert ctype is SCALAR_CTYPES[base], (cname, name, base, ctype)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_fails_loudly_without_gpu():
    from vila_b200 import _lib, ops
    lib = _lib.load()
    rc = lib.vila_layernorm(None, None, None, None, 1, 8, 1e-6, None)
    assert rc != 0 and b"no CUDA device" in lib.vila_last_error()
    with pytest.raises(RuntimeError):
        ops.linear(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    with pytest.raises(RuntimeError):
        LlavaLlamaModel(tiny_test_config())


def test_product_never_imports_oracle():
    for f in (ROOT / "vila_b200").rglob("*.py"):
        src = f.read_text()
        assert "import oracle" not in src and "from oracle" not in src, f


def test_configs_and_tokenizer():
    from vila_b200.model import SyntheticTokenizer, nvila_8b, nvila_lite_3b, nvila_video_8b
    c = nvila_8b()
    assert c.llm_cfg.head_dim == 128 and c.vision_tower_cfg.num_patches == 1024
    assert c.mm_hidden_size == 1152 and nvila_lite_3b().mm_projector_type == "mlp_downsample_3x3_fix"
    assert nvila_video_8b().num_video_frames == 64
    tok = SyntheticTokenizer(c)
    ids = tok("ab<image>\nc").input_ids
    assert ids.count(c.image_token_id) == 1 and ids[3] == c.newline_token_ids[0]
    assert tok("\n").input_ids == list(c.newline_token_ids)


def test_dynamic_s2_preprocess_block_sizes():
    from PIL import Image
    from vila_b200.model import media, nvila_8b_dynamic_s2
    cfg = nvila_8b_dynamic_s2()
    img = Image.new("RGB", (1600, 800), (120, 30, 200))
    tiles, bs = media.dynamic_s2_preprocess(img, list(cfg.s2_scales), 12, 448)
    # 1 + 4 tiles for the fixed scales, then rows x cols of the closest aspect ratio with >= 9 tiles
    assert bs[0] * bs[1] >= 9 and len(tiles) == 1 + 4 + bs[0] * bs[1]
    assert bs[1] > bs[0]  # landscape image -> more columns than rows
    tensors, block_sizes = media.process_images([img], cfg)
    assert block_sizes == [bs] and tensors[0].shape == (3, 448, 448)
    assert abs(float(tensors[0][0].mean()) - (120 / 255 - 0.5) / 0.5) < 1e-2
    text, images = media.extract_media(["look: ", img, "what?"], cfg)
    assert text == "look: <image>what?" and len(images) == 1  # bare token: the "\n" is the encoder's end token


def test_dynamic_s2_preprocess_matches_reference_fixture():
    """Host-side tiling (vila_b200.model.media) against tests/golden/media_preprocess.pt, which holds the
    output of the REFERENCE's mm_utils.dynamic_s2_preprocess (llava/mm_utils.py:341-405) on the same
    seeded images (oracle/gen_golden.py): block sizes, tile count, exact pixel sums and a strided
    thumbnail of every tile."""
    import numpy as np
    from PIL import Image
    from vila_b200.model import media
    fx = torch.load(ROOT / "tests" / "golden" / "media_preprocess.pt")
    assert len(fx) == 8
    for item in fx:
        w, h = item["size"]
        img = Image.fromarray(np.random.RandomState(item["seed"]).randint(0, 256, (h, w, 3), dtype=np.uint8))
        tiles, bs = media.dynamic_s2_preprocess(img, [448, 896, 1344], 12, 448)
        assert tuple(bs) == tuple(item["block_size"]) and len(tiles) == item["n_tiles"], item["size"]
        arrs = [np.asarray(t, dtype=np.int64) for t in tiles]
        assert [int(a.sum()) for a in arrs] == item["tile_sums"].tolist(), item["size"]
        thumbs = np.stack([a[::28, ::28, :] for a in arrs]).astype(np.uint8)
        assert np.array_equal(thumbs, item["tile_thumbs"].numpy()), item["size"]
