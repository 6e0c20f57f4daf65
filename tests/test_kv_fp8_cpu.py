"""CPU tests of the FP8 KV cache's host side: Config.kv_cache_dtype, checkpoint KV scales (found, defaulted, rejected,
read as fp32, ignored under "auto"), the KV page budget of an e4m3 target, and the new C ABI entries."""
import json
import math
from unittest import mock

import pytest
import torch

from ssd_b200 import lib as L
from ssd_b200.quant import parse_kv_cache_dtype, quantize_kv_fp8, resolve_kv_scales


@pytest.mark.parametrize("v,want", [("auto", "auto"), ("bf16", "auto"), ("bfloat16", "auto"), ("fp8", "fp8"),
                                    ("fp8_e4m3", "fp8")])
def test_kv_cache_dtype_parsing(v, want):
    assert parse_kv_cache_dtype(v) == want


def test_kv_cache_dtype_rejections():
    with pytest.raises(NotImplementedError, match="e5m2"):
        parse_kv_cache_dtype("fp8_e5m2")
    for bad in ("fp16", "int8", "", None, "FP8"):
        with pytest.raises(ValueError):
            parse_kv_cache_dtype(bad)


def test_config_takes_kv_cache_dtype(tmp_path):
    from ssd_b200 import synth
    from ssd_b200.config import Config
    t = synth.make_model_dir(str(tmp_path), "llama-tiny-target", "target", seed=0)
    assert Config(t).kv_cache_dtype == "auto"
    assert Config(t, kv_cache_dtype="bfloat16").kv_cache_dtype == "auto"
    assert Config(t, kv_cache_dtype="fp8_e4m3").kv_cache_dtype == "fp8"
    with pytest.raises(NotImplementedError):
        Config(t, kv_cache_dtype="fp8_e5m2")
    with pytest.raises(ValueError):
        Config(t, kv_cache_dtype="half")


def test_quantize_kv_fp8_saturates_and_rounds_to_nearest_even():
    y = torch.tensor([0.0, 1.0, 500.0, -1e4, 2 ** -10, 3 * 2 ** -10, 17.0, 19.0], dtype=torch.bfloat16)
    got = quantize_kv_fp8(y, 1.0).float().tolist()
    # 2^-10 is half the smallest subnormal step (ties to even -> 0); 3 * 2^-10 -> 2^-8; 17 is a tie between 16 and 18
    # (-> 16, even mantissa), 19 between 18 and 20 (-> 20)
    assert got == [0.0, 1.0, 448.0, -448.0, 0.0, 2 ** -8, 16.0, 20.0]
    # the division is IEEE y / s, not y * (1 / s)
    s = 0.0371
    y = torch.randn(4096, generator=torch.Generator().manual_seed(0)).to(torch.bfloat16)
    want = (y.float() / torch.full((4096,), s)).clamp(-448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(quantize_kv_fp8(y, s).view(torch.uint8), want.view(torch.uint8))


# ------------------------------------------------------------------------------------------------ checkpoint scales
def _checkpoint(path, layers=2, scales=None, dtype=torch.float32):
    from safetensors.torch import save_file
    path.mkdir()
    d, H, KV, hd, ffn, V = 128, 2, 1, 64, 256, 256
    g = torch.Generator().manual_seed(0)
    r = lambda *s: (0.02 * torch.randn(*s, generator=g)).to(torch.bfloat16)
    t = {"model.embed_tokens.weight": r(V, d), "lm_head.weight": r(V, d), "model.norm.weight": torch.ones(d).bfloat16()}
    for l in range(layers):
        p = f"model.layers.{l}."
        t.update({p + "self_attn.q_proj.weight": r(H * hd, d), p + "self_attn.k_proj.weight": r(KV * hd, d),
                  p + "self_attn.v_proj.weight": r(KV * hd, d), p + "self_attn.o_proj.weight": r(d, H * hd),
                  p + "mlp.gate_proj.weight": r(ffn, d), p + "mlp.up_proj.weight": r(ffn, d),
                  p + "mlp.down_proj.weight": r(d, ffn), p + "input_layernorm.weight": torch.ones(d).bfloat16(),
                  p + "post_attention_layernorm.weight": torch.ones(d).bfloat16()})
    for (kind, l), s in (scales or {}).items():
        t[f"model.layers.{l}.self_attn.{kind}_scale"] = torch.tensor(s, dtype=dtype)
    save_file(t, str(path / "model.safetensors"))
    cfg = {"model_type": "llama", "hidden_size": d, "num_hidden_layers": layers, "num_attention_heads": H,
           "num_key_value_heads": KV, "head_dim": hd, "intermediate_size": ffn, "vocab_size": V, "rms_norm_eps": 1e-5,
           "rope_theta": 500000.0, "max_position_embeddings": 2048}
    (path / "config.json").write_text(json.dumps(cfg))
    return str(path)


def _load(path, kv):
    from ssd_b200.config import load_hf_config
    from ssd_b200.loader import load_weights, spec_from_config
    return load_weights(path, spec_from_config(load_hf_config(path)), "cpu", kv_cache_dtype=kv)


def test_checkpoint_kv_scales_found_as_fp32(tmp_path):
    sc = {("k", 0): 0.0213, ("v", 0): 0.0119, ("k", 1): 0.0371, ("v", 1): 1 / 3}
    w = _load(_checkpoint(tmp_path / "m", scales=sc), "fp8")
    ks, vs = w["kv_scales"]
    f32 = lambda x: torch.tensor(x, dtype=torch.float32).item()
    assert ks == [f32(sc[("k", 0)]), f32(sc[("k", 1)])] and vs == [f32(sc[("v", 0)]), f32(sc[("v", 1)])]
    # not bf16-rounded: 0.0213 is not a bf16 value
    assert ks[0] != torch.tensor(0.0213).bfloat16().item()


def test_checkpoint_kv_scales_stored_as_bf16_read_exactly(tmp_path):
    sc = {("k", 0): 0.5, ("v", 0): 0.25, ("k", 1): 0.0213, ("v", 1): 3.0}
    ks, vs = _load(_checkpoint(tmp_path / "m", scales=sc, dtype=torch.bfloat16), "fp8")["kv_scales"]
    assert ks[1] == torch.tensor(0.0213).bfloat16().float().item() and vs == [0.25, 3.0]


def test_checkpoint_without_kv_scales_defaults_to_one(tmp_path):
    assert _load(_checkpoint(tmp_path / "m"), "fp8")["kv_scales"] == ([1.0, 1.0], [1.0, 1.0])


@pytest.mark.parametrize("sc,match", [
    ({("k", 0): 0.1, ("v", 0): 0.1}, "some layers only"),                          # layer 1 has none
    ({("k", 0): 0.1, ("v", 0): 0.1, ("k", 1): 0.1}, "some layers only"),           # layer 1 lacks v
    ({("k", 0): 0.1, ("v", 0): 0.0, ("k", 1): 0.1, ("v", 1): 0.1}, "finite and > 0"),
    ({("k", 0): -0.1, ("v", 0): 0.1, ("k", 1): 0.1, ("v", 1): 0.1}, "finite and > 0"),
    ({("k", 0): math.inf, ("v", 0): 0.1, ("k", 1): 0.1, ("v", 1): 0.1}, "finite and > 0"),
    ({("k", 0): math.nan, ("v", 0): 0.1, ("k", 1): 0.1, ("v", 1): 0.1}, "finite and > 0"),
])
def test_checkpoint_kv_scales_rejected(tmp_path, sc, match):
    with pytest.raises(ValueError, match=match):
        _load(_checkpoint(tmp_path / "m", scales=sc), "fp8")


def test_auto_loads_a_checkpoint_with_kv_scales_exactly_as_before(tmp_path):
    sc = {("k", 0): 0.1, ("v", 0): 0.2, ("k", 1): 0.3, ("v", 1): 0.4}
    a = _load(_checkpoint(tmp_path / "plain"), "auto")
    b = _load(_checkpoint(tmp_path / "scaled", scales=sc), "auto")
    assert "kv_scales" not in a and "kv_scales" not in b
    assert set(a) == set(b)
    for k in ("embed", "lm_head", "final_norm"):
        assert torch.equal(a[k], b[k])
    for la, lb in zip(a["layers"], b["layers"]):
        assert set(la) == set(lb)
        assert all(torch.equal(la[n], lb[n]) for n in la)


def test_resolve_kv_scales_draft_is_rejected():
    from ssd_b200.loader import load_weights
    with pytest.raises(ValueError, match="draft"):
        load_weights("/nonexistent", None, "cpu", is_target=False, kv_cache_dtype="fp8")
    assert resolve_kv_scales({}, 3) == ([1.0] * 3, [1.0] * 3)


# ------------------------------------------------------------------------------------------------ page budget
def test_fp8_target_pages_double_and_draft_sizes_from_the_rest(tmp_path):
    """With free memory binding (not the max_num_seqs * max_model_len cap), an e4m3 target gets twice the pages of a
    bf16 one, and the draft's cache is sized from what the target's pages leave."""
    from ssd_b200.config import Config
    from ssd_b200.loader import kv_block_bytes, kv_blocks_for, spec_from_config
    from ssd_b200 import synth
    t = synth.make_model_dir(str(tmp_path), "llama-tiny-target", "target", seed=0)
    d = synth.make_model_dir(str(tmp_path), "llama-tiny-draft", "draft", seed=0)
    cfg = Config(t, speculate=True, draft=d, max_num_seqs=32, max_model_len=4096, kvcache_block_size=256,
                 gpu_memory_utilization=0.5, kv_cache_dtype="fp8")
    ts, ds = spec_from_config(cfg.hf_config), spec_from_config(cfg.draft_hf_config)
    b16, b8 = kv_block_bytes(cfg, ts, 1), kv_block_bytes(cfg, ts, 1, fp8=True)
    assert b16 == 2 * b8 == 2 * ts.layers * 256 * ts.kv_heads * ts.head_dim * 2
    want = 32 * cfg.max_blocks * 2 + 2
    free = 40 * b16  # far below what `want` pages would need
    assert want > 200
    with mock.patch("torch.cuda.mem_get_info", return_value=(free, 80 << 30)):
        n16 = kv_blocks_for(cfg, ts, 1, 0.8)
        n8 = kv_blocks_for(cfg, ts, 1, 0.8, fp8=True)
        assert n16 == int(free * 0.5 * 0.8) // b16 and n8 == int(free * 0.5 * 0.8) // b8
        assert n8 == 2 * n16 < want
        d16 = kv_blocks_for(cfg, ds, 1, 0.75, reserved=n16 * b16)
        d8 = kv_blocks_for(cfg, ds, 1, 0.75, reserved=n8 * b8)
        # the target's pages cost the same bytes either way, so the draft gets the same pages
        assert d8 == d16 == int((free - n16 * b16) * 0.5 * 0.75) // kv_block_bytes(cfg, ds, 1)


# ------------------------------------------------------------------------------------------------ C ABI
def test_new_abi_entries_are_declared_and_bound():
    import re
    from pathlib import Path
    header = (Path(__file__).resolve().parent.parent / "include" / "ssdk.h").read_text()
    for name, nargs in (("ssdk_bind_kv_cache_fp8", 6), ("ssdk_rope_store_kv_fp8", 17), ("ssdk_paged_attn_fp8", 18),
                        ("ssdk_paged_attn_varlen_fp8", 18)):
        m = re.search(rf"\bint\s+{name}\s*\(([^;]*)\);", header)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(L.SIGNATURES[name][1]), name
    # the scale arguments are floats (by value for the ops, host arrays for the bind)
    assert L.SIGNATURES["ssdk_bind_kv_cache_fp8"][1][4:] == [L.c_f32p, L.c_f32p]
    import ctypes as C
    assert L.SIGNATURES["ssdk_paged_attn_fp8"][1][14:17] == [C.c_float] * 3
    assert L.SIGNATURES["ssdk_rope_store_kv_fp8"][1][14:16] == [C.c_float] * 2
