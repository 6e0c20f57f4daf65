"""An FP8 draft on the CPU side: Config.draft_quantization, FP8 draft checkpoints (found by their quantization_config or by
their e4m3 tensors), quantize-on-load of a bf16 draft, and the C ABI's runtime config, whose last field became draft_fp8
at the offset and size of the old reserved field."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest
import torch

from ssd_b200.quant import quantize_fp8_rowwise
from tests.test_fp8_cpu import _bf16_ckpt, _fp8_ckpt, _spec, _write

F8 = torch.float8_e4m3fn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HF = {"hidden_size": 256, "num_hidden_layers": 2, "num_attention_heads": 4, "num_key_value_heads": 2,
       "intermediate_size": 512, "vocab_size": 1024, "rms_norm_eps": 1e-5, "max_position_embeddings": 4096}


def _dirs(tmp_path, draft_qc=None, target_qc=None):
    out = []
    for name, qc in (("target", target_qc), ("draft", draft_qc)):
        d = tmp_path / name
        d.mkdir()
        (d / "config.json").write_text(json.dumps({**_HF, **({"quantization_config": qc} if qc else {})}))
        out.append(str(d))
    return out


@pytest.mark.parametrize("quantization", [None, "fp8"])
@pytest.mark.parametrize("draft_quantization", [None, "fp8"])
def test_draft_quantization_is_independent_of_quantization(tmp_path, quantization, draft_quantization):
    from ssd_b200.config import Config
    t, d = _dirs(tmp_path)
    c = Config(t, speculate=True, draft=d, quantization=quantization, draft_quantization=draft_quantization)
    assert (c.quantization, c.draft_quantization) == (quantization, draft_quantization)


def test_draft_quantization_rejections(tmp_path):
    from ssd_b200.config import Config
    t, d = _dirs(tmp_path)
    for bad in ("fp4", "int8", "FP8"):
        with pytest.raises(ValueError):
            Config(t, speculate=True, draft=d, draft_quantization=bad)


@pytest.mark.parametrize("qc", [
    {"quant_method": "fbgemm_fp8"},
    {"quant_method": "fp8"},
    {"quant_method": "compressed-tensors", "config_groups": {"group_0": {
        "targets": ["Linear"], "weights": {"num_bits": 8, "type": "float", "strategy": "channel", "symmetric": True}}}},
])
def test_fp8_draft_checkpoint_is_found_by_its_config(tmp_path, qc):
    from ssd_b200.config import Config
    t, d = _dirs(tmp_path, draft_qc=qc)
    c = Config(t, speculate=True, draft=d)
    assert c.draft_quantization == "fp8" and c.quantization is None


@pytest.mark.parametrize("qc,match", [
    ({"quant_method": "awq", "bits": 4}, "only FP8"),
    ({"quant_method": "gptq", "bits": 4}, "only FP8"),
    ({"quant_method": "fp8", "weight_block_size": [128, 128]}, "block-wise"),
    ({"quant_method": "compressed-tensors", "config_groups": {"group_0": {
        "weights": {"num_bits": 8, "type": "float", "strategy": "block"}}}}, "block-wise"),
])
def test_other_quantized_draft_checkpoints_are_refused(tmp_path, qc, match):
    from ssd_b200.config import Config
    t, d = _dirs(tmp_path, draft_qc=qc)
    with pytest.raises(NotImplementedError, match=match):
        Config(t, speculate=True, draft=d)


@pytest.mark.parametrize("scale_kind", ["channel", "tensor", "scalar"])
@pytest.mark.parametrize("scale_dtype", [torch.float32, torch.bfloat16])
def test_fp8_draft_checkpoint_loads_as_fp8_by_its_tensors(tmp_path, scale_kind, scale_dtype):
    """A draft checkpoint with e4m3 decoder linears and no quantization_config: loaded as FP8 with per-row scales, and
    draft_quantization then reads "fp8"."""
    from ssd_b200.loader import load_draft_weights, load_safetensors_weights
    f = _fp8_ckpt(_bf16_ckpt(torch.Generator().manual_seed(4)), scale_kind, scale_dtype)
    _write(tmp_path, f)
    cfg = SimpleNamespace(draft=str(tmp_path), draft_quantization=None)
    w = load_draft_weights(cfg, _spec(), "cpu")
    assert cfg.draft_quantization == "fp8"
    ref = load_safetensors_weights(str(tmp_path), _spec(), "cpu")  # the target's loader on the same files
    for lw, lr in zip(w["layers"], ref["layers"]):
        for name in ("qkv", "o", "gate_up", "down"):
            assert lw[name].dtype == F8 and lw[name + "_scale"].dtype == torch.float32
            assert torch.equal(lw[name].view(torch.uint8), lr[name].view(torch.uint8))
            assert torch.equal(lw[name + "_scale"], lr[name + "_scale"])
    assert w["embed"].dtype == torch.bfloat16 and w["lm_head"].dtype == torch.bfloat16


def test_partly_fp8_draft_checkpoint_is_completed_to_fp8(tmp_path):
    """A draft runs in one weight format: a bf16 linear next to e4m3 ones is quantized on load."""
    from ssd_b200.loader import load_draft_weights
    t = _bf16_ckpt(torch.Generator().manual_seed(5))
    f = _fp8_ckpt(t, "channel", torch.float32)
    for leaf in ("mlp.down_proj.weight", "mlp.down_proj.weight_scale", "mlp.down_proj.input_scale"):
        f.pop(f"model.layers.1.{leaf}")
    f["model.layers.1.mlp.down_proj.weight"] = t["model.layers.1.mlp.down_proj.weight"]
    _write(tmp_path, f)
    cfg = SimpleNamespace(draft=str(tmp_path), draft_quantization=None)
    w = load_draft_weights(cfg, _spec(), "cpu")
    assert cfg.draft_quantization == "fp8"
    assert all(lw[n].dtype == F8 for lw in w["layers"] for n in ("qkv", "o", "gate_up", "down"))
    w8, s = quantize_fp8_rowwise(t["model.layers.1.mlp.down_proj.weight"])
    assert torch.equal(w["layers"][1]["down"].view(torch.uint8), w8.view(torch.uint8))
    assert torch.equal(w["layers"][1]["down_scale"], s)


def test_draft_quantize_on_load_equals_rowwise_quantization(tmp_path):
    from ssd_b200.loader import load_draft_weights, load_safetensors_weights
    t = _bf16_ckpt(torch.Generator().manual_seed(6))
    _write(tmp_path, t)
    bf = load_safetensors_weights(str(tmp_path), _spec(), "cpu")
    cfg = SimpleNamespace(draft=str(tmp_path), draft_quantization="fp8")
    w = load_draft_weights(cfg, _spec(), "cpu")
    for l in range(_spec().layers):
        for name in ("qkv", "o", "gate_up", "down"):
            w8, s = quantize_fp8_rowwise(bf["layers"][l][name])
            assert torch.equal(w["layers"][l][name].view(torch.uint8), w8.view(torch.uint8)), (l, name)
            assert torch.equal(w["layers"][l][name + "_scale"], s), (l, name)
    for k in ("embed", "lm_head", "final_norm"):
        assert torch.equal(w[k], bf[k])
    # a bf16 draft without the option stays bf16
    cfg = SimpleNamespace(draft=str(tmp_path), draft_quantization=None)
    w = load_draft_weights(cfg, _spec(), "cpu")
    assert cfg.draft_quantization is None and w["layers"][0]["qkv"].dtype == torch.bfloat16


def test_runtime_cfg_layout_is_unchanged():
    """ssdk_runtime_cfg keeps eight int32 fields; draft_fp8 took the last one's place (offset 28, 4 bytes)."""
    from ssd_b200 import lib as L
    names = ["spec_k", "max_batch", "block_size", "max_blocks_per_seq", "use_graph", "use_pdl", "jit_speculate", "draft_fp8"]
    assert [f[0] for f in L.RuntimeCfg._fields_] == names
    assert C.sizeof(L.RuntimeCfg) == 32
    for i, n in enumerate(names):
        assert getattr(L.RuntimeCfg, n).offset == 4 * i and getattr(L.RuntimeCfg, n).size == 4
    rt = L.RuntimeCfg(1, 2, 3, 4, 5, 6, 7, 1)  # positional, as before
    assert rt.draft_fp8 == 1
    with open(os.path.join(ROOT, "include", "ssdk.h")) as f:
        hdr = f.read()
    body = hdr[hdr.index("typedef struct ssdk_runtime_cfg"):hdr.index("} ssdk_runtime_cfg;")]
    assert [ln.split()[1].rstrip(";") for ln in body.splitlines() if ln.strip().startswith("int32_t")] == names
