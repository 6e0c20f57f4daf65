"""FP8 weight-only quantization (ssd_b200/quant.py) and FP8 checkpoint loading, on the CPU."""
import json

import pytest
import torch

from ssd_b200.quant import E4M3_MAX, quantize_fp8_rowwise

F8 = torch.float8_e4m3fn


def test_quantize_matches_definition_and_error_bound():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * torch.exp2(torch.randn(64, 1, generator=g) * 6)).to(torch.bfloat16)
    w[5] = 0
    w8, s = quantize_fp8_rowwise(w)
    wf = w.float()
    amax = wf.abs().amax(1)
    assert w8.dtype == F8 and s.dtype == torch.float32
    assert torch.equal(s[amax > 0], amax[amax > 0] / E4M3_MAX)
    assert s[5] == 1.0
    want = (wf / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(F8)
    assert torch.equal(w8.view(torch.uint8), want.view(torch.uint8))
    back = w8.float() * s[:, None]
    assert bool(((back - wf).abs() <= 2 ** -4 * wf.abs() + s[:, None] * 2 ** -10).all())


def _spec():
    from ssd_b200.runner import ModelSpec
    return ModelSpec(hidden=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=1024)


def _bf16_ckpt(g):
    sp = _spec()
    t = {"model.embed_tokens.weight": torch.randn(sp.vocab, sp.hidden, generator=g),
         "lm_head.weight": torch.randn(sp.vocab, sp.hidden, generator=g), "model.norm.weight": torch.ones(sp.hidden)}
    shapes = {"self_attn.q_proj": (256, 256), "self_attn.k_proj": (128, 256), "self_attn.v_proj": (128, 256),
              "self_attn.o_proj": (256, 256), "mlp.gate_proj": (512, 256), "mlp.up_proj": (512, 256),
              "mlp.down_proj": (256, 512)}
    for l in range(sp.layers):
        for leaf, shp in shapes.items():
            t[f"model.layers.{l}.{leaf}.weight"] = torch.randn(*shp, generator=g) * 0.05
        t[f"model.layers.{l}.input_layernorm.weight"] = torch.ones(sp.hidden)
        t[f"model.layers.{l}.post_attention_layernorm.weight"] = torch.ones(sp.hidden)
    return {k: v.to(torch.bfloat16).contiguous() for k, v in t.items()}


def _fp8_ckpt(t, scale_kind, scale_dtype):
    """Quantize every decoder linear of a bf16 checkpoint dict the way published FP8 checkpoints store it."""
    out = {}
    for k, v in t.items():
        if k.startswith("model.layers.") and k.endswith("_proj.weight"):
            vf = v.float()
            if scale_kind == "channel":
                s = vf.abs().amax(1, keepdim=True) / E4M3_MAX
            else:
                s = vf.abs().amax() / E4M3_MAX
                s = s.reshape(1) if scale_kind == "tensor" else s.reshape(())
            out[k] = (vf / s).clamp(-E4M3_MAX, E4M3_MAX).to(F8)
            out[k + "_scale"] = s.to(scale_dtype).contiguous()
            out[k.replace(".weight", ".input_scale")] = torch.ones(1)
        else:
            out[k] = v
    return out


def _write(path, tensors):
    from safetensors.torch import save_file
    save_file(tensors, str(path / "model.safetensors"))


def _dequant(lw, name):
    return lw[name].float() * lw[name + "_scale"][:, None]


@pytest.mark.parametrize("scale_kind", ["channel", "tensor", "scalar"])
@pytest.mark.parametrize("scale_dtype", [torch.float32, torch.bfloat16])
def test_fp8_checkpoint_loads_with_per_row_scales(tmp_path, scale_kind, scale_dtype):
    from ssd_b200.loader import load_safetensors_weights, shard_packed_weights
    t = _bf16_ckpt(torch.Generator().manual_seed(1))
    f = _fp8_ckpt(t, scale_kind, scale_dtype)
    _write(tmp_path, f)
    sp = _spec()
    w = load_safetensors_weights(str(tmp_path), sp, "cpu")
    assert all(n.endswith("input_scale") for n in w["ignored"]) and len(w["ignored"]) == 14
    lw = w["layers"][1]
    for name, parts in (("qkv", ["q", "k", "v"]), ("gate_up", ["gate", "up"])):
        r0 = 0
        for p in parts:
            leaf = f"model.layers.1.{'self_attn' if name == 'qkv' else 'mlp'}.{p}_proj.weight"
            n = f[leaf].shape[0]
            assert torch.equal(lw[name][r0:r0 + n].view(torch.uint8), f[leaf].view(torch.uint8))
            want_s = f[leaf + "_scale"].float().reshape(-1).expand(n)
            assert torch.equal(lw[name + "_scale"][r0:r0 + n], want_s), (name, p)
            r0 += n
    for name, leaf in (("o", "self_attn.o_proj"), ("down", "mlp.down_proj")):
        full = f[f"model.layers.1.{leaf}.weight"]
        assert torch.equal(lw[name].view(torch.uint8), full.view(torch.uint8))
    # tensor-parallel shards dequantize to the shards of the dequantized full weights, bit for bit
    for tp in (2, 4):
        for rank in range(tp):
            ws = load_safetensors_weights(str(tmp_path), sp, "cpu", tp, rank)
            ref = shard_packed_weights(w, sp, tp, rank)
            for l in range(sp.layers):
                for name in ("qkv", "o", "gate_up", "down"):
                    a, b = _dequant(ws["layers"][l], name), _dequant(ref["layers"][l], name)
                    assert torch.equal(a, b), (tp, rank, l, name)
                    full = _dequant(w["layers"][l], name)
                    if name in ("o", "down"):
                        n = full.shape[1] // tp
                        assert torch.equal(a, full[:, rank * n:(rank + 1) * n])


def test_fp8_rejections(tmp_path):
    from ssd_b200.loader import load_safetensors_weights
    from ssd_b200.quant import checkpoint_quantization, parse_quantization
    with pytest.raises(ValueError):
        parse_quantization("int4")
    t = _bf16_ckpt(torch.Generator().manual_seed(2))
    f = _fp8_ckpt(t, "channel", torch.float32)
    _write(tmp_path, f)
    with pytest.raises(NotImplementedError, match="target model only"):
        load_safetensors_weights(str(tmp_path), _spec(), "cpu", allow_fp8=False)
    blk = dict(f)
    k = "model.layers.0.mlp.down_proj.weight"
    blk[k + "_scale_inv"] = blk.pop(k + "_scale")
    _write(tmp_path, blk)
    with pytest.raises(NotImplementedError, match="block-wise"):
        load_safetensors_weights(str(tmp_path), _spec(), "cpu")

    class Hf:
        quantization_config = {"quant_method": "fp8", "weight_block_size": [128, 128]}
    with pytest.raises(NotImplementedError, match="block-wise"):
        checkpoint_quantization(Hf)
    Hf.quantization_config = {"quant_method": "compressed-tensors", "config_groups": {
        "group_0": {"weights": {"num_bits": 8, "type": "float", "strategy": "channel"}}}}
    assert checkpoint_quantization(Hf) == "fp8"
    Hf.quantization_config = {"quant_method": "fbgemm_fp8"}
    assert checkpoint_quantization(Hf) == "fp8"


def test_bf16_checkpoint_loads_as_before(tmp_path):
    from ssd_b200.loader import load_safetensors_weights, load_weights
    t = _bf16_ckpt(torch.Generator().manual_seed(3))
    _write(tmp_path, t)
    sp = _spec()
    w = load_safetensors_weights(str(tmp_path), sp, "cpu")
    assert "ignored" not in w
    lw = w["layers"][0]
    assert set(lw) == {"qkv", "o", "gate_up", "down", "input_norm", "post_norm"}
    assert torch.equal(lw["qkv"], torch.cat([t[f"model.layers.0.self_attn.{p}_proj.weight"] for p in "qkv"]))
    assert torch.equal(lw["down"], t["model.layers.0.mlp.down_proj.weight"])
    # quantize on load: the same bytes as quantizing the loaded bf16 matrices
    wq = load_weights(str(tmp_path), sp, "cpu", quantization="fp8")
    for name in ("qkv", "o", "gate_up", "down"):
        w8, s = quantize_fp8_rowwise(w["layers"][0][name])
        assert torch.equal(wq["layers"][0][name].view(torch.uint8), w8.view(torch.uint8))
        assert torch.equal(wq["layers"][0][name + "_scale"], s)
    assert wq["embed"].dtype == torch.bfloat16 and wq["lm_head"].dtype == torch.bfloat16


def test_config_quantization_option(tmp_path):
    from ssd_b200.config import Config
    cfg = {"hidden_size": 256, "num_hidden_layers": 2, "num_attention_heads": 4, "num_key_value_heads": 2,
           "intermediate_size": 512, "vocab_size": 1024, "rms_norm_eps": 1e-5, "max_position_embeddings": 4096}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    assert Config(str(tmp_path)).quantization is None
    assert Config(str(tmp_path), quantization="fp8").quantization == "fp8"
    with pytest.raises(ValueError):
        Config(str(tmp_path), quantization="fp4")
    cfg["quantization_config"] = {"quant_method": "fbgemm_fp8"}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    assert Config(str(tmp_path)).quantization == "fp8"


@pytest.mark.parametrize("tp", [2, 4])
def test_tp_quantize_on_load_uses_full_row_scales(tp):
    """Every rank quantizes its own bf16 shard (quantize-on-load); with the ranks' o / down row amax reduced by MAX, each
    rank's FP8 shard is exactly the shard of the FP8 full weights, bit for bit."""
    from oracle.model import ModelCfg, random_weights
    from ssd_b200.loader import shard_packed_weights
    from ssd_b200.quant import quantize_layers_
    from ssd_b200.runner import ModelSpec
    c = ModelCfg(hidden=256, layers=2, heads=4, kv_heads=4, head_dim=64, ffn=512, vocab=1024)
    sp = ModelSpec(hidden=256, layers=2, heads=4, kv_heads=4, head_dim=64, ffn=512, vocab=1024)
    full = random_weights(c, 5)
    for lw in full["layers"]:  # rows whose amax sits in different column shards
        lw["o"][3, 7] = 2.0
        lw["down"][5, 500] = -3.0
    shards = [shard_packed_weights(full, sp, tp, r) for r in range(tp)]
    # what the MAX all-reduce over the ranks returns, in the order the ranks call it (layer by layer, o then down)
    amax = [[(shards[r]["layers"][l][n].float().abs().amax(1)) for r in range(tp)] for l in range(2) for n in ("o", "down")]
    want_full = quantize_layers_({**full, "layers": [dict(lw) for lw in full["layers"]]})
    for r in range(tp):
        calls = iter(amax)
        got = quantize_layers_(shards[r], lambda a: torch.stack(next(calls)).amax(0))
        ref = shard_packed_weights(want_full, sp, tp, r)
        for l in range(2):
            for n in ("qkv", "o", "gate_up", "down"):
                assert torch.equal(got["layers"][l][n].view(torch.uint8), ref["layers"][l][n].view(torch.uint8)), (r, l, n)
                assert torch.equal(got["layers"][l][n + "_scale"], ref["layers"][l][n + "_scale"]), (r, l, n)
    # without the reduction a rank's o / down scales would come from its own columns only
    alone = quantize_layers_(shard_packed_weights(full, sp, tp, 1))
    assert not torch.equal(alone["layers"][0]["o_scale"], want_full["layers"][0]["o_scale"])
