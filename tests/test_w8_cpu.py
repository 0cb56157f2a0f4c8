"""`load_in_8bit` on the host: the row-wise int8 quantizer and dequantizer (eagle_b200.quant), the pairing of a checkpoint saved
in transformers' bitsandbytes 8-bit format, and the refusals that happen before an engine is created.  No GPU."""
import json
import os

import pytest
import torch

from eagle_b200 import quant
from eagle_b200.checkpoint import iter_int8_pairs, save_target_checkpoint, target_weights_int8


def test_quantizer_rounds_half_even_saturates_and_keeps_zero_rows():
    w = torch.tensor([[127.0, 0.5, -0.5, 1.5, -2.5, 63.5],     # SCB 127: q = W exactly, ties to even
                      [0.0, 0.0, 0.0, 0.0, 0.0, 0.0],          # zero row: SCB 0, q 0, no NaN
                      [-3.0, 3.0, 1.0, -1.0, 0.0, 2.0]])       # |max| on both signs: +-127
    q, scb = quant.quantize_int8_rowwise(w)
    assert q.dtype == torch.int8 and scb.dtype == torch.float32 and q.shape == w.shape and scb.shape == (3,)
    assert scb.tolist() == [127.0, 0.0, 3.0]
    assert q[0].tolist() == [127, 0, 0, 2, -2, 64]
    assert q[1].tolist() == [0] * 6
    assert q[2].tolist() == [-127, 127, 42, -42, 0, 85]
    assert not torch.isnan(quant.dequantize_int8_rowwise(q, scb, torch.bfloat16).float()).any()


def test_quantizer_matches_the_stated_rule_on_random_weights():
    g = torch.Generator().manual_seed(5)
    for dtype in (torch.bfloat16, torch.float16):
        w = (torch.randn(67, 300, generator=g) * 0.03).to(dtype)
        w[3] = 0
        q, scb = quant.quantize_int8_rowwise(w)
        wf = w.float()
        want_scb = wf.abs().amax(1)
        assert torch.equal(scb, want_scb)
        inv = torch.where(want_scb > 0, 127.0 / want_scb.clamp_min(1e-30), torch.zeros_like(want_scb))
        want_q = torch.round(wf * inv[:, None]).clamp(-127, 127).to(torch.int8)
        assert torch.equal(q, want_q)
        assert int(q.abs().max()) == 127 and (q.abs().amax(1)[torch.arange(67) != 3] == 127).all()


def test_dequantize_is_transformers_expression():
    g = torch.Generator().manual_seed(6)
    q = torch.randint(-127, 128, (50, 96), generator=g, dtype=torch.int8)
    scb = torch.rand(50, generator=g) * 0.2
    scb[7] = 0
    for dtype in (torch.bfloat16, torch.float16):
        got = quant.dequantize_int8_rowwise(q, scb, dtype)
        # transformers/integrations/bitsandbytes.py dequantize_bnb_weight, evaluated literally
        want = (q * scb.view(-1, 1) * 7.874015718698502e-3).to(dtype)
        assert got.dtype == dtype and torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_projection_names():
    assert quant.is_target_projection("model.layers.3.self_attn.k_proj.weight")
    assert quant.is_target_projection("model.layers.11.mlp.down_proj.SCB")
    for name in ("lm_head.weight", "model.embed_tokens.weight", "model.layers.0.input_layernorm.weight",
                 "head.midlayer.self_attn.q_proj.weight", "model.layers.x.mlp.up_proj.weight"):
        assert not quant.is_target_projection(name)


def _hf_8bit_dir(tmp_path):
    """A tiny target directory in the layout transformers writes for a bitsandbytes 8-bit model."""
    g = torch.Generator().manual_seed(8)
    sd, want = {}, {}
    for p in quant.PROJECTIONS:
        w = (torch.randn(128, 64, generator=g) * 0.02).to(torch.bfloat16)
        q, scb = quant.quantize_int8_rowwise(w)
        sd[f"model.layers.0.{p}.weight"] = q
        sd[f"model.layers.0.{p}.SCB"] = scb
        sd[f"model.layers.0.{p}.weight_format"] = torch.tensor(0, dtype=torch.uint8)
        want[f"model.layers.0.{p}.weight"] = (q, scb)
    sd["lm_head.weight"] = torch.randn(32, 64, generator=g).to(torch.bfloat16)
    sd["model.norm.weight"] = torch.ones(64, dtype=torch.bfloat16)
    cfg = {"hidden_size": 64, "quantization_config": {"quant_method": "bitsandbytes", "load_in_8bit": True, "load_in_4bit": False}}
    d = str(tmp_path / "t8")
    save_target_checkpoint(d, cfg, sd)
    return d, want


def test_hf_8bit_checkpoint_yields_weight_scb_pairs(tmp_path):
    d, want = _hf_8bit_dir(tmp_path)
    cfg = json.load(open(os.path.join(d, "config.json")))
    assert target_weights_int8(cfg) is True  # stored int8: loaded as is, whatever load_in_8bit says
    seen = {}
    for k, v, scb in iter_int8_pairs(d):
        assert not k.endswith((".weight_format", ".SCB"))
        seen[k] = (v, scb)
    assert set(seen) == set(want) | {"lm_head.weight", "model.norm.weight"}
    for k, (q, scb) in want.items():
        assert torch.equal(seen[k][0], q) and torch.equal(seen[k][1], scb)
    assert seen["lm_head.weight"][1] is None and seen["lm_head.weight"][0].dtype == torch.bfloat16


def test_unpaired_int8_weight_is_refused(tmp_path):
    q, _ = quant.quantize_int8_rowwise(torch.randn(8, 16))
    d = str(tmp_path / "bad")
    save_target_checkpoint(d, {}, {"model.layers.0.mlp.up_proj.weight": q})
    with pytest.raises(ValueError, match="unpaired"):
        list(iter_int8_pairs(d))


def test_quantization_switches():
    assert target_weights_int8({}, load_in_8bit=True) is True
    assert target_weights_int8({}) is False
    with pytest.raises(ValueError, match="load_in_8bit=True"):
        target_weights_int8({}, load_in_4bit=True)
    for qc in ({"quant_method": "bitsandbytes", "load_in_4bit": True}, {"quant_method": "fp8"}, {"quant_method": "gptq", "bits": 4}):
        with pytest.raises(ValueError, match="supported: load_in_8bit"):
            target_weights_int8({"quantization_config": qc})


def test_from_pretrained_refuses_before_creating_an_engine(tmp_path, monkeypatch):
    from eagle_b200 import EaModel

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(EaModel, "__init__", no_engine)
    with pytest.raises(ValueError, match="4-bit"):
        EaModel.from_pretrained(base_model_path=str(tmp_path), ea_model_path=str(tmp_path), load_in_4bit=True)
    d = tmp_path / "fp8"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"], "quantization_config": {"quant_method": "fp8"}}))
    with pytest.raises(ValueError, match="unsupported quantization_config"):
        EaModel.from_pretrained(base_model_path=str(d), ea_model_path=str(d), load_in_8bit=True)
