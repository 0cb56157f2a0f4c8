"""FP8 target weights without a GPU: the block quantizer and dequantizer against transformers' own FP8 conversion ops, the
fine-grained FP8 checkpoint round trip, and every quantization_config / checkpoint refusal, raised before an engine exists."""
import json
from types import SimpleNamespace

import pytest
import torch

from eagle_b200 import quant
from eagle_b200.checkpoint import iter_fp8_pairs, save_target_checkpoint, target_weights_fp8, target_weights_int8

PROJ = "model.layers.0.mlp.up_proj.weight"


def transformers_ops():
    fp8 = pytest.importorskip("transformers.integrations.finegrained_fp8")
    from transformers import FineGrainedFP8Config
    hq = SimpleNamespace(quantization_config=FineGrainedFP8Config())  # the quantizer object the ops read the block size from
    return fp8.Fp8Quantize(hq), fp8.Fp8Dequantize(hq)


def weights(dtype):
    """Weights with an all-zero block, a saturating outlier block, blocks small enough for subnormal e4m3 codes and a Llama-width
    row block."""
    g = torch.Generator().manual_seed(0)
    out = []
    w = (torch.randn(384, 512, generator=g) * 0.02).to(dtype)
    w[:128, :128] = 0  # all-zero block
    w[128:256, 128:256] *= 1000  # the block amax maps to 448, the rest spreads over the whole range
    w[256:384, 256:384] = (torch.randn(128, 128, generator=g) * 0.02).to(dtype)
    w[300, 300] = 5.0  # one large value: the rest of its block quantizes into e4m3 subnormals
    out.append(w)
    out.append((torch.randn(128, 4096, generator=g) * 0.02).to(dtype))  # a 128-row slice of a Llama-3-8B projection
    return out


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantizer_and_dequantizer_equal_transformers(dtype):
    qop, dqop = transformers_ops()
    for w in weights(dtype):
        want = qop.convert({PROJ: [w]})
        q, s = quant.quantize_fp8_block(w)
        assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
        assert torch.equal(q.view(torch.uint8), want[PROJ].view(torch.uint8))
        assert torch.equal(s, want[PROJ[: -len("weight")] + "weight_scale_inv"])
        wd = dqop.convert({"weight$": [q], "weight_scale_inv": [s]}, full_layer_name=PROJ)[PROJ].to(dtype)
        assert torch.equal(quant.dequantize_fp8_block(q, s, dtype).view(torch.int16), wd.view(torch.int16))
    w = weights(dtype)[0]
    q, s = quant.quantize_fp8_block(w)
    codes = q.view(torch.uint8)
    assert int(codes[:128, :128].max()) == 0 and float(s[0, 0]) == 1.0  # all-zero block: scale 1, codes 0
    assert float(q[128:256, 128:256].float().abs().max()) == 448.0  # the block amax saturates to the largest e4m3 value
    sub = codes[256:384, 256:384] & 0x7F
    assert bool(((sub > 0) & (sub < 8)).any())  # e4m3 subnormal codes occur


def test_quantizer_refuses_ragged_shapes():
    for shape in ((128, 200), (100, 128)):
        with pytest.raises(ValueError, match="multiple of the 128"):
            quant.quantize_fp8_block(torch.randn(*shape))


def sd_small():
    g = torch.Generator().manual_seed(1)
    sd = {f"model.layers.0.{p}.weight": (torch.randn(256, 128, generator=g) * 0.02).to(torch.bfloat16) for p in quant.PROJECTIONS}
    sd["model.norm.weight"] = torch.ones(128, dtype=torch.bfloat16)
    sd["lm_head.weight"] = torch.randn(256, 128, generator=g).to(torch.bfloat16)
    return sd


def test_checkpoint_round_trip(tmp_path):
    sd = sd_small()
    d = str(tmp_path / "fp8")
    save_target_checkpoint(d, {"architectures": ["LlamaForCausalLM"], "num_hidden_layers": 1}, sd, fp8=True)
    cfg = json.load(open(f"{d}/config.json"))
    assert target_weights_fp8(cfg["quantization_config"], 1) is True
    seen = {k: (v, s) for k, v, s in iter_fp8_pairs(d)}
    assert set(seen) == set(sd)
    for k, w in sd.items():
        v, s = seen[k]
        if quant.is_target_projection(k):
            q, si = quant.quantize_fp8_block(w)
            assert torch.equal(v.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s, si)
        else:
            assert s is None and torch.equal(v, w)


def test_stored_checkpoint_refusals(tmp_path):
    def write(name, mutate):
        d = tmp_path / name
        save_target_checkpoint(str(d), {}, sd_small(), fp8=True)
        from safetensors.torch import load_file, save_file
        sd = load_file(str(d / "model.safetensors"))
        mutate(sd)
        save_file(sd, str(d / "model.safetensors"))
        return str(d)

    cases = [("static", lambda sd: sd.update({"model.layers.0.mlp.up_proj.activation_scale": torch.ones(1)}), "activation scales"),
             ("unpaired", lambda sd: sd.pop("model.layers.0.mlp.down_proj.weight_scale_inv"), "unpaired"),
             ("scale_shape", lambda sd: sd.update({"model.layers.0.mlp.up_proj.weight_scale_inv": torch.ones(1, 1)}), "128 x 128 block"),
             ("elsewhere", lambda sd: sd.update({"lm_head.weight": sd["lm_head.weight"].to(torch.float8_e4m3fn)}), "decoder projections only")]
    for name, mutate, match in cases:
        with pytest.raises(ValueError, match=match):
            list(iter_fp8_pairs(write(name, mutate)))


def test_quantization_config_rules():
    assert target_weights_fp8(None) is False
    assert target_weights_fp8({"load_in_8bit": True}) is False
    assert target_weights_fp8({"quant_method": "fp8"}) is True  # transformers' defaults: dynamic, 128 x 128
    assert target_weights_fp8({"quant_method": "fp8", "activation_scheme": "dynamic", "weight_block_size": [128, 128],
                               "modules_to_not_convert": ["lm_head"]}, 32) is True
    pytest.importorskip("transformers")
    from transformers import FineGrainedFP8Config
    assert target_weights_fp8(FineGrainedFP8Config(), 32) is True
    for bad, match in (({"activation_scheme": "static"}, "static"), ({"weight_block_size": [64, 64]}, "weight_block_size"),
                       ({"weight_block_size": None}, "weight_block_size"), ({"dequantize": True}, "dequantize"),
                       ({"modules_to_not_convert": ["up_proj"]}, "modules_to_not_convert"),
                       ({"modules_to_not_convert": ["model.layers.3.self_attn.q_proj"]}, "modules_to_not_convert")):
        with pytest.raises(ValueError, match=match):
            target_weights_fp8(dict({"quant_method": "fp8"}, **bad), 32)
    # the int8 switch keeps its contract
    with pytest.raises(ValueError, match="supported: load_in_8bit"):
        target_weights_int8({"quantization_config": {"quant_method": "fp8"}})


@pytest.fixture
def no_engine(monkeypatch):
    from eagle_b200 import EaModel

    def refuse(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(EaModel, "__init__", refuse)
    return EaModel


def test_from_pretrained_refusals_before_creating_an_engine(tmp_path, no_engine):
    EaModel = no_engine
    head = tmp_path / "head"
    head.mkdir()
    (head / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"]}))
    bf = tmp_path / "bf16"
    bf.mkdir()
    (bf / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"], "num_hidden_layers": 4}))
    common = dict(ea_model_path=str(head), torch_dtype=torch.bfloat16)
    for bad, match in (({"activation_scheme": "static"}, "static"), ({"weight_block_size": [128, 64]}, "weight_block_size"),
                       ({"weight_block_size": None}, "weight_block_size"), ({"dequantize": True}, "dequantize"),
                       ({"modules_to_not_convert": ["down_proj"]}, "modules_to_not_convert")):
        with pytest.raises(ValueError, match=match):
            EaModel.from_pretrained(base_model_path=str(bf), quantization_config=dict({"quant_method": "fp8"}, **bad), **common)
    with pytest.raises(ValueError, match="exclude each other"):
        EaModel.from_pretrained(base_model_path=str(bf), load_in_8bit=True, quantization_config={"quant_method": "fp8"}, **common)
    # stored FP8: load_in_8bit keeps its refusal, a 4-bit request stays "already quantized", a static checkpoint is refused
    d = tmp_path / "fp8"
    save_target_checkpoint(str(d), {"architectures": ["LlamaForCausalLM"], "num_hidden_layers": 1}, sd_small(), fp8=True)
    with pytest.raises(ValueError, match="unsupported quantization_config"):
        EaModel.from_pretrained(base_model_path=str(d), load_in_8bit=True, **common)
    with pytest.raises(ValueError, match="already quantized"):
        EaModel.from_pretrained(base_model_path=str(d), quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}, **common)
    cfg = json.load(open(d / "config.json"))
    cfg["quantization_config"]["activation_scheme"] = "static"
    (d / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="static"):
        EaModel.from_pretrained(base_model_path=str(d), **common)
    # an FP8 request on a checkpoint quantized otherwise
    d8 = tmp_path / "int8"
    d8.mkdir()
    (d8 / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"],
                                                "quantization_config": {"quant_method": "bitsandbytes", "load_in_8bit": True}}))
    with pytest.raises(ValueError, match="already quantized"):
        EaModel.from_pretrained(base_model_path=str(d8), quantization_config={"quant_method": "fp8"}, **common)
