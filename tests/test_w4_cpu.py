"""4-bit target weights without a GPU: the code tables, the quantizer / dequantizer rules, double-quantized absmax, the
bitsandbytes 4-bit checkpoint round trip and the refusals, all raised before an engine is created."""
import json
import os
import struct

import pytest
import torch

from eagle_b200 import quant
from eagle_b200.checkpoint import iter_4bit_triples, save_target_checkpoint, target_weights_4bit, target_weights_int8

# fp32 bit patterns of the tables (bitsandbytes' dDequantizeNF4 / dDequantizeFP4Tree constants)
NF4_BITS = [0xBF800000, 0xBF3239B1, 0xBF066B30, 0xBECA32A0, 0xBE91A24D, 0xBE3D353F, 0xBDBA7871, 0x00000000,
            0x3DA2FAFF, 0x3E24CAE3, 0x3E7C04DD, 0x3EAD033A, 0x3EE1A4B8, 0x3F1007AB, 0x3F3913B3, 0x3F800000]
FP4_BITS = [0x00000000, 0x3BAAAAAB, 0x3F2AAAAB, 0x3F800000, 0x3EAAAAAB, 0x3F000000, 0x3E2AAAAB, 0x3E800000]


def bits(t):
    return [struct.unpack("<I", struct.pack("<f", float(v)))[0] for v in t]


def test_code_table_bit_patterns():
    assert bits(quant.code_table("nf4")) == NF4_BITS
    fp4 = quant.code_table("fp4")
    assert bits(fp4[:8]) == FP4_BITS
    assert bits(fp4[8:]) == [b | 0x80000000 for b in FP4_BITS]  # code 8 is -0.0
    with pytest.raises(ValueError, match="quant_type"):
        quant.code_table("int4")


def test_pack_order_element_2j_in_the_high_nibble():
    # a block whose values are the table entries themselves, in code order: the codes are 0..15 and pack as 0x01, 0x23, ...
    table = quant.code_table("nf4")
    w = torch.cat([table, table.flip(0), table, table]).view(1, 64)
    packed, absmax = quant.quantize_4bit(w, "nf4")
    assert float(absmax[0, 0]) == 1.0
    assert packed[0, :8].tolist() == [0x01, 0x23, 0x45, 0x67, 0x89, 0xAB, 0xCD, 0xEF]
    assert packed[0, 8:16].tolist() == [0xFE, 0xDC, 0xBA, 0x98, 0x76, 0x54, 0x32, 0x10]
    assert quant.unpack_4bit(packed)[0, :16].tolist() == list(range(16))


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
def test_absmax_and_the_midpoint_rule(qt):
    g = torch.Generator().manual_seed(4)
    w = torch.randn(6, 128, generator=g)
    packed, absmax = quant.quantize_4bit(w, qt)
    assert torch.equal(absmax, w.abs().reshape(-1, 64).amax(1).reshape(6, 2))
    # nearest entry: no other table entry is strictly closer to the normalised value than the chosen one
    table = quant.code_table(qt).double()
    x = (w.reshape(-1, 64) * (1.0 / absmax.reshape(-1))[:, None]).reshape(6, 128).double()
    chosen = table[quant.unpack_4bit(packed)]
    assert bool(((x[..., None] - table).abs().min(-1).values == (x - chosen).abs()).all())
    # exact midpoints between neighbouring entries go to the lower entry (x must exceed a midpoint to move up)
    pos = table[:8].sort().values if qt == "fp4" else table.sort().values
    mids64 = (pos[1:] + pos[:-1]) / 2
    exact = mids64.float().double() == mids64  # the midpoints an fp32 value can hit
    assert int(exact.sum()) >= 1
    lower, mids = pos[:-1][exact], mids64[exact].float()
    w = torch.zeros(1, 64)
    w[0, 0] = 1.0  # absmax 1: the other values are taken as they are
    n = mids.numel()
    w[0, 1: 1 + n] = mids
    w[0, 1 + n: 1 + 2 * n] = torch.nextafter(mids, torch.full_like(mids, 2.0))  # one ulp above: the upper entry
    codes = quant.unpack_4bit(quant.quantize_4bit(w, qt)[0])[0]
    assert table[codes[1: 1 + n]].tolist() == lower.tolist()
    assert table[codes[1 + n: 1 + 2 * n]].tolist() == pos[1:][exact].tolist()


def test_fp4_sign_and_negative_zero():
    w = torch.zeros(1, 64)
    w[0, 0] = -1.0
    w[0, 1] = -1e-6  # rounds to magnitude 0 with the sign bit set: code 8, which dequantizes to -0.0
    w[0, 2] = 0.25
    packed, absmax = quant.quantize_4bit(w, "fp4")
    codes = quant.unpack_4bit(packed)[0]
    assert codes[:3].tolist() == [11, 8, 7] and codes[3:].eq(0).all()
    d = quant.dequantize_4bit(packed, absmax, "fp4", torch.bfloat16)
    assert d[0, 1].view(torch.int16).item() == torch.tensor(-0.0, dtype=torch.bfloat16).view(torch.int16).item()
    assert d[0, 3].view(torch.int16).item() == 0  # +0.0


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
def test_all_zero_blocks_dequantize_to_zero(qt):
    w = torch.randn(2, 128)
    w[1, 64:] = 0
    packed, absmax = quant.quantize_4bit(w, qt)
    assert float(absmax[1, 1]) == 0.0
    d = quant.dequantize_4bit(packed, absmax, qt, torch.float16)
    assert float(d[1, 64:].float().abs().max()) == 0.0


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_dequantizer_is_the_literal_formula(qt, dtype):
    g = torch.Generator().manual_seed(9)
    packed = torch.randint(0, 256, (5, 64), generator=g, dtype=torch.uint8)
    absmax = torch.rand(5, 2, generator=g) * 0.1
    absmax[0, 0] = 1e-40  # subnormal
    table = quant.code_table(qt).tolist()
    d = quant.dequantize_4bit(packed, absmax, qt, dtype)
    for r in range(5):
        for k in range(0, 128, 7):
            byte = int(packed[r, k // 2])
            code = byte >> 4 if k % 2 == 0 else byte & 15
            want = (torch.tensor(table[code], dtype=torch.float32) * absmax[r, k // 64]).to(dtype)
            assert d[r, k].view(torch.int16) == want.view(torch.int16), (r, k)


def test_nested_absmax_two_roundings():
    g = torch.Generator().manual_seed(3)
    a = torch.randint(0, 256, (600,), generator=g, dtype=torch.uint8)
    nested = torch.rand(3, generator=g)
    qmap = torch.randn(256, generator=g)
    offset = 0.0123456789
    out = quant.decompress_nested_absmax(a, nested, qmap, 256, offset)
    for i in range(0, 600, 13):
        prod = torch.tensor(float(qmap[int(a[i])]) * float(nested[i // 256]), dtype=torch.float64).float()  # first fp32 rounding
        want = (prod.double() + torch.tensor(offset, dtype=torch.float32).double()).float()                # second
        assert out[i].view(torch.int32) == want.view(torch.int32), i


def sd_small(dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(12)
    sd = {f"model.layers.0.{p}.weight": (torch.randn(128, 192 if "down" in p else 128, generator=g) * 0.02).to(dtype) for p in quant.PROJECTIONS}
    sd["lm_head.weight"] = torch.randn(32, 128, generator=g).to(dtype)
    sd["model.norm.weight"] = torch.ones(128, dtype=dtype)
    return sd


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("dq", [False, True])
def test_checkpoint_round_trip(tmp_path, qt, dq):
    sd = sd_small()
    d = str(tmp_path / "t4")
    save_target_checkpoint(d, {"hidden_size": 128, "torch_dtype": "bfloat16"}, sd, load_in_4bit=qt, double_quant=dq)
    cfg = json.load(open(os.path.join(d, "config.json")))
    assert target_weights_4bit(cfg["quantization_config"], torch.bfloat16, pre_quantized=True) == qt
    got = {k: (v, a) for k, v, a in iter_4bit_triples(d, qt, torch.bfloat16)}
    assert set(got) == set(sd)
    for k, w in sd.items():
        v, a = got[k]
        if not quant.is_target_projection(k):
            assert a is None and torch.equal(v, w)
            continue
        packed, absmax = quant.quantize_4bit(w, qt)
        assert torch.equal(v, packed)
        if dq:  # decompressed: close to the true absmax, not equal
            assert a.dtype == torch.float32 and a.shape == absmax.shape
            assert float((a - absmax).abs().max()) <= float(absmax.max()) / 50
        else:
            assert torch.equal(a, absmax)


def _write(tmp_path, name, mutate):
    d = str(tmp_path / name)
    save_target_checkpoint(d, {"hidden_size": 128, "torch_dtype": "bfloat16"}, sd_small(), load_in_4bit="nf4")
    from safetensors.torch import load_file, save_file
    p = os.path.join(d, "model.safetensors")
    sd = load_file(p)
    mutate(sd)
    save_file(sd, p)
    return d


def _state_edit(**kw):
    def f(sd):
        for k in [k for k in sd if "quant_state" in k]:
            st = json.loads(bytes(sd[k].tolist()).decode())
            st.update(kw)
            sd[k] = torch.tensor(list(json.dumps(st).encode()), dtype=torch.uint8)
    return f


def test_stored_4bit_refusals(tmp_path):
    cases = [("blocksize", _state_edit(blocksize=128), "blocksize 128"),
             ("dtype", _state_edit(dtype="float16"), "stored dtype"),
             ("shape", _state_edit(shape=[256, 96]), "multiple of 64"),
             ("qmap", lambda sd: sd.update({k: v * 1.0001 for k, v in sd.items() if k.endswith("quant_map")}), "quant_map differs"),
             ("qtype", _state_edit(quant_type="fp4"), "quant_type")]
    for name, mutate, match in cases:
        d = _write(tmp_path, name, mutate)
        with pytest.raises(ValueError, match=match):
            list(iter_4bit_triples(d, "nf4", torch.bfloat16))


def test_quantization_config_rules():
    bf = torch.bfloat16
    assert target_weights_4bit(None, bf) is None
    assert target_weights_4bit({"load_in_8bit": True}, bf) is None
    assert target_weights_4bit({"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}, bf) == "nf4"
    assert target_weights_4bit({"load_in_4bit": True}, bf) == "fp4"  # transformers' default quant type
    for compute in (None, "float32", torch.float32, "bfloat16", torch.bfloat16):
        assert target_weights_4bit({"load_in_4bit": True, "bnb_4bit_quant_type": "fp4", "bnb_4bit_compute_dtype": compute}, bf) == "fp4"

    class Cfg:  # a BitsAndBytesConfig stand-in: anything with to_dict()
        def to_dict(self):
            return {"load_in_4bit": True, "bnb_4bit_quant_type": "nf4", "bnb_4bit_quant_storage": "uint8"}

    assert target_weights_4bit(Cfg(), bf) == "nf4"
    for bad, match in (({"bnb_4bit_quant_type": "int4"}, "quant_type"), ({"bnb_4bit_compute_dtype": torch.float16}, "compute_dtype"),
                       ({"bnb_4bit_quant_storage": "bfloat16"}, "quant_storage"), ({"bnb_4bit_use_double_quant": True}, "double_quant"),
                       ({"quant_method": "gptq"}, "bitsandbytes")):
        with pytest.raises(ValueError, match=match):
            target_weights_4bit(dict({"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}, **bad), bf)
    assert target_weights_4bit({"load_in_4bit": True, "bnb_4bit_quant_type": "nf4", "bnb_4bit_use_double_quant": True}, bf,
                               pre_quantized=True) == "nf4"
    # the int8 switch keeps its contract: every 4-bit request is refused there
    with pytest.raises(ValueError, match="supported: load_in_8bit"):
        target_weights_int8({"quantization_config": {"quant_method": "bitsandbytes", "load_in_4bit": True}})


def test_quantizer_refuses_ragged_rows():
    with pytest.raises(ValueError, match="multiple of the blocksize"):
        quant.quantize_4bit(torch.randn(4, 96), "nf4")


def test_from_pretrained_4bit_refusals_before_creating_an_engine(tmp_path, monkeypatch):
    from eagle_b200 import EaModel

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(EaModel, "__init__", no_engine)
    with pytest.raises(ValueError, match="BitsAndBytesConfig"):
        EaModel.from_pretrained(base_model_path=str(tmp_path), ea_model_path=str(tmp_path), load_in_4bit=True)
    d = tmp_path / "bf16"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"]}))
    for bad, match in (({"bnb_4bit_quant_type": "int4"}, "quant_type"), ({"bnb_4bit_compute_dtype": "float16"}, "compute_dtype"),
                       ({"bnb_4bit_quant_storage": "float32"}, "quant_storage"), ({"bnb_4bit_use_double_quant": True}, "double_quant")):
        qc = dict({"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}, **bad)
        with pytest.raises(ValueError, match=match):
            EaModel.from_pretrained(base_model_path=str(d), ea_model_path=str(d), torch_dtype=torch.bfloat16, quantization_config=qc)
    for name, mutate, match in (("blocksize", _state_edit(blocksize=128), "blocksize 128"), ("dtype", _state_edit(dtype="float16"), "stored dtype"),
                                ("qmap", lambda sd: sd.update({k: -v for k, v in sd.items() if k.endswith("quant_map")}), "quant_map differs"),
                                ("shape", _state_edit(shape=[256, 96]), "multiple of 64")):
        t = _write(tmp_path, "fp_" + name, mutate)
        with open(os.path.join(t, "config.json")) as f:
            cfg = json.load(f)
        cfg["architectures"] = ["LlamaForCausalLM"]
        with open(os.path.join(t, "config.json"), "w") as f:
            json.dump(cfg, f)
        monkeypatch.setattr(EaModel, "__init__", no_engine)
        with pytest.raises(ValueError, match=match):
            EaModel.from_pretrained(base_model_path=t, ea_model_path=str(d), torch_dtype=torch.bfloat16)


def test_stored_4bit_size_mismatch_is_refused(tmp_path):
    trunc = lambda sd: sd.update({k: v[:-1].contiguous() for k, v in sd.items()  # noqa: E731
                                  if k.endswith("down_proj.weight.absmax")})
    d = _write(tmp_path, "trunc_absmax", trunc)
    with pytest.raises(ValueError, match="absmax values"):
        list(iter_4bit_triples(d, "nf4", torch.bfloat16))
    d = _write(tmp_path, "trunc_weight", lambda sd: sd.update({k: v[:-2].contiguous() for k, v in sd.items() if k.endswith("q_proj.weight")}))
    with pytest.raises(ValueError, match="packed bytes"):
        list(iter_4bit_triples(d, "nf4", torch.bfloat16))


def test_from_pretrained_refuses_conflicting_quantization_requests(tmp_path, monkeypatch):
    from eagle_b200 import EaModel

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(EaModel, "__init__", no_engine)
    head = tmp_path / "head"
    head.mkdir()
    (head / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"]}))
    d = str(tmp_path / "nf4")
    save_target_checkpoint(d, {"architectures": ["LlamaForCausalLM"], "hidden_size": 128, "torch_dtype": "bfloat16"}, sd_small(),
                           load_in_4bit="nf4")
    common = dict(base_model_path=d, ea_model_path=str(head), torch_dtype=torch.bfloat16)
    for kw, match in ((dict(load_in_8bit=True), "conflicts"), (dict(quantization_config={"load_in_8bit": True}), "conflicts"),
                      (dict(quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "fp4"}), "fp4 conflicts")):
        with pytest.raises(ValueError, match=match):
            EaModel.from_pretrained(**common, **kw)
    d8 = tmp_path / "int8"
    d8.mkdir()
    (d8 / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"],
                                                "quantization_config": {"quant_method": "bitsandbytes", "load_in_8bit": True}}))
    with pytest.raises(ValueError, match="already quantized"):
        EaModel.from_pretrained(base_model_path=str(d8), ea_model_path=str(head), torch_dtype=torch.bfloat16,
                                quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"})
    bf = tmp_path / "bf16"
    bf.mkdir()
    (bf / "config.json").write_text(json.dumps({"architectures": ["LlamaForCausalLM"]}))
    with pytest.raises(ValueError, match="exclude each other"):
        EaModel.from_pretrained(base_model_path=str(bf), ea_model_path=str(head), torch_dtype=torch.bfloat16, load_in_8bit=True,
                                quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"})
