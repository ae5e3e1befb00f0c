"""UniDepthV1 precision = "split" without a GPU: the packer (ConvNeXt and DINOv2 ViT-L encoders, the camera head's context
path) and the contract between the packer and the V1 engine's schedule (dry run: udb_v1_workspace_bytes).
tests/test_v1_split_gpu.py runs the mode on the GPU."""
import pytest
import torch

from test_v1_fp8_cpu import SMALL, _bytes, _model
from unidepth_b200._pack import split_weight

CPU = torch.device("cpu")
CASES = [("config_v1_cnvnxtl.json", SMALL), ("config_v1_cnvnxtl.json", None), ("config_v1_vitl14.json", None)]
IDS = ["small", "convnext_l", "vitl14"]


def _split_names(m):
    """Every operand the split packing stores as [N, 3K]."""
    s = m.spec
    names = [f"adapt.{l}.w_cam" for l in range(4)] + ["cam.inf.w1", "cam.inf.w2", "cam.agg.kv_w"]
    if m._engine_config().encoder == 1:
        names += ["patch_w"] + [f"blocks.{i}.{k}_w" for i in range(s.enc_depth) for k in ("qkv", "proj", "fc1", "fc2")]
    else:
        names += ["stem_w"] + [f"ds{i}.w" for i in range(1, 4)]
        names += [f"s{i}.b{j}.{k}" for i, d in enumerate(s.depths) for j in range(d) for k in ("w1", "w2")]
    return names


def _packs(cfg_name, arch, seed=None):
    m = _model(cfg_name, arch, seed=seed)
    T16, S16 = m._pack_tensors(CPU)
    m.precision = "split"
    T, S = m._pack_tensors(CPU)
    return m, T16, S16, T, S


@pytest.mark.parametrize("cfg_name,arch", CASES, ids=IDS)
def test_split_packer(cfg_name, arch):
    m, T16, S16, T, S = _packs(cfg_name, arch, seed=0 if arch else None)
    assert S == dict(S16, precision=1.0) and "precision" not in S16
    names = _split_names(m)
    assert set(T) == set(T16) | {f"adapt.{l}.w_cam" for l in range(4)}
    for n in names:
        w = T[n]
        ref = T16[n.replace("_cam", "")].float()
        N, K = ref.shape
        assert w.dtype == torch.float16 and tuple(w.shape) == (N, 3 * K), n
        hi, hi2, lo = w[:, :K], w[:, K:2 * K], w[:, 2 * K:]
        assert torch.equal(hi, hi2) and torch.equal(hi, T16[n.replace("_cam", "")]), n
    # hi + lo reconstructs the f32 weight to 2^-21 relative; lo is itself rounded to f16, so where it is subnormal (weights
    # below ~2^-3) the floor is half the f16 subnormal step, 2^-25
    sd = m.state_dict()
    srcs = {"cam.inf.w1": "pixel_decoder.camera_layer.in_features.proj1.weight",
            "cam.agg.kv_w": "pixel_decoder.camera_layer.aggregate.kv.weight",
            "adapt.3.w_cam": "pixel_decoder.input_adapter.input_adapters.3.1.weight"}
    srcs.update({"blocks.0.fc2_w": "pixel_encoder.blocks.0.mlp.fc2.weight"} if "patch_w" in names else
                {"s0.b0.w1": "pixel_encoder.stages.0.blocks.0.mlp.fc1.weight"})
    for n, src in srcs.items():
        w32 = sd[src].float()
        K = w32.shape[1]
        rec = T[n][:, :K].float() + T[n][:, 2 * K:].float()
        assert ((rec - w32).abs() <= 2.0 ** -21 * w32.abs() + 2.0 ** -25).all(), n
    # every operand that is not split is the f16 packing's, unchanged
    for k in T16:
        if k not in names:
            assert T[k].dtype == T16[k].dtype and torch.equal(T[k], T16[k]), k


def test_split_weight_layout():
    w = torch.randn(24, 64, dtype=torch.float64).float() * 3
    p = split_weight(w)
    assert tuple(p.shape) == (24, 192) and p.dtype == torch.float16
    assert torch.equal(p[:, :64], w.half()) and torch.equal(p[:, 64:128], w.half())
    assert torch.equal(p[:, 128:], (w - w.half().float()).half())


@pytest.mark.parametrize("cfg_name,arch", CASES, ids=IDS)
def test_schedule_accepts_exactly_the_split_operands(cfg_name, arch):
    m, T16, S16, T, S = _packs(cfg_name, arch)
    for B in (1, 4):
        for H, W in ((480, 640), (375, 1242), (1000, 400)):
            n, msg = _bytes(m, T, S, B, H, W)
            assert n > 0, msg
            # the f16 schedule is unchanged by the split operands being present
            n16, msg16 = _bytes(m, T16, S16, B, H, W)
            assert 0 < n16 < n, (n16, n, msg16)
    # dropping any split operand, or an operand next to one in the camera path, is reported by name
    names = _split_names(m)
    last = names[-1]
    for name in names[:7] + [names[7], last] + ["cam.agg.kv_b", "cam.inf.b2", "adapt.0.b"]:
        n, msg = _bytes(m, {k: v for k, v in T.items() if k != name}, S)
        assert n == 0 and name in msg, (name, msg)
    # an operand with the f16 layout in a split schedule is refused by name and shape
    for name in ("cam.inf.w2", "adapt.1.w_cam", names[8]):
        bad = dict(T)
        bad[name] = T16[name.replace("_cam", "")]
        n, msg = _bytes(m, bad, S)
        assert n == 0 and name in msg and "expected" in msg, (name, msg)
    # the f16 packing registered with precision 1 names the mode
    n, msg = _bytes(m, T16, dict(S16, precision=1.0))
    assert n == 0 and "precision 1" in msg and "split" in msg, msg
    # and a precision the V1 engine has no mode for is still refused
    n, msg = _bytes(m, T, dict(S, precision=3.0))
    assert n == 0 and "precision 3" in msg, msg


def test_unknown_precision_is_refused():
    m = _model("config_v1_cnvnxtl.json", SMALL)
    for bad in ("fp16", "bf16", "SPLIT"):
        m.precision = bad
        with pytest.raises(ValueError, match="precision must be 'split', 'f16' or 'fp8'"):
            m._pack_tensors(CPU)
    m.precision = "f16"
    key = m._fingerprint()
    m.precision = "split"
    assert m._fingerprint() != key and m._fingerprint()[0] == "split"
