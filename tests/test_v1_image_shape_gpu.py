"""UniDepthV1 at network shapes other than the config's (`model.image_shape`) on the GPU: the whole `infer` at each shape
of the reference goldens (tests/golden/v1_*_net*.npz) against those goldens and against the oracle at every pixel; a
change of shape and back in every precision mode against freshly built models; shapes the engine refuses."""
import copy
import json
import os

import pytest
import torch

from test_v1_image_shape_cpu import GOLDEN, SHAPE_CASES, oracle_infer, sampled, shape_case

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _model(cfg, sd, image_shape=None):
    from unidepth_b200 import UniDepthV1
    m = UniDepthV1(copy.deepcopy(cfg))
    m.load_state_dict(sd, strict=True)
    if image_shape is not None:
        m.image_shape = list(image_shape)
    return m.to("cuda:0").eval()


def _default_cfg(name):
    return json.load(open(os.path.join(GOLDEN, "config_v1_vitl14.json" if "vitl14" in name else "config_v1_cnvnxtl.json")))


# measured on an H100 80GB HBM3 (700 W power limit; the test prints them as V1SHAPEPARITY lines), asserted with a 1.5x
# margin: (depth ARel, depth max-rel, K rel), the larger of the sampled golden pixels and the oracle's full maps
V1SHAPE_MEASURED = {
    "v1_cnvnxtl_net384x512_480x640": (1.615e-4, 8.848e-4, 5.940e-5),
    "v1_cnvnxtl_net470x630_480x640": (1.596e-4, 8.754e-4, 2.431e-5),
    "v1_cnvnxtl_net470x630_gtK_375x1242": (1.369e-4, 6.279e-4, 1.173e-4),
    "v1_cnvnxtl_net448x448_480x640": (1.655e-4, 7.645e-4, 1.563e-4),
    "v1_vitl14_net378x504_480x640": (2.245e-4, 9.680e-4, 6.943e-5),
    "v1_vitl14_net518x686_480x640": (2.235e-4, 8.599e-4, 1.038e-4),
    "v1_vitl14_net518x686_gtK_375x1242": (4.039e-4, 1.107e-3, 1.067e-4),
    "v1_vitl14_net448x448_480x640": (1.748e-4, 8.285e-4, 1.131e-4),
}


def _check(out, ref, meta, name, label, sample):
    key = (lambda t, k: sampled(t, k, meta)) if sample else (lambda t, k: t)
    d, dr = key(out["depth"].float().cpu(), "depth"), ref["depth"]
    rel = (d - dr).abs() / dr
    k, kr = out["intrinsics"].cpu(), ref["intrinsics"]
    kerr = max(((k[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    pts, pr = key(out["points"].float().cpu(), "points"), ref["points"]
    perr = ((pts - pr).abs() / pr.abs().clamp(min=0.1 * pr.abs().mean())).mean().item()
    print(f"V1SHAPEPARITY {label} {name}: depth ARel {rel.mean().item():.3e} max {rel.max().item():.3e}; intrinsics rel "
          f"{kerr:.3e}; points mean rel {perr:.3e}")
    m = V1SHAPE_MEASURED[name]
    assert rel.mean().item() < 1e-3
    assert rel.mean().item() < 1.5 * m[0] and rel.max().item() < 1.5 * m[1] and kerr < 1.5 * m[2], (name, label, rel.mean().item(),
                                                                                                    rel.max().item(), kerr)
    assert perr < 5e-3


@pytest.mark.parametrize("name", SHAPE_CASES)
def test_infer_at_network_shape_against_reference(name):
    _dev()
    cfg, sd, rgb, K, meta, z = shape_case(name)
    m = _model(_default_cfg(name), sd, meta["image_shape"])     # the config's shape, then the attribute the user sets
    out = m.infer(rgb, K)
    assert tuple(out["depth"].shape[-2:]) == tuple(meta["shape"][1:])
    golden = {k: torch.from_numpy(z[k]) for k in ("depth", "intrinsics", "points")}
    _check(out, golden, meta, name, "golden", sample=True)
    ref = oracle_infer(name, sd, cfg, rgb, K)
    _check(out, ref, meta, name, "full_resolution_oracle", sample=False)
    m.use_cuda_graph = False
    eager = m.infer(rgb, K)
    assert all(torch.equal(eager[k], out[k]) for k in out)


def _synthetic(cfg_name):
    cfg = json.load(open(os.path.join(GOLDEN, cfg_name)))
    if "vitl14" in cfg_name:
        from unidepth_v1_vit_oracle import make_v1_vit_state_dict
        return cfg, make_v1_vit_state_dict(cfg, 0)
    from fixture import make_v1_state_dict
    return cfg, make_v1_state_dict(cfg, 0)


@pytest.mark.parametrize("precision", ["f16", "split", "fp8"])
@pytest.mark.parametrize("cfg_name,new_shape", [("config_v1_cnvnxtl.json", (470, 630)), ("config_v1_vitl14.json", (378, 504))])
def test_shape_change_and_back_in_every_precision(cfg_name, new_shape, precision):
    """default shape -> new shape -> default: at the new shape the outputs are those of a model built with that
    image_shape in its config, back at the default those of its own first call; the weights are not repacked."""
    _dev()
    cfg, sd = _synthetic(cfg_name)
    g = torch.Generator().manual_seed(11)
    rgb = torch.randint(0, 256, (2, 3, 480, 640), dtype=torch.uint8, generator=g).cuda()
    m = _model(cfg, sd)
    m.precision = precision
    first = m.infer(rgb)
    packed = m._packed[0]
    ptrs = {k: t.data_ptr() for k, t in packed.items()}
    m.image_shape = list(new_shape)
    at_new = m.infer(rgb)
    assert m._packed[0] is packed and all(t.data_ptr() == ptrs[k] for k, t in packed.items())
    assert "tokens_pos" not in packed and "pos" not in packed
    fresh_cfg = copy.deepcopy(cfg)
    fresh_cfg["data"]["image_shape"] = list(new_shape)
    fresh = _model(fresh_cfg, sd)
    fresh.precision = precision
    want = fresh.infer(rgb)
    del fresh
    assert all(torch.equal(at_new[k], want[k]) for k in want), precision
    assert not torch.equal(at_new["depth"], first["depth"])
    m.image_shape = list(cfg["data"]["image_shape"])
    back = m.infer(rgb)
    assert all(torch.equal(back[k], first[k]) for k in first), precision
    assert m._packed[0] is packed and all(t.data_ptr() == ptrs[k] for k, t in packed.items())


@pytest.mark.parametrize("bad,exc,text", [([64, 64], NotImplementedError, "Nystrom"), ([616, 462], NotImplementedError, "portrait"),
                                          ([32, 640], ValueError, "at least 64")])
def test_refused_shape_launches_nothing_and_keeps_the_previous_engine(bad, exc, text):
    _dev()
    from unidepth_b200 import _cabi
    cfg, sd = _synthetic("config_v1_cnvnxtl.json")
    g = torch.Generator().manual_seed(12)
    rgb = torch.randint(0, 256, (1, 3, 480, 640), dtype=torch.uint8, generator=g).cuda()
    m = _model(cfg, sd)
    first = m.infer(rgb)
    engine = m._engine
    m.image_shape = bad
    torch.cuda.synchronize()
    n0 = _cabi.launch_count()
    with pytest.raises(exc, match=text):
        m.infer(rgb)
    torch.cuda.synchronize()
    assert _cabi.launch_count() == n0
    assert m._engine is engine
    m.image_shape = list(cfg["data"]["image_shape"])
    again = m.infer(rgb)
    assert m._engine is engine and all(torch.equal(again[k], first[k]) for k in first)
