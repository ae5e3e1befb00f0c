"""The GEMM's TMA-store epilogue against its general epilogue (unidepth_b200/csrc/gemm.cu).

Plain ROWS stores with an identity row map take the TMA epilogue; UDB_GEMM_TMA_EPILOGUE=0 sends the same call through
the general one.  Both run the same per-element arithmetic in the same order, so every output must be bit-identical,
and the NaN canaries around the written region must survive both.  Calls outside the TMA epilogue's conditions must
keep taking the general epilogue."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

f16, f32 = torch.float16, torch.float32
PATTERN = {f32: (torch.int32, 0x7FC0DEAD), f16: (torch.int16, 0x7E5A)}   # quiet NaNs with a recognisable payload
ENV = "UDB_GEMM_TMA_EPILOGUE"


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _ops():
    from unidepth_b200 import ops
    return ops


def _used():
    from unidepth_b200 import _cabi
    return _cabi.lib().udb_gemm_tma_epilogue_used()


def sentinel(shape, dtype, dev):
    it, pat = PATTERN[dtype]
    return torch.full(shape, pat, dtype=it, device=dev).view(dtype)


def bits(t):
    return t.view(PATTERN[t.dtype][0])


def on_path(tma, fn):
    """fn() with the TMA epilogue allowed (tma) or switched off; returns fn's result and whether it was used"""
    old = os.environ.get(ENV)
    os.environ[ENV] = "1" if tma else "0"
    try:
        r = fn()
        torch.cuda.synchronize()
        return r, _used()
    finally:
        if old is None:
            del os.environ[ENV]
        else:
            os.environ[ENV] = old


def compare(M, N, K, *, bias, act, gamma, resid_mode, out32, seed, col0=None, extra_cols=40):
    """Run one GEMM on both paths into NaN-filled buffers (1 row above, 2 below, col0 columns left, the rest right of the
    written [M, N] region) and require bit-identical buffers and untouched canaries.  resid_mode: None, "separate"
    (f32 column slice of another buffer) or "inplace" (resid is out)."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(seed)
    odt = f32 if out32 else f16
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(dev)
    b = torch.randn(N, generator=g).to(dev) if bias else None
    gm = (torch.rand(N, generator=g) + 0.5).to(dev) if gamma else None
    r0 = torch.randn(M, N + 8, generator=g).to(dev)[:, 4:4 + N] if resid_mode else None
    if col0 is None:
        col0 = 4 if out32 else 8                 # a 16-byte aligned column slice, ldc > N
    shape = (M + 3, col0 + N + extra_cols)

    def run():
        buf = sentinel(shape, odt, dev)
        out = buf[1:1 + M, col0:col0 + N]
        resid = r0
        if resid_mode == "inplace":
            out.copy_(r0)
            resid = out
        ops.gemm(a, w, bias=b, act=act, gamma=gm, resid=resid, out=out)
        return buf

    old, used_old = on_path(False, run)
    new, used_new = on_path(True, run)
    assert used_old == 0
    name = f"M{M} N{N} K{K} {'f32' if out32 else 'f16'} resid={resid_mode}"
    mask = torch.zeros(shape, dtype=torch.bool, device=dev)
    mask[1:1 + M, col0:col0 + N] = True
    it, pat = PATTERN[odt]
    for buf, tag in ((old, "general"), (new, "tma")):
        bad = (bits(buf)[~mask] != pat).sum().item()
        assert bad == 0, f"{name} {tag}: {bad} canary cells were modified"
    diff = (bits(old) != bits(new)).sum().item()
    assert diff == 0, f"{name}: {diff} cells differ between the general and the TMA epilogue"
    return used_new


# The encoder's four GEMMs at the flagship shape (ViT-L/14, 8 images of 480x640: 8 x 1611 tokens) with their epilogues
ENCODER = {
    "qkv": dict(N=3072, K=1024, bias=True, act="none", gamma=False, resid_mode=None, out32=False),
    "proj": dict(N=1024, K=1024, bias=True, act="none", gamma=True, resid_mode="inplace", out32=True),
    "fc1": dict(N=4096, K=1024, bias=True, act="gelu", gamma=False, resid_mode=None, out32=False),
    "fc2": dict(N=1024, K=4096, bias=True, act="none", gamma=True, resid_mode="inplace", out32=True),
}


def _act(name):
    ops = _ops()
    return {"none": ops.ACT_NONE, "gelu": ops.ACT_GELU, "leaky": ops.ACT_LEAKY}[name]


@pytest.mark.parametrize("which", sorted(ENCODER))
def test_encoder_gemms(which):
    c = dict(ENCODER[which])
    c["act"] = _act(c["act"])
    assert compare(12888, seed=len(which), col0=0, extra_cols=0, **c) == 1


NS = [256, 192, 128, 64, 32]                     # one N per tile width
MS = [1, 127, 129, 12888]
KS = [64, 1024, 4096]
EPIS = [("bias", "none", False, None), ("bias", "gelu", False, None), ("bias", "leaky", True, "separate"),
        ("bias", "none", True, "inplace"), (None, "none", False, None)]
CASES = [(N, M, KS[(i + j) % len(KS)], EPIS[(i + 2 * j) % len(EPIS)], (i + j) % 2 == 0)
         for i, N in enumerate(NS) for j, M in enumerate(MS)]


@pytest.mark.parametrize("N,M,K,epi,out32", CASES)
def test_matches_general_epilogue(N, M, K, epi, out32):
    bias, act, gamma, resid_mode = epi
    if resid_mode and not out32:
        resid_mode = None        # a residual takes the TMA epilogue only with an f32 out (test_general_path_kept)
    used = compare(M, N, K, bias=bias is not None, act=_act(act), gamma=gamma, resid_mode=resid_mode, out32=out32,
                   seed=N * 131 + M * 7 + K)
    assert used == 1


@pytest.mark.parametrize("out32", [False, True])
def test_every_residual_mode(out32):
    for resid_mode in (None, "separate", "inplace") if out32 else (None,):
        for K in KS:
            assert compare(129, 256, K, bias=True, act=_act("gelu"), gamma=True, resid_mode=resid_mode, out32=out32,
                           seed=K) == 1


def test_general_path_kept():
    """Calls outside the TMA epilogue's conditions still run (and pass) on the general epilogue."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(3)
    M, N, K = 257, 256, 128
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    r32 = torch.randn(M, N, generator=g).to(dev)
    big16 = torch.empty(M, N + 16, dtype=f16, device=dev)
    big32 = torch.empty(M, N + 8, dtype=f32, device=dev)

    def path(**kw):
        (_, used) = on_path(True, lambda: ops.gemm(a, w, bias=bias, **kw))
        return used

    assert path() == 1                                                    # plain f16 out: eligible
    assert path(out=big32[:, 4:4 + N]) == 1                               # 16-byte aligned f32 slice, ldc > N
    assert path(out=big16[:, :N], out2=torch.empty(M, N, dtype=f16, device=dev)) == 0             # second output
    assert path(out_split=True) == 0                                                              # split-f16 output
    assert path(out=torch.empty(2 * M, N, dtype=f16, device=dev), rows_per_group=64, group_stride=128) == 0  # row map
    assert path(resid=r32[:4], resid_mod=4, out_dtype=f32) == 0                                   # residual row map
    assert path(resid=r32.half()) == 0                                                            # f16 residual
    assert path(resid=r32) == 0                                                                   # f32 resid, f16 out
    assert path(out=big16[:, 4:4 + N]) == 0                                                       # 8-byte aligned out
    assert path(out=torch.empty(M, N + 4, dtype=f16, device=dev)[:, :N]) == 0                     # f16 pitch % 16 B != 0
    assert path(out=big32[:, 4:4 + N], resid=r32) == 1                                            # f32 resid, f32 out
    stats = torch.empty(M, 2, 2, dtype=f32, device=dev)
    assert path(out=big32[:, 4:4 + N], ln_stats_out=stats, ln_parts=2, ln_part_cols=128) == 0     # fused LayerNorm
    os.environ[ENV] = "0"
    try:
        ops.gemm(a, w, bias=bias)
        assert _used() == 0                                                                       # switched off
    finally:
        del os.environ[ENV]
