"""Host-side layout checks of udb_gemm_f16, udb_attention_f16 and udb_conv3x3_halo_f16 (include/udb.h).

Every call runs in a fresh interpreter with CUDA_VISIBLE_DEVICES="" and plain integers as fake device pointers, so no
kernel can launch even on a machine with a GPU, even if a check were missing or came after the first CUDA call.  For each
rejected layout the test asserts that the call fails, that udb_last_error() names the offending argument and that
udb_launch_count() did not move.  A valid call with the same fake pointers must get past the checks and fail later, at
the tensor-map or driver step, with a different message: the checks are not over-strict."""
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BASE = 1 << 28          # fake device addresses, 1 KB aligned
P = {name: BASE + i * (1 << 22) for i, name in enumerate(
    ("a", "w", "out", "out2", "resid", "bias", "gamma", "ln_c1", "head_w", "stats", "q", "k", "v", "x"))}

GEMM = {"a": P["a"], "w": P["w"], "M": 256, "N": 128, "K": 64, "lda": 64, "ldw": 64, "a_mode": 0,
        "bias": P["bias"], "out": P["out"], "out_f32": 1, "ldc": 128, "store_mode": 0}
GEMM_RES = dict(GEMM, resid=P["resid"], resid_f32=1, ldr=128)
GEMM_F16 = dict(GEMM, out_f32=0, out2=P["out2"])
CONV = dict(GEMM, M=2 * 30 * 40, N=64, K=9 * 64, lda=64, ldw=9 * 64, a_mode=1, conv_B=2, conv_H=30, conv_W=40, conv_C=64,
            conv_inH=30, conv_inW=40, conv_off=-1, conv_TH=8, conv_TW=16, conv_cstride=64, ldc=64, store_mode=2)
CONV_PRE = dict(CONV, conv_inH=32, conv_inW=42, conv_off=0)
HEAD = dict(CONV_PRE, N=32, store_mode=3, ldc=1, head_w=P["head_w"])
CONVT = dict(GEMM, M=2 * 9 * 13, N=4 * 32, K=128, lda=128, ldw=128, store_mode=1, ldc=32, ct_k=2, ct_cout=32, ct_h=9, ct_w=13,
             ct_pad=1, resid=P["resid"], resid_f32=1)
ATTN = {"q": P["q"], "k": P["k"], "v": P["v"], "out": P["out"], "B": 2, "heads": 2, "seq_q": 256, "seq_k": 256, "head_dim": 64,
        "ldq": 128, "ldk": 128, "ldv": 128, "ldo": 128, "scale": 0.125}
ATTN_SPLIT = dict(ATTN, ldq=256, ldk=256, ldv=256, ldo=256, split=1, lo_off_q=128, lo_off_k=128, lo_off_v=128, lo_off_o=128)
HALO = {"x": P["x"], "w": P["w"], "bias": P["bias"], "B": 1, "H": 32, "W": 32, "C": 64, "cstride": 128, "coff": 64, "cout": 64,
        "out": P["out"], "ldc": 64}
HALO_HEAD = dict(HALO, cout=32, out=0, ldc=0, head_w=P["head_w"], head_out=P["out"])

# valid calls: they must pass every layout check (and then fail without a device)
VALID = {
    "gemm": ("gemm", GEMM), "gemm_resid": ("gemm", GEMM_RES), "gemm_f16_out2": ("gemm", GEMM_F16),
    "gemm_split_out": ("gemm", dict(GEMM_F16, ldc=256, out_split=128)),
    "gemm_column_slice": ("gemm", dict(GEMM, out=P["out"] + 16, ldc=200)),
    "gemm_row_map": ("gemm", dict(GEMM_RES, rows_per_group=100, group_stride=101, row_offset=1, resid_mod=100, resid_row_offset=1)),
    "gemm_rows_just_below_2^32": ("gemm", dict(GEMM, M=1 << 20, ldc=4096)),
    "conv": ("gemm", CONV), "conv_prepadded": ("gemm", CONV_PRE), "conv_head": ("gemm", HEAD), "convt": ("gemm", CONVT),
    "attn": ("attn", ATTN), "attn_split": ("attn", ATTN_SPLIT),
    "attn_slices": ("attn", dict(ATTN, ldq=192, q_col0=64, ldo=200, o_col0=2)),
    "halo": ("halo", HALO), "halo_head": ("halo", HALO_HEAD), "halo_column_slice": ("halo", dict(HALO, out=P["out"] + 4, ldc=66)),
}

# rejected layouts: (which call, struct fields, regexes the error message must match)
REJECT = {
    # --- GEMM
    "gemm_M0": ("gemm", dict(GEMM, M=0), [r"M=0", r">= 1"]),
    "gemm_N0": ("gemm", dict(GEMM, N=0), [r"N=0", r">= 1"]),
    "gemm_K0": ("gemm", dict(GEMM, K=0), [r"K=0", r">= 1"]),
    "gemm_out_f32_misaligned": ("gemm", dict(GEMM, out=P["out"] + 8), [r"`out`", r"16-byte"]),
    "gemm_out_f16_misaligned": ("gemm", dict(GEMM_F16, out=P["out"] + 4), [r"`out`", r"8-byte"]),
    "gemm_out2_misaligned": ("gemm", dict(GEMM_F16, out2=P["out2"] + 2), [r"`out2`"]),
    "gemm_resid_f32_misaligned": ("gemm", dict(GEMM_RES, resid=P["resid"] + 8), [r"`resid`", r"16-byte"]),
    "gemm_resid_f16_misaligned": ("gemm", dict(GEMM_RES, resid=P["resid"] + 2, resid_f32=0), [r"`resid`", r"8-byte"]),
    "gemm_bias_misaligned": ("gemm", dict(GEMM, bias=P["bias"] + 4), [r"`bias`"]),
    "gemm_gamma_misaligned": ("gemm", dict(GEMM, gamma=P["gamma"] + 8), [r"`gamma`"]),
    "gemm_ln_c1_misaligned": ("gemm", dict(GEMM, ln_stats_in=P["stats"], ln_c1=P["ln_c1"] + 4, ln_parts=1, ln_part_cols=64),
                              [r"`ln_c1`"]),
    "gemm_head_w_misaligned": ("gemm", dict(HEAD, head_w=P["head_w"] + 4), [r"`head_w`"]),
    "gemm_ldc_not_mult4": ("gemm", dict(GEMM, ldc=130), [r"`ldc`", r"multiple of 4"]),
    "gemm_ldr_not_mult4": ("gemm", dict(GEMM_RES, ldr=130), [r"`ldr`", r"multiple of 4"]),
    "gemm_ldc_below_N": ("gemm", dict(GEMM, ldc=64), [r"`ldc`", r"overlap"]),
    "gemm_ldc_below_N_plus_split": ("gemm", dict(GEMM_F16, ldc=128, out_split=128), [r"`ldc`", r"out_split"]),
    "gemm_ldr_below_N": ("gemm", dict(GEMM_RES, ldr=64), [r"`ldr`", r"overlap"]),
    "gemm_conv_ldc_below_N": ("gemm", dict(CONV, ldc=32), [r"`ldc`"]),
    "gemm_out_rows_past_2^32": ("gemm", dict(GEMM, M=(1 << 20) + 1, ldc=4096), [r"`out` row offset", r"2\^32"]),
    "gemm_resid_rows_past_2^32": ("gemm", dict(GEMM_RES, M=(1 << 16) + 1, ldr=1 << 16), [r"`resid` row offset"]),
    "gemm_row_map_past_2^32": ("gemm", dict(GEMM, rows_per_group=128, group_stride=1 << 25, ldc=128), [r"`out` row offset"]),
    "gemm_negative_group_stride": ("gemm", dict(GEMM, rows_per_group=128, group_stride=-128), [r"`group_stride`"]),
    "gemm_convt_past_2^32": ("gemm", dict(CONVT, M=64 * 1024 * 1024, ct_h=1024, ct_w=1024), [r"`out` row offset"]),
    "gemm_convtile_past_2^32": ("gemm", dict(CONV, conv_B=1 << 10, conv_H=1 << 11, conv_W=1 << 11, conv_inH=1 << 11,
                                             conv_inW=1 << 11, ldc=1024, N=1024), [r"`out` row offset"]),
    "gemm_conv_inH_prepadded": ("gemm", dict(CONV_PRE, conv_inH=30), [r"`conv_inH`"]),
    "gemm_conv_inW_zero_pad": ("gemm", dict(CONV, conv_inW=42), [r"`conv_inW`"]),
    "gemm_conv_off": ("gemm", dict(CONV, conv_off=1), [r"`conv_off`"]),
    # --- attention
    "attn_B0": ("attn", dict(ATTN, B=0), [r"B=0", r">= 1"]),
    "attn_heads0": ("attn", dict(ATTN, heads=0), [r"heads=0", r">= 1"]),
    "attn_seq_q0": ("attn", dict(ATTN, seq_q=0), [r"seq_q=0", r">= 1"]),
    "attn_seq_k0": ("attn", dict(ATTN, seq_k=0), [r"seq_k=0", r">= 1"]),
    "attn_out_misaligned": ("attn", dict(ATTN, out=P["out"] + 2), [r"`out`", r"4-byte"]),
    "attn_o_col0_odd": ("attn", dict(ATTN, o_col0=1, ldo=136), [r"`o_col0`", r"even"]),
    "attn_ldo_short": ("attn", dict(ATTN, o_col0=8), [r"`ldo`"]),
    "attn_ldq_short": ("attn", dict(ATTN, q_col0=8), [r"`ldq`"]),
    "attn_ldk_short": ("attn", dict(ATTN, k_col0=64), [r"`ldk`"]),
    "attn_ldv_short": ("attn", dict(ATTN, v_col0=64), [r"`ldv`"]),
    "attn_split_lo_off_o_odd": ("attn", dict(ATTN_SPLIT, lo_off_o=127), [r"`lo_off_o`", r"even"]),
    "attn_split_ldo_short": ("attn", dict(ATTN_SPLIT, ldo=128), [r"`ldo`"]),
    "attn_split_seq_k0": ("attn", dict(ATTN_SPLIT, seq_k=0), [r"seq_k=0"]),
    # --- halo conv
    "halo_B0": ("halo", dict(HALO, B=0), [r"B=0", r">= 1"]),
    "halo_H0": ("halo", dict(HALO, H=0), [r"H=0", r">= 1"]),
    "halo_W0": ("halo", dict(HALO, W=0), [r"W=0", r">= 1"]),
    "halo_channels_past_cstride": ("halo", dict(HALO, coff=96), [r"`coff`", r"`cstride`"]),
    "halo_ldc_odd": ("halo", dict(HALO, ldc=65), [r"`ldc`", r"even"]),
    "halo_ldc_below_cout": ("halo", dict(HALO, ldc=32), [r"`ldc`", r"cout"]),
    "halo_out_misaligned": ("halo", dict(HALO, out=P["out"] + 2), [r"`out`", r"4-byte"]),
    "halo_head_w_null": ("halo", dict(HALO_HEAD, head_w=0), [r"`head_w`"]),
    "halo_bias_null": ("halo", dict(HALO, bias=0), [r"bias"]),
}

# what a valid call meets after the checks without a device: the tensor-map encoder or the driver
LATER_FAILURE = r"cuTensorMap|cudaFuncSetAttribute|launch|CUDA|device"


def _child_main():
    """Runs in the fresh interpreter: one call per case (JSON on stdin), results as JSON on stdout."""
    import ctypes as C

    from unidepth_b200 import _cabi
    lib = _cabi.lib()
    structs = {"gemm": (_cabi.Gemm, lib.udb_gemm_f16), "attn": (_cabi.Attn, lib.udb_attention_f16),
               "halo": (_cabi.ConvHalo, lib.udb_conv3x3_halo_f16)}
    res = {}
    for name, (kind, fields) in json.load(sys.stdin).items():
        cls, fn = structs[kind]
        s = cls()
        for k, v in fields.items():
            setattr(s, k, v)
        n0 = lib.udb_launch_count()
        rc = fn(C.byref(s), None)
        res[name] = {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}
    json.dump(res, sys.stdout)


_RESULTS = {}


def _results():
    if not _RESULTS:
        cases = {n: (k, f) for n, (k, f, _) in REJECT.items()}
        cases.update({"valid:" + n: v for n, v in VALID.items()})
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
        code = "import sys; sys.path.insert(0, 'tests'); import test_kernel_args_cpu as t; t._child_main()"
        out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, input=json.dumps(cases), capture_output=True,
                             text=True, check=True).stdout
        _RESULTS.update(json.loads(out))
    return _RESULTS


@pytest.mark.parametrize("name", sorted(REJECT))
def test_layout_is_rejected_before_any_cuda_call(name):
    _, _, patterns = REJECT[name]
    r = _results()[name]
    print(f"{name}: rc {r['rc']} '{r['msg']}'")
    assert r["rc"] != 0, name
    for pat in patterns:
        assert re.search(pat, r["msg"]), (name, pat, r["msg"])
    assert not re.search(LATER_FAILURE, r["msg"]), (name, r["msg"])   # stopped by the layout check, not by the device
    assert r["launched"] == 0


@pytest.mark.parametrize("name", sorted(VALID))
def test_valid_layout_gets_past_the_checks(name):
    r = _results()["valid:" + name]
    print(f"{name}: rc {r['rc']} '{r['msg']}'")
    assert r["rc"] != 0 and r["launched"] == 0           # no device: it cannot succeed
    assert re.search(LATER_FAILURE, r["msg"]), (name, r["msg"])
    for _, _, patterns in REJECT.values():                # and no layout check fired
        assert not all(re.search(p, r["msg"]) for p in patterns), (name, r["msg"])


def test_ops_reject_non_unit_stride_outputs():
    """ops.gemm / conv3x3 / conv_transpose_ks / attention assert stride(-1) == 1 on out, out2 and resid before any call
    into the library (CPU tensors never reach it: the stride assertion comes first)."""
    import torch
    from unidepth_b200 import ops
    a, w = torch.zeros(4, 64, dtype=torch.float16), torch.zeros(32, 64, dtype=torch.float16)
    bad32 = torch.zeros(32, 4).t()                        # [4, 32] with stride(-1) == 4
    bad16 = torch.zeros(32, 4, dtype=torch.float16).t()
    for kw in ({"out": bad32}, {"out2": bad16}, {"resid": bad32}):
        with pytest.raises(AssertionError, match="stride"):
            ops.gemm(a, w, **kw)
    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16)
    wc = torch.zeros(32, 9 * 64, dtype=torch.float16)
    bad_map = torch.zeros(1, 4, 32, 4).transpose(2, 3)   # [1, 4, 4, 32], stride(-1) == 4
    for kw in ({"out": bad_map}, {"resid": bad_map}, {"out2": bad_map.half()}):
        with pytest.raises(AssertionError, match="stride"):
            ops.conv3x3(x, wc, **kw)
    with pytest.raises(AssertionError, match="stride"):
        ops.conv_transpose_ks(a, w, 1, 32, (2, 2), out=bad_map)
    q = torch.zeros(128, 64, dtype=torch.float16)
    with pytest.raises(AssertionError, match="stride"):
        ops.attention(q, q, q, torch.zeros(64, 128, dtype=torch.float16).t(), B=1, heads=1, seq_q=128, seq_k=128, head_dim=64)
