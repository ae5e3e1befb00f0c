"""The GEMM, attention and halo-conv kernels on their own, across the arguments they accept, against float64 references
with per-element bounds (derived in tests/kernel_ref.py).  Every case also checks that

  * each output lives inside a larger buffer (extra rows, extra columns, a column offset) filled with a NaN bit pattern,
    and every cell outside the written region still holds that exact pattern afterwards;
  * a second run gives bit-identical outputs;
  * the largest err / bound ratio is printed (run with -s to see them)."""
import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R

pytestmark = pytest.mark.gpu

f16, f32 = torch.float16, torch.float32
PATTERN = {f32: (torch.int32, 0x7FC0DEAD), f16: (torch.int16, 0x7E5A)}   # quiet NaNs with a recognisable payload


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _ops():
    from unidepth_b200 import ops
    return ops


def sentinel(shape, dtype, dev):
    it, pat = PATTERN[dtype]
    return torch.full(shape, pat, dtype=it, device=dev).view(dtype)


def bits(t):
    return t.view(PATTERN[t.dtype][0])


def untouched(buf, mask, name):
    it, pat = PATTERN[buf.dtype]
    outside = bits(buf)[~mask]
    bad = (outside != pat).sum().item()
    assert bad == 0, f"{name}: {bad} cells outside the written region were modified"


def twice(run, name):
    """run() (re)initialises its buffers, launches and returns them; the two runs must agree bit for bit"""
    first = [t.clone() for t in run()]
    second = run()
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(first, second)):
        assert torch.equal(bits(x), bits(y)), f"{name}: output {i} differs between two identical runs"
    return second


def region(shape, rows, cols, dev):
    m = torch.zeros(shape, dtype=torch.bool, device=dev)
    m[rows, cols] = True
    return m


# ------------------------------------------------------------------------------------------------ GEMM, matrix mode
NS = [256, 768, 192, 576, 640, 320, 32, 96]          # tile widths 256, 256, 192, 192, 128, 64, 32, 32
MS = [1, 127, 129, 128 * 132 + 1]                     # 132 SMs: the last size gives every CTA >= 2 tiles and a ragged wave
KS = [8, 56, 72, 200, 1024]                           # K < 64, K tails, several k-blocks
EPIS = ["plain", "bias", "gelu", "leaky", "gamma_resid32", "resid16", "inplace", "out2_leaky", "out2_plain"]
GEMM_CASES = [(N, M, KS[(i + j) % len(KS)], EPIS[(4 * i + j) % len(EPIS)], (i + j) % 2 == 0)
              for i, N in enumerate(NS) for j, M in enumerate(MS)]


@pytest.mark.parametrize("N,M,K,epi,out32", GEMM_CASES)
def test_gemm_matrix(N, M, K, epi, out32):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(N * 131 + M * 7 + K)
    odt = f32 if out32 else f16
    lda = (K + 7) // 8 * 8 + 24                                            # strided A: lda > K
    a = (torch.randn(M, lda, generator=g)).half().to(dev)[:, :K]
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev) if epi != "plain" else None
    act = {"gelu": ops.ACT_GELU, "leaky": ops.ACT_LEAKY}.get(epi, ops.ACT_NONE)
    gamma = (torch.rand(N, generator=g) + 0.5).to(dev) if epi in ("gamma_resid32", "inplace") else None
    rdt = {"gamma_resid32": f32, "resid16": f16, "inplace": odt}.get(epi)
    r0 = None
    if rdt is not None:                                                    # residual: column slice of a wider buffer
        r0 = torch.randn(M, N + 8, generator=g).to(dev).to(rdt)[:, 4:4 + N]
    shape = (M + 3, N + 40)                                                # 1 row above, 2 below, 4 columns left, 36 right
    mask = region(shape, slice(1, 1 + M), slice(4, 4 + N), dev)
    with_out2 = epi.startswith("out2")

    def run():
        buf = sentinel(shape, odt, dev)
        out = buf[1:1 + M, 4:4 + N]
        resid = r0
        if epi == "inplace":
            out.copy_(r0)
            resid = out
        buf2 = sentinel(shape, f16, dev) if with_out2 else None
        out2 = buf2[1:1 + M, 4:4 + N] if with_out2 else None
        ops.gemm(a, w, bias=bias, act=act, gamma=gamma, resid=resid, out=out, out2=out2, out2_leaky=epi == "out2_leaky")
        return [buf] + ([buf2] if with_out2 else [])

    res = twice(run, f"gemm {M}x{N}x{K} {epi}")
    ref, bnd = R.gemm_ref(a, w, bias=bias, act=act, gamma=gamma, resid=r0)
    if not out32:
        bnd = R.f16_out(ref, bnd)
    name = f"gemm M{M} N{N} K{K} {epi} {'f32' if out32 else 'f16'}"
    untouched(res[0], mask, name)
    R.within(res[0][1:1 + M, 4:4 + N], ref, bnd, name)
    if with_out2:
        ref2 = F.leaky_relu(ref, 0.01) if epi == "out2_leaky" else ref
        untouched(res[1], mask, name + " out2")
        R.within(res[1][1:1 + M, 4:4 + N], ref2, R.f16_out(ref2, bnd), name + " out2")


def test_gemm_row_map():
    """ROWS store with a row map (tokens of 3 images -> rows b*T + 1 + n, gaps between images) and a residual indexed by
    m % resid_mod + resid_row_offset (the position table), into a column slice: only the mapped cells may change."""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(11)
    Bn, Np, N, K = 3, 259, 192, 200
    T = Np + 3
    a = torch.randn(Bn * Np, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    pos = torch.randn(T, N, generator=g).to(dev)
    shape = (Bn * T + 2, N + 12)
    mask = torch.zeros(shape, dtype=torch.bool, device=dev)
    for b in range(Bn):
        mask[b * T + 1:b * T + 1 + Np, 4:4 + N] = True

    def run():
        buf = sentinel(shape, f32, dev)
        ops.gemm(a, w, bias=bias, resid=pos, out=buf[:, 4:4 + N], rows_per_group=Np, group_stride=T, row_offset=1,
                 resid_mod=Np, resid_row_offset=1)
        return [buf]

    buf, = twice(run, "row map")
    ref, bnd = R.gemm_ref(a, w, bias=bias, resid=pos[1:1 + Np].repeat(Bn, 1))
    untouched(buf, mask, "row map")
    got = torch.cat([buf[b * T + 1:b * T + 1 + Np, 4:4 + N] for b in range(Bn)])
    R.within(got, ref, bnd, "gemm row map")


# ------------------------------------------------------------------------------------------------ GEMM, conv / CONVT
@pytest.mark.parametrize("tile,N", [((8, 16), 64), ((16, 8), 96), ((4, 32), 64), ((1, 128), 96)])
def test_conv3x3_tiles(tile, N):
    """zero-padded 3x3 conv, every spatial tile shape, on a 19 x 37 map (no tile multiple), into a column slice"""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(tile[0] * 1000 + N)
    B, H, W, C = 2, 19, 37, 64
    x = torch.randn(B, H, W, C, generator=g).half().to(dev)
    w = (torch.randn(N, 9 * C, generator=g) / (9 * C) ** 0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    shape = (B, H, W, N + 8)
    mask = region(shape, slice(None), slice(None), dev)
    mask[..., :4] = False
    mask[..., 4 + N:] = False

    def run():
        buf = sentinel(shape, f32, dev)
        ops.conv3x3(x, w, bias=bias, act=ops.ACT_LEAKY, out=buf[..., 4:4 + N], tile=tile)
        return [buf]

    buf, = twice(run, f"conv3x3 tile {tile}")
    ref, bnd = R.conv3x3_ref(F.pad(x, (0, 0, 1, 1, 1, 1)), w, bias=bias, act=R.ACT_LEAKY)
    untouched(buf, mask, f"conv3x3 tile {tile}")
    R.within(buf[..., 4:4 + N], ref, bnd, f"conv3x3 tile {tile} N{N}")


@pytest.mark.parametrize("prepadded,resid32", [(False, False), (False, True), (True, False), (True, True)])
def test_conv3x3_c192_channel_slice(prepadded, resid32):
    """C = 192 read as a channel slice [64, 256) of a 320-channel buffer, zero pad or prepadded, gamma + residual (f16 or
    f32), f16 / f32 output in a column slice plus the leaky f16 copy"""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(192 + 2 * prepadded + resid32)
    B, H, W, C, Ct, N = 1, 21, 30, 192, 320, 192
    p = 1 if prepadded else 0
    xb = torch.randn(B, H + 2 * p, W + 2 * p, Ct, generator=g).half().to(dev)
    w = (torch.randn(N, 9 * C, generator=g) / (9 * C) ** 0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    gamma = (torch.rand(N, generator=g) + 0.5).to(dev)
    odt = f32 if resid32 else f16
    resid = torch.randn(B, H, W, N + 4, generator=g).to(dev).to(odt)[..., :N]
    shape = (B, H, W, N + 12)
    mask = region(shape, slice(None), slice(None), dev)
    mask[..., :8] = False
    mask[..., 8 + N:] = False

    def run():
        buf, buf2 = sentinel(shape, odt, dev), sentinel(shape, f16, dev)
        ops.conv3x3(xb, w, bias=bias, gamma=gamma, resid=resid, out=buf[..., 8:8 + N], out2=buf2[..., 8:8 + N],
                    prepadded=prepadded, c_off=64, c_used=C)
        return [buf, buf2]

    buf, buf2 = twice(run, "conv3x3 C192")
    xs = xb[..., 64:64 + C]
    ref, bnd = R.conv3x3_ref(xs if prepadded else F.pad(xs, (0, 0, 1, 1, 1, 1)), w, bias=bias, gamma=gamma, resid=resid)
    name = f"conv3x3 C192 slice {'prepadded' if prepadded else 'zero pad'} resid {'f32' if resid32 else 'f16'}"
    untouched(buf, mask, name)
    untouched(buf2, mask, name + " out2")
    R.within(buf[..., 8:8 + N], ref, bnd if resid32 else R.f16_out(ref, bnd), name)
    ref2 = F.leaky_relu(ref, 0.01)
    R.within(buf2[..., 8:8 + N], ref2, R.f16_out(ref2, bnd), name + " out2")


def test_conv3x3_head_store():
    """HEAD store (N = 32): LeakyReLU + 1x1 + clamp + exp fused, f32 plane between sentinel planes"""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(32)
    B, H, W, C = 2, 19, 37, 128
    xp = torch.randn(B, H + 2, W + 2, C, generator=g).half().to(dev)
    w = (torch.randn(32, 9 * C, generator=g) / (9 * C) ** 0.5).half().to(dev)
    bias = torch.randn(32, generator=g).to(dev)
    hw = (torch.randn(32, generator=g) * 0.3).to(dev)
    shape = (B + 2, H, W)
    mask = region(shape, slice(1, 1 + B), slice(None), dev)

    def run():
        buf = sentinel(shape, f32, dev)
        ops.conv3x3(xp, w, bias=bias, prepadded=True, act=ops.ACT_LEAKY, head_w=hw, head_b=0.1, head_add=2.0, out=buf[1:1 + B])
        return [buf]

    buf, = twice(run, "conv3x3 head")
    v, vb = R.conv3x3_ref(xp, w, bias=bias)
    ref, bnd = R.head_ref(v, vb, hw, 0.1, 2.0)
    untouched(buf, mask, "conv3x3 head")
    R.within(buf[1:1 + B], ref, bnd, "gemm HEAD store")


@pytest.mark.parametrize("k,pad,cout", [(1, 1, 96), (1, 0, 32), (2, 0, 32), (2, 1, 96), (4, 1, 32), (4, 0, 96)])
def test_conv_transpose_store(k, pad, cout):
    """CONVT (pixel-shuffle) store with an f32 residual and the leaky f16 copy; with pad = 1 the border stays untouched"""
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(k * 100 + pad * 10 + cout)
    B, h, w_, cin = 2, 9, 13, 128
    x = torch.randn(B * h * w_, cin, generator=g).half().to(dev)
    wp = (torch.randn(k * k * cout, cin, generator=g) / cin ** 0.5).half().to(dev)
    bp = torch.randn(k * k * cout, generator=g).to(dev)
    shape = (B, h * k + 2 * pad, w_ * k + 2 * pad, cout)
    resid = torch.randn(shape, generator=g).to(dev)
    idx = R.convt_index(B, h, w_, k, cout, pad, device=dev)
    mask = torch.zeros(shape, dtype=torch.bool, device=dev)
    mask.view(-1)[idx.reshape(-1)] = True

    def run():
        out, out2 = sentinel(shape, f32, dev), sentinel(shape, f16, dev)
        ops.conv_transpose_ks(x, wp, k, cout, (h, w_), bias=bp, resid=resid, out=out, out2=out2, pad=pad)
        return [out, out2]

    out, out2 = twice(run, "convT")
    ref, bnd = R.gemm_ref(x, wp, bias=bp, resid=resid.view(-1)[idx])
    name = f"convT k{k} pad{pad} cout{cout}"
    untouched(out, mask, name)
    untouched(out2, mask, name + " out2")
    R.within(out.view(-1)[idx], ref, bnd, name)
    ref2 = F.leaky_relu(ref, 0.01)
    R.within(out2.view(-1)[idx], ref2, R.f16_out(ref2, bnd), name + " out2")


# ------------------------------------------------------------------------------------------------ attention
def _attention(q, k, v, scale, name, *, q_col0=0, o_col0=0, o_pad=16, fused=False, split=False):
    """Lay q [B,H,Sq,64], k / v [B,H,Sk,64] out as the engines do (fused qkv, or q alone + kv), run the kernel into a
    sentinel buffer with o_col0 / ldo > H*64, and check it.  Returns the output as [B, H, Sq, 64]."""
    ops, dev = _ops(), _dev()
    B, H, Sq, _ = q.shape
    Sk = k.shape[2]
    D = H * 64
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(t.shape[0] * t.shape[2], D)
    if fused:
        qkv = torch.cat([rows(q), rows(k), rows(v)], 1).to(dev)
        args = (qkv, qkv, qkv)
        cols = dict(q_col0=0, k_col0=D, v_col0=2 * D)
    elif split:                                            # split-f16 operands: [hi | lo], lo = 0 (the values are f16)
        pack = lambda t: torch.cat([rows(t), torch.zeros_like(rows(t))], 1).to(dev)
        args = (pack(q), pack(k), pack(v))
        cols = dict(lo_off_in=D)
    else:
        qb = torch.cat([torch.zeros(B * Sq, q_col0, dtype=f16), rows(q)], 1).to(dev)
        kv = torch.cat([rows(k), rows(v)], 1).to(dev)
        args = (qb, kv, kv)
        cols = dict(q_col0=q_col0, k_col0=0, v_col0=D)
    ldo = (o_col0 + D + 7) // 8 * 8 + o_pad                 # a multiple of 8, > o_col0 + H*64 when o_pad > 0
    shape = (B * Sq + 3, ldo)
    mask = region(shape, slice(1, 1 + B * Sq), slice(o_col0, o_col0 + D), dev)

    def run():
        buf = sentinel(shape, f16, dev)
        ops.attention(*args, buf[1:1 + B * Sq], B=B, heads=H, seq_q=Sq, seq_k=Sk, head_dim=64, o_col0=o_col0, scale=scale, **cols)
        return [buf]

    buf, = twice(run, name)
    untouched(buf, mask, name)
    got = buf[1:1 + B * Sq, o_col0:o_col0 + D].view(B, Sq, H, 64).permute(0, 2, 1, 3)
    ref, bnd = R.attention_ref(q.to(dev), k.to(dev), v.to(dev), scale, f16_p=not split)
    R.within(got, ref, bnd, name)
    return got


SK = [1, 2, 15, 16, 17, 127, 128, 129, 255, 256, 257, 384, 385]   # 384 = 3 stages x 128: the K/V ring wraps on a tile edge
SQ = [1, 63, 64, 65, 127, 128, 129]
ATTN_GRID = [(SQ[(i + s) % len(SQ)], sk, 1 + (i + s) % 2) for i, sk in enumerate(SK) for s in (0, 3)]


@pytest.mark.parametrize("Sq,Sk,B", ATTN_GRID)
def test_attention_lengths(Sq, Sk, B):
    g = torch.Generator().manual_seed(Sq * 1000 + Sk)
    q, k, v = R.attn_inputs(B, 2, Sq, Sk, g)
    _attention(q, k, v, 0.125, f"attention B{B} Sq{Sq} Sk{Sk}", q_col0=64 * (Sk % 2), o_col0=2 * (Sq % 3), o_pad=8 * (Sk % 3))


@pytest.mark.parametrize("Sq,Sk,fused", [(1611, 1611, True), (1453, 1453, True), (128, 1000, False), (1000, 128, False)])
def test_attention_engine_lengths(Sq, Sk, fused):
    """V2 ViT-L tokens (1 + 35*46), V1 ViT-L tokens (1 + 33*44), the Nystrom landmark attentions (1000 <-> 128)"""
    g = torch.Generator().manual_seed(Sq + Sk)
    q, k, v = R.attn_inputs(2, 4, Sq, Sk, g)
    _attention(q, k, v, 0.125, f"attention engine Sq{Sq} Sk{Sk}", fused=fused)


@pytest.mark.parametrize("hd", [32, 48])
def test_attention_zero_padded_heads(hd):
    """decoder prompt blocks: true head dim 32 (ViT-S: hidden 256 / 8 heads) or 48, zero-padded to 64, explicit scale;
    the padded output dims must be exactly 0"""
    g = torch.Generator().manual_seed(hd)
    q, k, v = R.attn_inputs(2, 8, 600, 600, g)
    for t in (q, k, v):
        t[..., hd:] = 0
    got = _attention(q, k, v, hd ** -0.5, f"attention padded head dim {hd}")
    assert (bits(got[..., hd:].contiguous()) == 0).all()


def test_attention_batch_isolation():
    """B = 3, seq_k = 258 (2 valid keys in the last tile); image b+1's keys score 30 above image b's"""
    g = torch.Generator().manual_seed(3)
    q, k, v = R.isolation_inputs(3, 130, 258, g)
    _attention(q, k, v, 0.125, "attention batch isolation")


def test_attention_one_hot_row():
    """one key outscores every other by > 40: the output is that key's V row to f16 precision"""
    g = torch.Generator().manual_seed(4)
    q, k, v = R.isolation_inputs(1, 64, 300, g, step=0.0)
    k[0, 0, 137, 0] = 45.0 / (4.0 * 0.125)
    got = _attention(q, k, v, 0.125, "attention one-hot row")
    vr = v[0, 0, 137].to(got.device).float()
    assert ((got[0, 0].float() - vr).abs() <= R.U16 * vr.abs() + 1e-7).all()


def test_attention_large_logits():
    """scale * s spans more than 100 within a row: outputs stay finite and inside the bound"""
    g = torch.Generator().manual_seed(5)
    q, k, v = R.attn_inputs(2, 2, 200, 300, g, q_gain=6.0, k_gain=6.0)
    s = (q.double() @ k.double().transpose(-1, -2)) * 0.125
    assert (s.amax(-1) - s.amin(-1)).min().item() > 100
    got = _attention(q, k, v, 0.125, "attention large logits")
    assert torch.isfinite(got.float()).all()


def test_attention_split_kernel():
    """fp32 split kernel: seq_q / seq_k not multiples of 64, 3 heads, hi-only output (lo_off_out = 0)"""
    g = torch.Generator().manual_seed(6)
    q, k, v = R.attn_inputs(2, 3, 150, 203, g)
    _attention(q, k, v, 0.125, "attention split kernel", split=True)


# ------------------------------------------------------------------------------------------------ halo conv
HALO_CASES = [
    # B, H, W, C, cstride, coff, cout, head, ldc_extra
    (2, 40, 21, 64, 128, 64, 64, False, 0),      # engine.cu lr conv: second half of the shared MLP map
    (2, 40, 21, 64, 128, 64, 32, True, 0),       # the Cout = 32 head on a channel slice
    (1, 17, 9, 192, 192, 0, 32, True, 0),        # 3-stage ring, 3 slabs per tile
    (1, 16, 8, 256, 256, 0, 32, False, 6),       # 2-stage ring wrapping inside every tile (4 slabs), column-slice output
    (1, 1, 1, 64, 64, 0, 64, False, 8),          # maps smaller than one 16 x 8 tile
    (2, 5, 7, 128, 128, 0, 32, True, 0),
    (2, 160, 100, 64, 64, 0, 64, False, 4),      # 260 tiles: more than one per SM
]


@pytest.mark.parametrize("B,H,W,C,cs,coff,cout,head,extra", HALO_CASES)
def test_conv3x3_halo(B, H, W, C, cs, coff, cout, head, extra):
    ops, dev = _ops(), _dev()
    g = torch.Generator().manual_seed(H * 100 + W + C + cout)
    xp = torch.randn(B, H + 2, W + 2, cs, generator=g).half().to(dev)
    w = (torch.randn(cout, 9 * C, generator=g) / (9 * C) ** 0.5).half().to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    name = f"halo B{B} {H}x{W} C{C}/{cs}+{coff} cout{cout} {'head' if head else 'f16 leaky'}"
    xs = xp[..., coff:coff + C]
    if head:
        hw = (torch.randn(32, generator=g) * 0.3).to(dev)
        shape = (B + 1, H, W)
        mask = region(shape, slice(0, B), slice(None), dev)

        def run():
            buf = sentinel(shape, f32, dev)
            ops.conv3x3_halo(xp, w, bias=bias, act=ops.ACT_LEAKY, c_off=coff, c_used=C, head_w=hw, head_b=0.1, head_add=2.0,
                             out=buf[:B])
            return [buf]

        buf, = twice(run, name)
        v, vb = R.conv3x3_ref(xs, w, bias=bias)
        ref, bnd = R.head_ref(v, vb, hw, 0.1, 2.0)
        untouched(buf, mask, name)
        R.within(buf[:B], ref, bnd, name)
    else:
        c0 = 2 if extra else 0
        shape = (B, H, W, cout + extra)
        mask = region(shape, slice(None), slice(None), dev)
        mask[..., :c0] = False
        mask[..., c0 + cout:] = False

        def run():
            buf = sentinel(shape, f16, dev)
            ops.conv3x3_halo(xp, w, bias=bias, act=ops.ACT_LEAKY, c_off=coff, c_used=C, out=buf[..., c0:c0 + cout])
            return [buf]

        buf, = twice(run, name)
        ref, bnd = R.conv3x3_ref(xs, w, bias=bias, act=R.ACT_LEAKY)
        untouched(buf, mask, name)
        R.within(buf[..., c0:c0 + cout], ref, R.f16_out(ref, bnd), name)
