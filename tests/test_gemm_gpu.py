"""wgmma GEMM / conv / convT kernel vs a plain PyTorch fp32 reference of the same op (operands
rounded to f16 exactly as the kernel sees them, fp32 math).  Tolerances: fp32 accumulation-order
noise for f32 outputs, one f16 ulp for f16 outputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _close(got, ref, tol, name):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"{name}: max abs err {err:.3e} (ref max {scale:.3e})")
    assert err <= tol * max(scale, 1.0), (name, err, scale)


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 128, 128), (1000, 1024, 1024), (12888, 3072, 1024),
                                   (1611, 384, 1536), (300, 64, 640), (130, 32, 192), (256, 64, 200)])
def test_gemm_plain(M, N, K):
    from unidepth_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N)
    a = torch.randn(M, K, generator=g).to(dev).half()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    ref = a.float() @ w.float().t() + bias
    out32 = ops.gemm(a, w, bias=bias, out_dtype=torch.float32)
    _close(out32, ref, 2e-5, f"gemm f32 {M}x{N}x{K}")
    out16 = ops.gemm(a, w, bias=bias, out_dtype=torch.float16)
    _close(out16, ref, 1e-3, f"gemm f16 {M}x{N}x{K}")


def test_gemm_epilogues():
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(0)
    M, N, K = 777, 512, 256
    a = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) / K ** 0.5).half()
    bias = torch.randn(N, device=dev)
    gamma = torch.rand(N, device=dev) + 0.5
    resid = torch.randn(M, N, device=dev)
    lin = a.float() @ w.float().t() + bias
    _close(ops.gemm(a, w, bias=bias, act=ops.ACT_GELU, out_dtype=torch.float32), F.gelu(lin), 2e-5, "gelu")
    _close(ops.gemm(a, w, bias=bias, act=ops.ACT_LEAKY, out_dtype=torch.float32), F.leaky_relu(lin, 0.01), 2e-5, "leaky")
    _close(ops.gemm(a, w, bias=bias, gamma=gamma, resid=resid, out_dtype=torch.float32), resid + gamma * lin, 2e-5, "gamma+resid f32")
    r16 = resid.half()
    _close(ops.gemm(a, w, bias=bias, resid=r16, out_dtype=torch.float32), r16.float() + lin, 2e-5, "resid f16")
    # in-place residual stream (out aliases resid)
    x = resid.clone()
    ops.gemm(a, w, bias=bias, gamma=gamma, resid=x, out=x)
    _close(x, resid + gamma * lin, 2e-5, "in-place residual")
    # second output = leaky(out) in f16
    out2 = torch.empty(M, N, device=dev, dtype=torch.float16)
    o = ops.gemm(a, w, bias=bias, out_dtype=torch.float32, out2=out2)
    _close(out2, F.leaky_relu(o, 0.01), 1e-3, "out2 leaky")
    # row mapping: tokens of B images -> rows b*T + 1 + n, residual = pos[1 + n]
    Bn, Np = 3, 259
    T = Np + 1
    a2 = torch.randn(Bn * Np, K, device=dev).half()
    pos = torch.randn(T, N, device=dev)
    x = torch.zeros(Bn * T, N, device=dev)
    ops.gemm(a2, w, bias=bias, resid=pos, out=x, rows_per_group=Np, group_stride=T, row_offset=1,
             resid_mod=Np, resid_row_offset=1)
    ref = (a2.float() @ w.float().t() + bias).view(Bn, Np, N) + pos[1:]
    _close(x.view(Bn, T, N)[:, 1:], ref, 2e-5, "token row mapping")
    assert x.view(Bn, T, N)[:, 0].abs().max().item() == 0.0


@pytest.mark.parametrize("B,H,W,C,N,tile", [(1, 16, 32, 64, 64, (8, 16)), (2, 35, 46, 128, 256, (8, 16)),
                                            (1, 70, 92, 256, 128, (8, 16)), (1, 20, 33, 64, 32, (4, 32))])
def test_conv3x3_zero_pad(B, H, W, C, N, tile):
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(1)
    x = torch.randn(B, C, H, W, device=dev).half()
    w = (torch.randn(N, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    bias = torch.randn(N, device=dev)
    ref = F.conv2d(x.float(), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    xn = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops.conv3x3(xn, wp, bias=bias, out_dtype=torch.float32, tile=tile)
    _close(out, ref, 3e-5, f"conv3x3 {B}x{H}x{W}x{C}->{N}")
    # RCU-style epilogue: gamma*conv + x, plus leaky copy
    if N == C:
        gamma = torch.rand(N, device=dev) + 0.5
        out2 = torch.empty(B, H, W, N, device=dev, dtype=torch.float16)
        o = ops.conv3x3(xn, wp, bias=bias, gamma=gamma, resid=xn, out_dtype=torch.float16, out2=out2)
        r = gamma * ref + xn.float()
        _close(o, r, 1.5e-3, "conv3x3 rcu epilogue")
        _close(out2, F.leaky_relu(r, 0.01), 1.5e-3, "conv3x3 rcu out2")


def test_conv3x3_reflect_and_head():
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(2)
    B, H, W, C, N = 2, 37, 50, 64, 32
    x = torch.randn(B, C, H, W, device=dev).half()
    w = (torch.randn(N, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    bias = torch.randn(N, device=dev)
    xp = F.pad(x.float(), (1, 1, 1, 1), mode="reflect")
    ref = F.conv2d(xp, w.float(), bias)
    xn = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    xpad = ops.reflect_pad1(xn)
    assert torch.equal(xpad.float(), xp.permute(0, 2, 3, 1))
    out = ops.conv3x3(xpad, wp, bias=bias, out_dtype=torch.float32, prepadded=True)
    _close(out, ref.permute(0, 2, 3, 1), 3e-5, "conv3x3 reflect")
    hw = torch.randn(32, device=dev) * 0.3
    hb = 0.1
    head = ops.conv3x3(xpad, wp, bias=bias, prepadded=True, act=ops.ACT_LEAKY, head_w=hw, head_b=hb, head_add=2.0)
    hr = torch.exp((F.leaky_relu(ref, 0.01) * hw.view(1, -1, 1, 1)).sum(1).add(hb).clip(-8, 8) + 2.0)
    _close(head, hr, 3e-5, "conv3x3 head")


@pytest.mark.parametrize("k,cout", [(1, 128), (2, 64), (4, 32)])
def test_conv_transpose(k, cout):
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(3)
    B, h, w_, cin = 2, 9, 13, 128
    x = torch.randn(B, cin, h, w_, device=dev).half()
    wt = (torch.randn(cin, cout, k, k, device=dev) / cin ** 0.5).half()
    bias = torch.randn(cout, device=dev)
    lat = torch.randn(B, h * k, w_ * k, cout, device=dev).half()
    ref = F.conv_transpose2d(x.float(), wt.float(), bias, stride=k).permute(0, 2, 3, 1) + lat.float()
    xm = x.permute(0, 2, 3, 1).reshape(B * h * w_, cin).contiguous()
    wp = wt.permute(2, 3, 1, 0).reshape(k * k * cout, cin).contiguous()
    bp = bias.repeat(k * k).contiguous()
    out2 = torch.empty_like(lat)
    out = ops.conv_transpose_ks(xm, wp, k, cout, (h, w_), bias=bp, resid=lat, out=lat.clone(), out2=out2)
    _close(out, ref, 1.5e-3, f"convT k={k}")
    _close(out2, F.leaky_relu(ref, 0.01), 1.5e-3, f"convT k={k} out2")


def test_padded_linear_border_fill_and_channel_slice_conv():
    """LN->Linear written into a reflect-padded buffer + 3x3 conv over a channel slice of it."""
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(4)
    B, H, W, Cin, C2 = 2, 21, 30, 128, 256
    x = torch.randn(B * H * W, Cin, device=dev).half()
    wl = (torch.randn(C2, Cin, device=dev) / Cin ** 0.5).half()
    bl = torch.randn(C2, device=dev)
    mp = torch.zeros(B, H + 2, W + 2, C2, device=dev, dtype=torch.float16)
    ops.conv_transpose_ks(x, wl, 1, C2, (H, W), bias=bl, out=mp, pad=1)
    ops.reflect_border_fill(mp)
    lin = (x.float() @ wl.float().t() + bl).view(B, H, W, C2).permute(0, 3, 1, 2)
    ref_pad = F.pad(lin, (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1)
    _close(mp, ref_pad, 1.5e-3, "padded linear + border fill")
    for i in range(2):
        wc = (torch.randn(64, 128, 3, 3, device=dev) / (9 * 128) ** 0.5).half()
        bc = torch.randn(64, device=dev)
        wp = wc.permute(0, 2, 3, 1).reshape(64, 9 * 128).contiguous()
        out = ops.conv3x3(mp, wp, bias=bc, prepadded=True, out_dtype=torch.float32, c_off=128 * i, c_used=128)
        ref = F.conv2d(mp.float().permute(0, 3, 1, 2)[:, 128 * i:128 * (i + 1)], wc.float(), bc).permute(0, 2, 3, 1)
        _close(out, ref, 3e-5, f"conv3x3 channel slice {i}")


@pytest.mark.parametrize("C,N,H,W", [(64, 32, 37, 50), (128, 64, 40, 21), (64, 32, 490, 644)])
def test_conv3x3_halo(C, N, H, W):
    """Halo-reuse conv kernel (shifted UMMA descriptors) vs F.conv2d on the reflect-padded input."""
    from unidepth_b200 import ops
    dev = _dev()
    torch.manual_seed(5)
    B = 2
    x = torch.randn(B, C, H, W, device=dev).half()
    w = (torch.randn(N, C, 3, 3, device=dev) / (9 * C) ** 0.5).half()
    bias = torch.randn(N, device=dev)
    xp = F.pad(x.float(), (1, 1, 1, 1), mode="reflect")
    ref = F.conv2d(xp, w.float(), bias)
    xpad = xp.permute(0, 2, 3, 1).contiguous().half()
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    if N == 64:
        out = ops.conv3x3_halo(xpad, wp, bias=bias)
        _close(out, ref.permute(0, 2, 3, 1), 1.5e-3, f"halo conv {C}->{N}")
    else:
        hw = torch.randn(32, device=dev) * 0.3
        head = ops.conv3x3_halo(xpad, wp, bias=bias, act=ops.ACT_LEAKY, head_w=hw, head_b=0.1, head_add=2.0)
        hr = torch.exp((F.leaky_relu(ref, 0.01) * hw.view(1, -1, 1, 1)).sum(1).add(0.1).clip(-8, 8) + 2.0)
        _close(head, hr, 3e-5, f"halo conv head {C}->{N} {H}x{W}")


def test_split_f16_gemm_layernorm_attention():
    """Split-f16 precise mode (udb_gemm_t.a_split_k / out_split, udb_layernorm_t.out_split, udb_attn_t.split): operands
    as hi + lo f16 pairs through the SAME wgmma GEMM, attention in fp32.  Against float64 the error must drop from
    f16's ~3e-4 to ~1e-6."""
    import torch
    from unidepth_b200 import ops
    dev = "cuda:0"
    g = torch.Generator(device="cpu").manual_seed(7)
    M, K, N = 777, 1024, 384

    def split(t):
        hi = t.half()
        return hi, (t - hi.float()).half()

    a = torch.randn(M, K, generator=g).to(dev)
    w = (torch.randn(N, K, generator=g) * 0.05).to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    ah, al = split(a)
    wh, wl = split(w)
    a2 = torch.cat([ah, al], 1).contiguous()
    w3 = torch.cat([wh, wh, wl], 1).contiguous()
    ref = (a.double() @ w.double().T + bias.double())
    out32 = ops.gemm(a2, w3, bias=bias, a_split_k=K, out_dtype=torch.float32)
    err = ((out32.double() - ref).abs().max() / ref.abs().max()).item()
    plain = ops.gemm(ah, wh, bias=bias, out_dtype=torch.float32)
    err16 = ((plain.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"split GEMM max err / max|ref|: {err:.2e} (plain f16 operands: {err16:.2e})")
    assert err < 2e-5 and err16 > 20 * err       # measured 6.7e-6 vs 2.5e-4 (the lo.lo term is dropped)
    # split output: hi + lo reproduces the f32 result to ~2^-21
    o2 = ops.gemm(a2, w3, bias=bias, a_split_k=K, out_split=True)
    rec = o2[:, :N].float() + o2[:, N:].float()
    assert ((rec - out32).abs().max() / out32.abs().max()).item() < 4e-6
    # LayerNorm with a split output
    x = torch.randn(300, 1024, generator=g).to(dev) * 3 + 1
    lw, lb = torch.randn(1024, generator=g).to(dev), torch.randn(1024, generator=g).to(dev)
    y2 = ops.layernorm(x, lw, lb, 1e-6, out_split=True)
    yref = torch.nn.functional.layer_norm(x.double(), (1024,), lw.double(), lb.double(), 1e-6)
    rec = y2[:, :1024].float() + y2[:, 1024:].float()
    assert ((rec.double() - yref).abs().max() / yref.abs().max()).item() < 6e-6
    # fp32 attention on split operands (ragged lengths: 150 queries, 203 keys, 2 images x 3 heads)
    B, Hh, Sq, Sk = 2, 3, 150, 203
    q, k, v = (torch.randn(B * S, Hh * 64, generator=g).to(dev) for S in (Sq, Sk, Sk))
    pack = lambda t: torch.cat(split(t), 1).contiguous()
    o = torch.empty(B * Sq, 2 * Hh * 64, device=dev, dtype=torch.float16)
    ops.attention(pack(q), pack(k), pack(v), o, B=B, heads=Hh, seq_q=Sq, seq_k=Sk, head_dim=64,
                  lo_off_in=Hh * 64, lo_off_out=Hh * 64)
    rec = (o[:, :Hh * 64].float() + o[:, Hh * 64:].float()).view(B, Sq, Hh, 64)
    qd, kd, vd = (t.double().view(B, -1, Hh, 64).transpose(1, 2) for t in (q, k, v))
    aref = torch.softmax(qd @ kd.transpose(-1, -2) / 8.0, -1) @ vd
    err = ((rec.double().transpose(1, 2) - aref).abs().max() / aref.abs().max()).item()
    print(f"split attention max err: {err:.2e}")
    assert err < 1e-5


@pytest.mark.parametrize("D", [1024, 768, 384, 640, 320, 96])
def test_fused_layernorm_producer_consumer(D):
    """udb_gemm_t.ln_*: a residual-updating GEMM writes per-part row statistics + the f16 copy of its rows; the next GEMM
    applies LayerNorm algebraically in its epilogue.  Reference: LayerNorm(x) @ W^T + b in float64 on the producer's f32 output.
    D picks the producer's tile width (256, 192, 128, 64 and 32: at 32 one column group, so parts of 32 columns); below
    D = 384 the consumer is D wide too, so it also runs the 64- and 32-column tiles."""
    from unidepth_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(D)
    M, K0 = 1500, 256
    N2 = 640 if D >= 384 else D
    bn = next(b for b in (256, 192, 128, 64, 32) if D % b == 0)
    groups = 2 if bn >= 64 else 1
    parts, pc = D // bn * groups, bn // groups
    a = torch.randn(M, K0, generator=g).to(dev).half()
    w0 = (torch.randn(D, K0, generator=g) / 16).to(dev).half()
    x_in = (torch.randn(M, D, generator=g) * 1.5 + 0.3).to(dev)            # residual stream with a non-zero mean
    gamma = torch.rand(D, generator=g).to(dev)
    x = x_in.clone()
    x16 = torch.empty(M, D, device=dev, dtype=torch.float16)
    stats = torch.zeros(M, parts, 2, device=dev)
    ops.gemm(a, w0, gamma=gamma, resid=x, out=x, out2=x16, out2_leaky=False, ln_stats_out=stats, ln_parts=parts, ln_part_cols=pc)
    xr = x_in.double() + gamma.double() * (a.double() @ w0.double().T)
    assert (x.double() - xr).abs().max().item() < 2e-4
    assert (x16.float() - x).abs().max().item() <= 2.0 ** -10 * x.abs().max().item()
    # merged statistics == row mean / variance
    mean_p, m2_p = stats[..., 0].double(), stats[..., 1].double()
    mean = mean_p.mean(1)
    var = (m2_p.sum(1) + pc * ((mean_p - mean[:, None]) ** 2).sum(1)) / D
    assert (mean - x.double().mean(1)).abs().max().item() < 1e-5
    assert ((var - x.double().var(1, unbiased=False)).abs() / x.double().var(1, unbiased=False)).max().item() < 1e-5
    # consumer
    lnw, lnb = (1 + 0.2 * torch.randn(D, generator=g)).to(dev), (0.1 * torch.randn(D, generator=g)).to(dev)
    w1 = (torch.randn(N2, D, generator=g) / 32).to(dev)
    b1 = torch.randn(N2, generator=g).to(dev)
    wf = (w1 * lnw).half()
    c1 = wf.float().sum(1).contiguous()
    c2 = (w1 @ lnb + b1).contiguous()
    y = ops.gemm(x16, wf.contiguous(), bias=c2, out_dtype=torch.float32, ln_stats_in=stats, ln_c1=c1, ln_parts=parts, ln_part_cols=pc,
                 ln_eps=1e-6)
    ref = torch.nn.functional.layer_norm(x.double(), (D,), lnw.double(), lnb.double(), 1e-6) @ w1.double().T + b1.double()
    err = ((y.double() - ref).abs().max() / ref.abs().max()).item()
    h = torch.nn.functional.layer_norm(x, (D,), lnw, lnb, 1e-6).half()
    plain = ops.gemm(h, w1.half().contiguous(), bias=b1, out_dtype=torch.float32)
    err_plain = ((plain.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"fused LN->Linear D={D}: max err / max|ref| {err:.2e} (stand-alone LayerNorm + GEMM: {err_plain:.2e})")
    assert err < 3 * max(err_plain, 3e-4)
