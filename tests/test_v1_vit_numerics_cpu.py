"""UniDepthV1 ViT-L/14: the GPU's residual against the reference is f16 operand rounding, not logic (CPU, no kernel involved).

The V1 ViT-L intrinsics on the GT-K golden case measure 2.0e-4 on the GPU (tests/test_v1_vit_gpu.py::V1VIT_MEASURED), above
the 1e-4 that UniDepthV2 holds.  The model below is the fp32 oracle with ONE change in the encoder: every operand of the patch
embedding, the Linear layers and the attention products is rounded to f16 before the fp32 product, attention probabilities and
outputs are rounded to f16, and each block output is stored in f16 as the tap kernel stores it -- what the wgmma kernels are
fed (DESIGN.md section 2).  The decoder stays fp32, so the model is a LOWER bound of the rounding the GPU does.  It reproduces
the GT-K intrinsics error to within 10% (1.8e-4 against 2.0e-4 measured); the depth residual is mostly the decoder's."""
import json
import os

import torch
import torch.nn.functional as F

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _infer_with_f16_encoder_operands(sd, cfg, rgb, K):
    import unidepth_v1_vit_oracle as OV
    q16 = lambda t: t.to(torch.float16).to(torch.float32)
    lin, sdpa, conv, enc = OV._lin, OV._sdpa, F.conv2d, OV.vit_encoder_v1

    def lin16(x, s, prefix, bias=True):
        return F.linear(q16(x), q16(s[prefix + ".weight"]), s.get(prefix + ".bias") if bias else None)

    def sdpa16(q, k, v):
        q, k, v = q16(q), q16(k), q16(v)
        s = (q @ k.transpose(-1, -2)) / (q.shape[-1] ** 0.5)
        p = torch.exp(s - s.max(-1, keepdim=True).values)
        return q16((q16(p) @ v) / p.sum(-1, keepdim=True))

    def conv16(x, w, b=None, *a, **k):
        return conv(q16(x), q16(w), b, *a, **k)

    def enc16(sd_, image, *a, **k):
        F.conv2d = conv16                  # the patch embedding only: the decoder's convolutions stay fp32
        try:
            outs, cls = enc(sd_, image, *a, **k)
        finally:
            F.conv2d = conv
        return [q16(t) for t in outs], cls

    OV._lin, OV._sdpa, OV.vit_encoder_v1 = lin16, sdpa16, enc16
    try:
        return OV.infer_v1_vit(sd, cfg, rgb, K)
    finally:
        OV._lin, OV._sdpa, OV.vit_encoder_v1 = lin, sdpa, enc


def test_f16_encoder_operand_rounding_explains_the_gtk_intrinsics_error():
    from test_v1_vit_cpu import like_golden, v1_vit_case_inputs
    from test_v1_vit_gpu import V1VIT_MEASURED
    for name in ("v1_vitl14_480x640", "v1_vitl14_gtK_375x1242"):
        cfg, sd, rgb, K, meta, z = v1_vit_case_inputs(GOLD, name)
        out = _infer_with_f16_encoder_operands(sd, cfg, rgb, K)
        k, kr = out["intrinsics"], torch.from_numpy(z["intrinsics"])
        kerr = max(((k[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        rel = (like_golden(out["depth"], "depth", meta) - torch.from_numpy(z["depth"])).abs() / torch.from_numpy(z["depth"])
        arel = rel.mean().item()
        m_arel, _, m_k = V1VIT_MEASURED["golden_" + name]
        print(f"{name}: f16 encoder operands: depth ARel {arel:.2e} K {kerr:.2e} | measured on the GPU: {m_arel:.2e} {m_k:.2e} | "
              f"ratio {arel / m_arel:.2f} {kerr / m_k:.2f}")
        # a lower bound everywhere (the decoder's f16 GEMMs and convolutions, which dominate the depth residual, are not
        # modelled) ...
        assert 0.2 < kerr / m_k < 2.0 and 0.2 < arel / m_arel < 2.0, (name, kerr, arel)
        if m_k > 1e-4:
            # ... and where the intrinsics exceed 1e-4, encoder rounding alone accounts for most of them
            assert 0.5 < kerr / m_k < 2.0, (name, kerr, m_k)
