"""CPU restatement of the reference DCNv2 op (TEST INFRASTRUCTURE).

Follows src/lib/models/networks/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:
  dmcn_im2col_bilinear :18-47, modulated_deformable_im2col_gpu_kernel :118-180
and the host loop of src/dcn_v2_cuda.c:61-97 (bias + W . col).  Written with differentiable
torch ops in float64 so that torch.autograd supplies the reference gradients (the CUDA backward
of the reference uses fp32 atomics and is not bit-reproducible, SURVEY.md section 7).

Pinned by: the zero-offset known-answer test of DCNv2/test.py:32-65 (tests/test_dcn_oracle.py)
and a cross-check against torchvision.ops.deform_conv2d (third party, same offset layout).
"""
import torch


def _pair(v):
    return (int(v[0]), int(v[1])) if isinstance(v, (tuple, list)) else (int(v), int(v))


def dcn_v2_forward(x, offset, mask, weight, bias, stride=1, padding=1, dilation=1, deformable_groups=1):
    """stride, padding and dilation are ints or (h, w) pairs (the C ABI's anisotropic form)."""
    x = x.double(); offset = offset.double(); mask = mask.double(); weight = weight.double()
    B, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1      # dcn_v2_cuda.c:40-41
    Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    KT = kh * kw
    dg = deformable_groups
    cpg = Cin // dg
    hs = (torch.arange(Ho, dtype=torch.float64) * sh - ph).view(1, Ho, 1)
    ws = (torch.arange(Wo, dtype=torch.float64) * sw - pw).view(1, 1, Wo)
    cols = []
    xf = x.reshape(B, Cin, H * W)
    for g in range(dg):
        xg = xf[:, g * cpg:(g + 1) * cpg]
        for t in range(KT):
            i, j = t // kw, t % kw
            dy = offset[:, g * 2 * KT + 2 * t]            # :155-159 (2t = h, 2t+1 = w)
            dx = offset[:, g * 2 * KT + 2 * t + 1]
            m = mask[:, g * KT + t]
            h_im = hs + i * dh + dy                       # B,Ho,Wo
            w_im = ws + j * dw + dx
            inside = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)     # :165
            h_low = torch.floor(h_im); w_low = torch.floor(w_im)
            lh = h_im - h_low; lw = w_im - w_low
            hh = 1 - lh; hw = 1 - lw
            h_low = h_low.long(); w_low = w_low.long(); h_high = h_low + 1; w_high = w_low + 1

            def corner(hi, wi, ok):
                # an out-of-range corner is never read (v = 0): a select, so a NaN / Inf that the clamped index
                # happens to hit stays out of the sum (v * ok would give NaN * 0 = NaN)
                ok = ok & inside
                idx = (hi.clamp(0, H - 1) * W + wi.clamp(0, W - 1)).view(B, 1, Ho * Wo).expand(B, cpg, Ho * Wo)
                v = xg.gather(2, idx).view(B, cpg, Ho, Wo)
                return torch.where(ok.unsqueeze(1), v, 0.0)

            v1 = corner(h_low, w_low, (h_low >= 0) & (w_low >= 0))            # :31-41
            v2 = corner(h_low, w_high, (h_low >= 0) & (w_high <= W - 1))
            v3 = corner(h_high, w_low, (h_high <= H - 1) & (w_low >= 0))
            v4 = corner(h_high, w_high, (h_high <= H - 1) & (w_high <= W - 1))
            val = (hh * hw).unsqueeze(1) * v1 + (hh * lw).unsqueeze(1) * v2 + \
                  (lh * hw).unsqueeze(1) * v3 + (lh * lw).unsqueeze(1) * v4   # :43-46
            # outside samples: val stays 0 (:160-168) even where a NaN / Inf offset made the corner weights NaN;
            # val * m is stored for them too (:174), so a NaN mask gives NaN there
            val = torch.where(inside.unsqueeze(1), val, 0.0)
            cols.append((val * m.unsqueeze(1), g, t))                          # :174
    # col[b, c, t, p] ordered as the weight's (c, kh, kw) axes
    col = torch.zeros(B, Cin, KT, Ho, Wo, dtype=torch.float64)
    full = []
    for g in range(dg):
        per_t = [c for c, gg, _ in cols if gg == g]
        full.append(torch.stack(per_t, dim=2))                                 # B,cpg,KT,Ho,Wo
    col = torch.cat(full, dim=1)
    out = torch.einsum("ock,bckp->bop", weight.reshape(Cout, Cin, KT), col.reshape(B, Cin, KT, Ho * Wo))
    out = out.view(B, Cout, Ho, Wo)
    if bias is not None:
        out = out + bias.double().view(1, Cout, 1, 1)                          # dcn_v2_cuda.c:72-78
    return out
