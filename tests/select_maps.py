"""Seeded score maps for the selection tests (tests/test_select_oracle*.py): one generator per distribution that
makes the peak-NMS + top-K selection take a different branch.  Every map is float32 and is built on the device
it is asked for, so the GPU tests make their large batches in place."""
import torch

KINDS = ["noise", "blobs", "ties", "plateau", "zero", "few", "negative", "neg_const", "mixed", "tiny", "huge", "ramp"]


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def make_map(kind, B, C, H, W, seed=0, device="cpu"):
    g = _gen(seed, device)
    shape = (B, C, H, W)
    rand = lambda: torch.rand(shape, generator=g, device=device)
    if kind == "noise":        # head-like: most scores small, a long tail (bench.py's input)
        return torch.sigmoid(torch.randn(shape, generator=g, device=device) - 2.19)
    if kind == "blobs":        # saturated Gaussian blobs, a few per image: 1.0 plateaus, < K peaks in most classes
        hm = rand() * 0.01
        ys = torch.arange(H, device=device, dtype=torch.float32).view(H, 1)
        xs = torch.arange(W, device=device, dtype=torch.float32).view(1, W)
        for b in range(B):
            for _ in range(6):
                c = int(torch.randint(0, C, (1,), generator=g, device=device))
                cy, cx = (torch.rand(2, generator=g, device=device) * torch.tensor([H, W], device=device)).tolist()
                r = 1.0 + float(torch.rand(1, generator=g, device=device)) * max(H, W) / 8
                blob = torch.clamp(1.4 * torch.exp(-((ys - cy) ** 2 + (xs - cx) ** 2) / (2 * r * r)), max=1.0)
                hm[b, c] = torch.maximum(hm[b, c], blob)
        return hm
    if kind == "ties":         # quantised: equal peaks across classes and CTAs
        return torch.randint(0, 9, shape, generator=g, device=device).float() / 8
    if kind == "plateau":      # every pixel a peak of one score: overflows every buffer
        return torch.full(shape, 0.5, device=device)
    if kind == "zero":
        return torch.zeros(shape, device=device)
    if kind == "few":          # fewer than K positive peaks per image: zero fillers in index order
        hm = torch.zeros(shape, device=device)
        n = max(1, min(40, C * H * W // 16))
        idx = torch.randint(0, C * H * W, (B, n), generator=g, device=device)
        val = torch.rand((B, n), generator=g, device=device) * 0.9 + 0.05
        return hm.view(B, -1).scatter_(1, idx, val).view(shape)
    if kind == "negative":     # every score negative: non-peak zeros outrank every negative peak
        return -torch.sigmoid(torch.randn(shape, generator=g, device=device) - 2.19)
    if kind == "neg_const":    # no zeros at all: the fill ranks negatives, ties by index
        return torch.full(shape, -0.25, device=device)
    if kind == "mixed":        # mostly negative, rare positives, some -0.0 pixels (peaks among negatives): +0 and -0
        v = torch.sigmoid(torch.randn(shape, generator=g, device=device) - 2.19) - 0.9     # fillers interleave
        return torch.where(rand() < 0.05, torch.full_like(v, -0.0), v)
    if kind == "tiny":         # every positive peak below 2^-16, part of them fp32 subnormals: histogram bin 0
        v = rand() * 1e-5
        sub = rand() < 0.3
        return torch.where(sub, v * 1e-33, v)
    if kind == "huge":         # scores in [1, 1e30]: all in the top histogram bin
        return torch.pow(10.0, rand() * 30.0)
    if kind == "ramp":         # every plane brighter than all before it: stale threshold, overflow, flush rescan
        ramp = torch.linspace(0.01, 0.99, C, device=device).view(1, C, 1, 1)
        return rand() * 0.01 + ramp
    raise ValueError(kind)


def ulp_neighbours(B, C, H, W, centres, seed=0, device="cpu", spread=8):
    """Logit maps whose values sit within `spread` ulps of one centre per class (the sigmoid maps many of them to
    one float: peaks by collision)."""
    g = _gen(seed, device)
    cen = torch.tensor(centres, dtype=torch.float32, device=device)
    pick = cen[torch.arange(C, device=device) % len(centres)].view(1, C, 1, 1).expand(B, C, H, W)
    step = torch.randint(-spread, spread + 1, (B, C, H, W), generator=g, device=device, dtype=torch.int32)
    return (pick.contiguous().view(torch.int32) + step).view(torch.float32)


def poison(hm, seed=0, density=4, inf_stride=16):
    """Writes NaN / +inf / -inf into every plane of hm (in place, any float dtype): at the four corners, at lane
    edges of a few rows (x = 0, 3, 4 and W-1), a 2x2 +inf plateau, a 3x3 -inf block (its centre is a -inf peak)
    and `density` more at random places.  Every plane gets them, so the planes on both sides of every CTA boundary
    do too; +inf only goes into the planes of classes c % inf_stride == 0 (NaN in the others), so that the +inf
    peaks do not fill the whole top-K."""
    B, C, H, W = hm.shape
    g = _gen(seed, "cpu")
    nan, pinf, ninf = float("nan"), float("inf"), float("-inf")
    pat = torch.zeros(H, W)
    mask = torch.zeros(H, W, dtype=torch.bool)

    def put(y, x, v):
        pat[y, x] = v
        mask[y, x] = True

    for (y, x), v in zip([(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)], (nan, pinf, ninf, nan)):
        put(y, x, v)
    for j, x in enumerate(sorted({0, min(3, W - 1), min(4, W - 1), W - 1})):
        put(1 + (5 * j + seed) % max(1, H - 2), x, (ninf, nan, pinf, nan)[j % 4])
    if H >= 6 and W >= 8:
        xa, xb = W // 3, W // 2
        pat[1:3, xa:xa + 2] = pinf; mask[1:3, xa:xa + 2] = True
        pat[H - 3:H, xb - 1:xb + 2] = ninf; mask[H - 3:H, xb - 1:xb + 2] = True
        put(H // 2, 1, nan)
    for _ in range(density):
        y = int(torch.randint(0, H, (1,), generator=g)); x = int(torch.randint(0, W, (1,), generator=g))
        put(y, x, (nan, pinf, ninf)[int(torch.randint(0, 3, (1,), generator=g))])
    with_inf = (torch.arange(C) % inf_stride == 0).view(1, C, 1, 1)
    planes = torch.where(with_inf, pat, torch.where(pat == pinf, torch.full_like(pat, nan), pat))
    hm.copy_(torch.where(mask.to(hm.device), planes.to(device=hm.device, dtype=hm.dtype), hm))
    return hm
