"""One launch (after one warm-up) of every non-decode hot-path kernel at BASELINE-config geometries, for
`ncu --set full -k regex:k_` captures.  Not a benchmark: numbers under ncu are never bench values."""
import sys
import torch
sys.path.insert(0, '.')
from centernet_b200 import decode as D, losses as L
from centernet_b200.dcn_v2_func import DCNv2Function

g = torch.Generator(device='cuda').manual_seed(317)
B, C, H, W, M = 32, 80, 128, 128, 128
logits = torch.randn(B, C, H, W, device='cuda', generator=g) - 2.19
pred = torch.clamp(torch.sigmoid(logits), 1e-4, 1 - 1e-4).requires_grad_(True)
cls = torch.randint(0, C, (B, M), device='cuda', generator=g); cx = torch.randint(0, W, (B, M), device='cuda', generator=g)
cy = torch.randint(0, H, (B, M), device='cuda', generator=g); rad = torch.randint(0, 12, (B, M), device='cuda', generator=g)
val = torch.ones(B, M, dtype=torch.uint8, device='cuda')
heat = torch.sigmoid(logits)
Bp = 64
h1 = torch.sigmoid(torch.randn(Bp, 1, H, W, device='cuda', generator=g) - 2.19); wh = torch.rand(Bp, 2, H, W, device='cuda') * 32
kps = torch.randn(Bp, 34, H, W, device='cuda') * 6; reg = torch.rand(Bp, 2, H, W, device='cuda')
hm_hp = torch.sigmoid(torch.randn(Bp, 17, H, W, device='cuda', generator=g) - 1); hpo = torch.rand(Bp, 2, H, W, device='cuda')
Be = 8
maps = [torch.sigmoid(torch.randn(Be, C, H, W, device='cuda', generator=g) - 2.19) for _ in range(5)]
regs = [torch.rand(Be, 2, H, W, device='cuda') for _ in range(4)]
ind = torch.randint(0, H * W, (B, M), device='cuda', generator=g); tgt = torch.rand(B, M, 2, device='cuda'); rmask = torch.ones(B, M, dtype=torch.uint8, device='cuda')
out2 = torch.randn(B, 2, H, W, device='cuda', requires_grad=True)
# DCN layer 64@128x128 -> 64, B=16 (largest dla_34 layer)
Bd = 16
x = torch.randn(Bd, 64, H, W, device='cuda', generator=g, requires_grad=True)
off = (torch.randn(Bd, 18, H, W, device='cuda', generator=g) * 2).requires_grad_(True)
msk = torch.sigmoid(torch.randn(Bd, 9, H, W, device='cuda', generator=g)).requires_grad_(True)
wgt = (torch.randn(64, 64, 3, 3, device='cuda', generator=g) / 24).requires_grad_(True)
bias = torch.zeros(64, device='cuda', requires_grad=True)
for rep in range(2):
    gt = L.splat_gaussian(cls, cx, cy, rad, val, C, H, W)
    L.FocalSplatLoss()(pred, cls, cx, cy, rad, val).backward()
    L._neg_loss(pred, gt).backward()
    L.RegL1Loss()(out2, rmask, ind, tgt).backward()
    D._h_aggregate(heat, 0.1); D._v_aggregate(heat, 0.1)
    D.multi_pose_decode(h1, wh, kps, reg=reg, hm_hp=hm_hp, hp_offset=hpo, K=100)
    D.exct_decode(*maps, *regs, K=40, num_dets=1000)
    y = DCNv2Function(1, 1, 1, 1)(x, off, msk, wgt, bias)
    y.sum().backward()
    torch.cuda.synchronize()
print('ok')
