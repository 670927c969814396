"""Times the other hot-path kernels on BASELINE-config geometries (one H100) and prints achieved GB/s against
their algorithmic bytes (SURVEY.md section 8d): focal(+splat) fwd+bwd, edge aggregation, multi_pose / exct decode."""
import sys, json
import torch
sys.path.insert(0, '.')
from centernet_b200 import decode as D, losses as L

def timeit(fn, iters=20, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters

g = torch.Generator(device='cuda').manual_seed(317)
out = {}
B, C, H, W, M = 32, 80, 128, 128, 128
logits = torch.randn(B, C, H, W, device='cuda', generator=g) - 2.19
pred = torch.clamp(torch.sigmoid(logits), 1e-4, 1 - 1e-4).requires_grad_(True)
cls = torch.randint(0, C, (B, M), device='cuda', generator=g); cx = torch.randint(0, W, (B, M), device='cuda', generator=g)
cy = torch.randint(0, H, (B, M), device='cuda', generator=g); rad = torch.randint(0, 12, (B, M), device='cuda', generator=g)
val = torch.ones(B, M, dtype=torch.uint8, device='cuda')
gt = L.splat_gaussian(cls, cx, cy, rad, val, C, H, W)
n = B * C * H * W
ms = timeit(lambda: L.FocalSplatLoss()(pred, cls, cx, cy, rad, val))
out['focal_splat_fwd+grad B=32'] = dict(ms=ms, gbs=2 * n * 4 / ms / 1e6, alg_bytes=2 * n * 4, img_s=B / ms * 1e3)
ms = timeit(lambda: L._neg_loss(pred, gt))
out['focal_dense_gt_fwd+grad B=32'] = dict(ms=ms, gbs=4 * n * 4 / ms / 1e6, alg_bytes=4 * n * 4, img_s=B / ms * 1e3)
ms = timeit(lambda: L.splat_gaussian(cls, cx, cy, rad, val, C, H, W))
out['splat_gaussian B=32'] = dict(ms=ms, gbs=n * 4 / ms / 1e6, alg_bytes=n * 4)
heat = torch.sigmoid(logits)
ms = timeit(lambda: D._h_aggregate(heat, 0.1))
out['h_aggregate B=32'] = dict(ms=ms, gbs=2 * n * 4 / ms / 1e6, alg_bytes=2 * n * 4)
ms = timeit(lambda: D._v_aggregate(heat, 0.1))
out['v_aggregate B=32'] = dict(ms=ms, gbs=2 * n * 4 / ms / 1e6, alg_bytes=2 * n * 4)
# multi_pose B=64
Bp = 64
h1 = torch.sigmoid(torch.randn(Bp, 1, H, W, device='cuda', generator=g) - 2.19); wh = torch.rand(Bp, 2, H, W, device='cuda') * 32
kps = torch.randn(Bp, 34, H, W, device='cuda') * 6; reg = torch.rand(Bp, 2, H, W, device='cuda')
hm_hp = torch.sigmoid(torch.randn(Bp, 17, H, W, device='cuda', generator=g) - 1); hpo = torch.rand(Bp, 2, H, W, device='cuda')
ms = timeit(lambda: D.multi_pose_decode(h1, wh, kps, reg=reg, hm_hp=hm_hp, hp_offset=hpo, K=100))
out['multi_pose_decode B=64'] = dict(ms=ms, gbs=Bp * 1224448 / ms / 1e6, alg_bytes=Bp * 1224448, img_s=Bp / ms * 1e3)
# exct B=32, K=40
Be = 8
maps = [torch.sigmoid(torch.randn(Be, C, H, W, device='cuda', generator=g) - 2.19) for _ in range(5)]
regs = [torch.rand(Be, 2, H, W, device='cuda') for _ in range(4)]
ms = timeit(lambda: D.exct_decode(*maps, *regs, K=40, num_dets=1000), iters=5)
out['exct_decode K=40 B=8'] = dict(ms=ms, img_s=Be / ms * 1e3, gbs=Be * 26.27e6 / ms / 1e6, alg_bytes=Be * 26.27e6)
ms = timeit(lambda: D.exct_decode(*maps, *regs, K=100, num_dets=1000), iters=2, warm=1)
out['exct_decode K=100 B=8'] = dict(ms=ms, img_s=Be / ms * 1e3)
for k, v in out.items():
    print(k, json.dumps({a: (round(b, 3) if isinstance(b, float) else b) for a, b in v.items()}))
