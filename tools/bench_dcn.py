"""Times the DCNv2 forward/backward kernels on dla_34-style layers (H100): wgmma (3xTF32) forward vs the
fp32 CUDA-core forward vs torchvision.ops.deform_conv2d (if present), and checks them against each other."""
import sys, time
import torch
sys.path.insert(0, '.')
from centernet_b200._lib import C, ptr, stream_ptr, workspace

def run(B, Cin, H, W, Cout, iters=20):
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    off = torch.randn(B, 18, H, W, device='cuda', generator=g) * 2
    msk = torch.sigmoid(torch.randn(B, 9, H, W, device='cuda', generator=g))
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) / (3 * Cin ** 0.5)
    bias = torch.randn(Cout, device='cuda', generator=g)
    out_tc = torch.empty(B, Cout, H, W, device='cuda'); out_fp = torch.empty_like(out_tc)
    nb = C.dcnv2_workspace_bytes(B, Cin, Cout, H, W, 3, 3, 1, 1, 1, 1)
    ws = workspace(nb, x.device)
    s = stream_ptr(x)
    def tc(): C.dcnv2_forward(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(bias), ptr(out_tc), B, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1, 1, 1, 1, ptr(ws), ws.numel(), s)
    def fp(): C.dcnv2_forward(ptr(x), ptr(off), ptr(msk), ptr(w), ptr(bias), ptr(out_fp), B, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1, 1, 1, 1, 0, 0, s)
    res = {}
    for name, fn in (('wgmma_3xtf32', tc), ('fp32_cuda_core', fp)):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters): fn()
        e1.record(); torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / iters
    try:
        from torchvision.ops import deform_conv2d
        for _ in range(3): ref = deform_conv2d(x, off, w, bias, padding=1, mask=msk)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters): ref = deform_conv2d(x, off, w, bias, padding=1, mask=msk)
        e1.record(); torch.cuda.synchronize()
        res['torchvision'] = e0.elapsed_time(e1) / iters
        err_tv = (out_fp - ref).abs().max().item()
    except Exception as e:
        err_tv = str(e)[:40]
    # forward + backward through autograd (this library: wgmma forward + fp32 backward kernels)
    try:
        from centernet_b200.dcn_v2_func import DCNv2Function
        from torchvision.ops import deform_conv2d
        leaves = [t.clone().requires_grad_(True) for t in (x, off, msk, w, bias)]
        fn = DCNv2Function(1, 1, 1, 1)
        def ours():
            for t in leaves: t.grad = None
            fn(*leaves).sum().backward()
        def tv():
            for t in leaves: t.grad = None
            deform_conv2d(leaves[0], leaves[1], leaves[3], leaves[4], padding=1, mask=leaves[2]).sum().backward()
        for name, f in (('fwd+bwd_ours', ours), ('fwd+bwd_torchvision', tv)):
            for _ in range(2): f()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5): f()
            e1.record(); torch.cuda.synchronize()
            res[name] = e0.elapsed_time(e1) / 5
    except Exception as e:
        res['fwd+bwd_error'] = -1.0
        print('fwd+bwd timing failed:', str(e)[:100])
    flops = 2.0 * Cout * Cin * 9 * H * W * B
    print('B=%d %d@%dx%d->%d: ' % (B, Cin, H, W, Cout) + ', '.join('%s %.3f ms (%.1f TFLOP/s)' % (k, v, flops / v / 1e9) for k, v in res.items()),
          '| max|tc-fp32| = %.2e, max|fp32-tv| = %s' % ((out_tc - out_fp).abs().max().item(), err_tv))

if __name__ == '__main__':
    for shp in [(16, 64, 128, 128, 64), (16, 128, 64, 64, 128), (16, 256, 32, 32, 256), (16, 512, 16, 16, 256), (64, 64, 128, 128, 64)]:
        run(*shp)
