"""Back-to-back hot decodes overlap: k_select_hot is launched as a programmatic dependent of the previous launch on
its stream and keeps its per-image tickets in per-stream library storage that every launch leaves zero.  Every chain
below runs without synchronisation between calls and must return, bit for bit, what the same calls return when run
one at a time with a torch.cuda.synchronize() after each."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _maps(B, seed, C=80, logits=False, dt=torch.float32):
    """bench.py's synthetic heads (heat = sigmoid(randn - 2.19), wh = rand * 32, reg = rand)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, C, 128, 128, device="cuda", generator=g) - 2.19
    heat = x if logits else torch.sigmoid(x)
    wh = torch.rand(B, 2, 128, 128, device="cuda", generator=g) * 32
    reg = torch.rand(B, 2, 128, 128, device="cuda", generator=g)
    return heat.to(dt), wh.to(dt), reg.to(dt)


def _call(m, logits=False, K=100):
    from centernet_b200 import decode as D
    fn = D.ctdet_decode_from_logits if logits else D.ctdet_decode
    return lambda: fn(m[0], m[1], reg=m[2], K=K)


def _serial(calls):
    out = []
    for f in calls:
        out.append(f())
        torch.cuda.synchronize()
    return out


def _chain(calls):
    out = [f() for f in calls]
    torch.cuda.synchronize()
    return out


def _same(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), "call %d of the chain differs from its serial run" % i


def test_long_chain_bench_batches_and_small_batches():
    """>= 200 calls: the three bench batches (B = 64) interleaved with B = 1 and 8 (small-batch plan, images
    finalized from shared memory and multi-segment finalizes)."""
    from centernet_b200._lib import C
    bench = [_maps(64, 317 + i) for i in range(3)]
    small = [_maps(1, 11), _maps(8, 12)]
    order = []
    for i in range(210):
        order.append(bench[i % 3] if i % 3 != 2 else small[(i // 3) % 2])
    calls = [_call(m) for m in order]
    want = _serial(calls)
    l0 = C.launch_count()
    got = _chain(calls)
    assert C.launch_count() - l0 == len(calls), "one launch per call"
    _same(got, want)


def test_chain_mixes_fp32_half_and_logits():
    specs = [(torch.float32, False), (torch.bfloat16, False), (torch.float32, True), (torch.bfloat16, True),
             (torch.float16, False), (torch.float16, True)]
    maps = [(_maps(64, 500 + i, logits=lg, dt=dt), lg) for i, (dt, lg) in enumerate(specs)]
    calls = [_call(*maps[i % len(maps)]) for i in range(60)]
    _same(_chain(calls), _serial(calls))


def test_workspace_of_each_call_aliases_the_previous_one():
    """The C entry point with the workspace freed and reallocated per call (the caching allocator hands back the same
    block), and with one workspace shared by every call, filled with garbage first."""
    from centernet_b200._lib import C
    bats = [_maps(64, 317 + i) for i in range(3)] + [_maps(8, 40)]
    nbytes = max(C.topk_workspace_bytes(m[0].shape[0], 80, 128, 128, 100) for m in bats)
    shared = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def run(m, ws):
        dets = torch.empty((m[0].shape[0], 100, 6), dtype=torch.float32, device="cuda")
        C.ctdet_decode(m[0].data_ptr(), m[1].data_ptr(), m[2].data_ptr(), 0, m[0].shape[0], 80, 128, 128, 100,
                       dets.data_ptr(), ws.data_ptr(), ws.numel(), st)   # raises on an error status
        return dets

    want = _serial([(lambda m=m: run(m, torch.empty(nbytes, dtype=torch.uint8, device="cuda"))) for m in bats])
    ptrs, got = set(), []
    for i in range(40):
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        ptrs.add(ws.data_ptr())
        got.append(run(bats[i % 4], ws))
        del ws
    for i in range(40):
        got.append(run(bats[i % 4], shared))
    torch.cuda.synchronize()
    assert len(ptrs) == 1, "the workspaces did not alias"
    _same(got, [want[i % 4] for i in range(80)])


def test_torch_kernel_rewrites_the_next_heat_map_in_place():
    srcs = [_maps(64, 317 + i) for i in range(3)]
    buf = srcs[0][0].clone()
    want = [_call(m)() for m in srcs]
    torch.cuda.synchronize()
    from centernet_b200 import decode as D
    got = []
    for i in range(30):
        buf.copy_(srcs[i % 3][0])
        got.append(D.ctdet_decode(buf, srcs[i % 3][1], reg=srcs[i % 3][2], K=100))
    torch.cuda.synchronize()
    _same(got, [want[i % 3] for i in range(30)])


def test_two_streams_decode_at_once():
    bats = [_maps(64, 317 + i) for i in range(3)] + [_maps(8, 60), _maps(1, 61)]
    want = _serial([_call(m) for m in bats])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    g1, g2 = [], []
    for i in range(40):
        with torch.cuda.stream(s1):
            g1.append(_call(bats[i % 5])())
        with torch.cuda.stream(s2):
            g2.append(_call(bats[(i + 2) % 5])())
    torch.cuda.synchronize()
    _same(g1, [want[i % 5] for i in range(40)])
    _same(g2, [want[(i + 2) % 5] for i in range(40)])


def test_new_stream_after_default_stream_and_growing_image_count():
    """A chain on the default stream, then one on a fresh stream whose image count grows mid-chain (400 and then 1000
    two-class images: their ticket arrays outgrow the first one while earlier launches are still in flight)."""
    small, bench = _maps(8, 70), _maps(64, 317)
    many, more = _maps(400, 71, C=2), _maps(1000, 72, C=2)
    order = [small, bench, many, small, more, bench, many, more, small]
    want = _serial([_call(m) for m in order])
    got = _chain([_call(m) for m in order])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got2 = [_call(m)() for m in order * 3]
    torch.cuda.synchronize()
    _same(got, want)
    _same(got2, want * 3)
