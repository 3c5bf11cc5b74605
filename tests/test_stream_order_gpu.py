"""Stage entries whose temporaries live only for one call (resid_ln_linear_f16, person_post, anny_person_post,
refine_chain) are asynchronous on the caller's stream: their scratch is allocated, used and freed in that stream's
order, and nothing waits for the device.  Each entry is called several times in a row on a side stream, each call
right behind the kernel that writes its input, all queued behind a long-running kernel.  The calls must return before
that stream has run, and every call must give the bits of a call on the current stream; a scratch freed before its
kernels had run would be reused by the next call and show up as wrong bits."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

REPEATS = 3
SLEEP_CYCLES = 1_000_000_000  # about half a second of device work at the H100's clocks


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _resid_ln_linear(dev):
    from multihmr_b200 import ops

    g = _gen(1)
    M, D, N, Ka = 1370, 384, 1536, 384
    a = torch.randn(M, Ka, generator=g).to(dev).half()
    wp = (torch.randn(D, Ka, generator=g) / math.sqrt(Ka)).to(dev).half()
    bp, ls = (torch.randn(D, generator=g) * 0.1).to(dev), (torch.rand(D, generator=g) * 0.5 + 0.1).to(dev)
    ln_g, ln_b = (torch.rand(D, generator=g) + 0.5).to(dev), (torch.randn(D, generator=g) * 0.2).to(dev)
    w, b = (torch.randn(N, D, generator=g) / math.sqrt(D)).to(dev), (torch.randn(N, generator=g) * 0.1).to(dev)
    x0 = (torch.randn(M, D, generator=g) * 1.5 + 0.7).to(dev)

    def run(x):
        out = ops.resid_ln_linear_f16(a, wp, bp, ls, x, ln_g, ln_b, w, b, gelu=True)
        return x, out

    return x0, run


def _person_post(dev):
    from multihmr_b200 import ops

    g = _gen(2)
    nb, Pm, B, S = 10, 8, 3, 448
    dec0 = torch.randn(Pm, 318 + nb + 13, generator=g).to(dev)
    offset = (torch.rand(Pm, 2, generator=g) - 0.5).to(dev)
    K = torch.zeros(B, 3, 3)
    K[:, 0, 0] = K[:, 1, 1] = torch.tensor([400.0, 650.0, 900.0])
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 224.0, 230.0, 1.0
    K = K.to(dev)
    det_b = torch.tensor([0, 0, 1, 2, 2, 2, 0, 0], dtype=torch.int32, device=dev)
    det_y = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32).to(dev)
    det_x = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32).to(dev)
    count = torch.tensor([6], dtype=torch.int32, device=dev)
    focal_norm = S / (2 * math.tan(math.radians(30)))

    def run(dec):
        return tuple(ops.person_post(dec, nb, offset, K, det_b, det_y, det_x, count, Pm, focal_norm).values())

    return dec0, run


def _anny_person_post(dev):
    from multihmr_b200 import ops

    g = _gen(3)
    J, nb, Pm, B, S, D = 163, 11, 8, 3, 448, 384
    hid0 = torch.randn(B, D, generator=g).to(dev)
    w2, b2 = (torch.randn(D, generator=g) / math.sqrt(D)).to(dev), torch.tensor([0.1], device=dev)
    fov_max = torch.tensor([2.2], device=dev)
    rot6d = torch.randn(Pm, 6 * J, generator=g).to(dev)
    useful = torch.tensor([0.0, 0.3, 1.0])[torch.arange(J) % 3].to(dev)
    shape0 = (torch.randn(Pm, nb, generator=g) * 3).to(dev)
    offset = (torch.rand(Pm, 2, generator=g) - 0.5).to(dev)
    dist_pp = torch.randn(Pm, generator=g).to(dev)
    det_b = torch.tensor([0, 1, 1, 2, 2, 0, 0, 0], dtype=torch.int32, device=dev)
    det_y = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32).to(dev)
    det_x = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32).to(dev)
    count = torch.tensor([5], dtype=torch.int32, device=dev)

    def run(hid):  # K = None: every person's outputs go through the camera regressed from hid
        o = ops.anny_person_post(hid, w2, b2, fov_max, None, S, rot6d, J, useful, shape0.clone(), offset, dist_pp,
                                 det_b, det_y, det_x, count, Pm)
        return tuple(o.values())

    return hid0, run


def _refine_chain(dev):
    from multihmr_b200 import ops

    g = torch.Generator(device=dev).manual_seed(4)
    D, depth, R, Pm = 384, 4, 300, 12
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    L = {"Wproj": r(depth, D, D) / math.sqrt(D), "bproj": r(depth, D) * 0.1,
         "ls1": torch.rand(depth, D, device=dev, generator=g) * 0.5 + 0.1,
         "ln2_g": torch.rand(depth, D, device=dev, generator=g) + 0.5, "ln2_b": r(depth, D) * 0.2,
         "Wfc1": r(depth, 4 * D, D) / math.sqrt(D), "bfc1": r(depth, 4 * D) * 0.1,
         "Wfc2": r(depth, D, 4 * D) / math.sqrt(4 * D), "bfc2": r(depth, D) * 0.1,
         "ls2": torch.rand(depth, D, device=dev, generator=g) * 0.5 + 0.1}
    o16 = r(depth, R, D).half()
    rowidx = torch.randperm(R, device=dev, generator=g)[:Pm].int()
    count = torch.tensor([9], dtype=torch.int32, device=dev)
    x0 = r(Pm, D) * 1.5 + 0.7

    def run(x):
        return (ops.refine_chain(L, o16, rowidx, count, x),)

    return x0, run


@pytest.mark.parametrize("case", [_resid_ln_linear, _person_post, _anny_person_post, _refine_chain],
                         ids=["resid_ln_linear_f16", "person_post", "anny_person_post", "refine_chain"])
def test_entry_is_stream_ordered(cuda_device, case):
    src, run = case(cuda_device)
    want = run(src.clone())
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        got = [run(src.clone()) for _ in range(REPEATS)]  # clone: the kernel that writes the input, on `side`
        returned_early = not side.query()
    side.synchronize()
    assert returned_early, "the calls waited for their stream"
    for out in got:
        assert len(out) == len(want)
        for a, b in zip(out, want):
            assert torch.equal(a, b)
