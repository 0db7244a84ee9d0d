"""Device time of a link's send + receive pair on a loop-back link: 24 pairs per CUDA graph, CUDA events."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pipeedge_b200 import _lib   # noqa: E402  pylint: disable=wrong-import-position
from pipeedge_b200._lib import LIB, check   # noqa: E402  pylint: disable=wrong-import-position

dev = torch.device('cuda', 0)
for label, shape, bit, with_b in (('raw 8x197x768', (8, 197, 768), 0, False), ('raw+add 8x197x768', (8, 197, 768), 0, True),
                                  ('q8 32x198x768 a+b', (32, 198, 768), 8, True), ('raw 32x128x768', (32, 128, 768), 0, False)):
    a = torch.randn(shape, device=dev)
    b = torch.randn(shape, device=dev)
    dst = torch.empty_like(a)
    items, n = shape[0], shape[1] * shape[2]
    h = ctypes.c_void_p()
    check(LIB.pe_link_open_local(a.numel() * 4 + 4096, 4, bit, ctypes.byref(h)))
    side = torch.cuda.Stream()

    def pair():
        s = torch.cuda.current_stream().cuda_stream
        check(LIB.pe_link_put(h, a.data_ptr(), b.data_ptr() if with_b else None, n, None, None, 0, items, bit,
                              _lib.PE_CLAMP_AUTO if bit else 0, s))
        check(LIB.pe_link_get(h, dst.data_ptr(), None, items, n, 0, s))
    with torch.cuda.stream(side):
        for _ in range(3):
            pair()
        side.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            for _ in range(24):
                pair()
    torch.cuda.synchronize()
    for _ in range(3):
        g.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(10):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    us = s.elapsed_time(e) * 1e3 / 240
    print(f"  {label}: {us:.2f} us per put + wait + get", flush=True)
    LIB.pe_link_close(h)
