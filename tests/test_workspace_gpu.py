"""The scratch cache every host wrapper uses (_native._workspace): one buffer per (device, stream) in the caller's pool,
grown on demand; while the stream is being captured into a CUDA graph, a graph-pool buffer that the pool never sees."""
import pytest
import torch

from deepi2p_b200._native import _workspace

pytestmark = pytest.mark.gpu


def test_eager_buffers_are_cached_per_device_and_stream_and_grow(cuda):
    pool = {}
    side = torch.cuda.Stream(device=cuda)
    cur = torch.cuda.current_stream(cuda).cuda_stream
    a = _workspace(pool, 100, cuda)
    assert a.numel() == 1 << 20 and a.device == cuda                 # the default floor
    assert _workspace(pool, 1 << 20, cuda) is a
    assert _workspace(pool, 0, torch.device("cuda")) is a            # no index: the current device
    b = _workspace(pool, 100, cuda, side)
    assert b is not a and _workspace(pool, 100, cuda, side) is b
    with torch.cuda.stream(side):
        assert _workspace(pool, 100, cuda) is b                      # None: the current stream
    c = _workspace(pool, (1 << 20) + 1, cuda)
    assert c.numel() == (1 << 20) + 1 and _workspace(pool, 100, cuda) is c
    assert pool == {(cuda.index, cur): c, (cuda.index, side.cuda_stream): b}
    exact = {}
    assert _workspace(exact, 12, cuda, floor=0).numel() == 12
    assert _workspace(exact, 4, cuda, floor=0).numel() == 12


def test_a_capturing_stream_gets_a_graph_buffer_that_is_not_cached(cuda):
    pool = {}
    s = torch.cuda.Stream(device=cuda)
    key = (cuda.index, s.cuda_stream)
    eager = _workspace(pool, 100, cuda, s)
    s.wait_stream(torch.cuda.current_stream(cuda))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        captured = _workspace(pool, 2 << 20, cuda, s)
        captured.fill_(7)
    assert captured.numel() == 2 << 20 and captured.data_ptr() != eager.data_ptr()
    assert pool == {key: eager}                    # neither cached nor did it replace the eager buffer
    later = _workspace(pool, 2 << 20, cuda, s)     # an eager call after the capture grows its own buffer
    assert later is not captured and later.data_ptr() != captured.data_ptr() and pool == {key: later}
    g.replay()
    torch.cuda.synchronize()
    assert bool((captured == 7).all())
