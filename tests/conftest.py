import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def rel_l2(a, b):
    import torch
    a = a.detach().float().cpu()
    b = b.detach().float().cpu()
    return float(torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b).clamp_min(1e-20))


@pytest.fixture
def rel():
    return rel_l2


class ThreadGroup:
    """TEST DOUBLE for a torch.distributed process group: R ranks as threads of this process.  `run(fn)` calls
    fn(rank) on R threads; while it runs, torch.distributed.all_to_all_single / barrier operate on this group through
    in-process buffers (with a device synchronisation around the exchange, so it also serves single-GPU tests of the
    engine's multi-rank code path).  Test infrastructure only."""

    def __init__(self, world, monkeypatch):
        import threading
        import torch
        import torch.distributed as dist
        self.world = world
        self.bar = threading.Barrier(world)
        self.slots = [None] * world
        self.tls = threading.local()
        group = self

        def sync():
            if torch.cuda.is_available():
                torch.cuda.synchronize()

        def a2a(recv, send, group=None, **kw):
            g, r = group, group.tls.rank
            sync()
            g.slots[r] = send
            g.bar.wait()
            chunk = send.numel() // g.world
            for s_ in range(g.world):
                recv.view(-1)[s_ * chunk:(s_ + 1) * chunk].copy_(g.slots[s_].view(-1)[r * chunk:(r + 1) * chunk])
            sync()
            g.bar.wait()

        def barrier(group=None, **kw):
            (group or self).bar.wait()

        monkeypatch.setattr(dist, "all_to_all_single", a2a)
        monkeypatch.setattr(dist, "barrier", barrier)

    def run(self, fn):
        import threading
        out, err = [None] * self.world, [None] * self.world

        def body(r):
            self.tls.rank = r
            try:
                out[r] = fn(r)
            except BaseException as e:          # noqa: BLE001 -- re-raised on the main thread
                err[r] = e
                self.bar.abort()

        ts = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for e in err:
            if e is not None:
                raise e
        return out
