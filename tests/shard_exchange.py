"""A stand-in for retrieval.ShardExchange that runs W ranks of a sharded protocol on one device, for the GPU tests of
the sharded paths (the streamed passes and the row-blocked re-ranking)."""
import threading

import torch

_EMPTY = object()


class Shards:
    """W ranks of the protocol on one device, in W threads that run one at a time: a rank runs until its next exchange,
    leaves its part there and hands over to the next rank; the exchange returns once every rank's part is in."""

    def __init__(self, world):
        self.world = world
        self.cv = threading.Condition()
        self.turn = 0
        self.slots = []

    def run(self, fn):
        """fn(exchange) on every rank; returns the per-rank results, re-raising the first rank's error."""
        out, errs = [None] * self.world, [None] * self.world

        def worker(rank):
            with self.cv:
                self.cv.wait_for(lambda: self.turn == rank)
            try:
                out[rank] = fn(Exchange(self, rank))
            except BaseException as e:  # noqa: BLE001 -- re-raised below
                errs[rank] = e
            finally:
                with self.cv:
                    self.turn = (rank + 1) % self.world
                    self.cv.notify_all()

        threads = [threading.Thread(target=worker, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        self.errors = errs
        for e in errs:
            if e is not None:
                raise e
        return out


class Exchange:
    """One rank's view of `Shards`, with the methods of retrieval.ShardExchange."""

    def __init__(self, shards, rank):
        self.s, self.rank, self.world, self.calls = shards, rank, shards.world, 0

    def _all(self, part):
        s = self.s
        with s.cv:
            if len(s.slots) <= self.calls:
                s.slots.append([_EMPTY] * self.world)
            slot = s.slots[self.calls]
            slot[self.rank] = part
            self.calls += 1
            s.turn = (self.rank + 1) % self.world
            s.cv.notify_all()
            if not s.cv.wait_for(lambda: s.turn == self.rank and all(p is not _EMPTY for p in slot), timeout=600):
                raise RuntimeError(f"rank {self.rank}: exchange {self.calls - 1} never completed")
            return list(slot)

    def objects(self, obj):
        return self._all(obj)

    def rows(self, t, counts):
        parts = self._all(t)
        assert [p.shape[0] for p in parts] == list(counts)
        return torch.cat(parts)

    def max_(self, t):
        parts = self._all(t.clone())
        return t.copy_(torch.stack(parts).amax(0))

    def sum_(self, t):
        parts = self._all(t.clone())
        return t.copy_(torch.stack(parts).sum(0, dtype=t.dtype))
