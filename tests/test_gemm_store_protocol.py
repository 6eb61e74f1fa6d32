"""Model check on the CPU of the GEMM's shared-memory store path (gigaam_b200/csrc/gemm_sm90.cuh, store_tile_tma), restated as
Python coroutines under the random scheduler of test_attention_protocol_model.py.

One consumer warpgroup: four warps, warp 0 holding the leader thread.  It owns two store slots and walks a list of tiles;
a tile is either stored through the slots in an even number of chunks (8 fp32, 4 fp16, 2 GLU), chunk c in slot c & 1, or
straight from the fragment (the tile that straddles the live row count), which leaves the slots alone.  Per chunk: the
leader waits until every bulk store but the most recent one has read its slot (cp.async.bulk.wait_group.read 1), the
warpgroup meets on its named barrier, each warp writes its 16 rows of the slot, fences them to the async proxy, the
warpgroup meets again and the leader issues the bulk store and commits it.  A bulk store reads its slot, then writes global
memory, each at a time of the scheduler's choosing; stores may finish out of order.  Before the kernel's closing barrier
the leader waits for all its stores (wait_group 0).

Checked: no slot is written while a bulk store may still read it; every bulk store reads the chunk it was issued for, from
all four warps; nothing is outstanding when the warpgroup exits.  Sanity cases show that the checker catches a reuse
without the wait_group.read, a store issued before the second barrier, and an exit without the wait_group 0."""
import random

import pytest

from test_attention_protocol_model import Barrier, ProtocolError, _schedule

WARPS = 4


class StoreSlots:
    def __init__(self, tiles, rng, wait_read=True, second_barrier=True, wait_all=True):
        self.tiles, self.rng = tiles, rng
        self.wait_read, self.second_barrier, self.wait_all = wait_read, second_barrier, wait_all
        self.bar = Barrier("named barrier", WARPS)
        self.slot = [[None] * WARPS for _ in range(2)]   # chunk tag each warp last wrote into each slot
        self.groups = []                                  # committed bulk stores, oldest first
        self.bulk = []                                    # pending engine steps of the bulk stores
        self.stored = []                                  # chunk tags whose global write has happened
        self.exited = 0

    def _reading(self, s):
        return [g for g in self.groups if g["slot"] == s and not g["read"]]

    def _issue(self, tag, s):
        g = {"tag": tag, "slot": s, "read": False, "done": False}
        self.groups.append(g)

        def read(g=g):
            if any(t != g["tag"] for t in self.slot[g["slot"]]):
                raise ProtocolError(f"bulk store of chunk {g['tag']} read slot {g['slot']} as {self.slot[g['slot']]}")
            g["read"] = True

            def write(g=g):
                g["done"] = True
                self.stored.append(g["tag"])
            self.bulk.append(write)
        self.bulk.append(read)

    def warp(self, w):
        meets = 0

        def meet():
            nonlocal meets
            self.bar.arrive(f"warp{w}")
            j, meets = meets, meets + 1
            return lambda: self.bar.ready(j)

        for t, chunks in enumerate(self.tiles):
            for c in range(chunks):                       # chunks == 0: the tile is stored directly
                s = c & 1
                if w == 0 and self.wait_read:
                    yield lambda: all(g["read"] for g in self.groups[:-1])          # wait_group.read 1
                yield meet()
                if self._reading(s):
                    raise ProtocolError(f"warp {w} rewrites slot {s} (tile {t} chunk {c}) while a bulk store may still read it")
                self.slot[s][w] = (t, c)                  # the warp's 16 rows, then fence.proxy.async
                if self.second_barrier:
                    yield meet()
                if w == 0:
                    self._issue((t, c), s)                # tma_store_2d + commit_group
        if w == 0 and self.wait_all:
            yield lambda: all(g["done"] for g in self.groups)                    # wait_group 0
        yield meet()                                      # the closing cluster barrier: the CTA exits after it
        self.exited += 1
        if self.exited == WARPS and not all(g["done"] for g in self.groups):
            raise ProtocolError("the warpgroup exits with bulk stores outstanding")

    def run(self):
        roles = {f"warp{w}": self.warp(w) for w in range(WARPS)}
        _schedule(self.rng, roles, {"bulk": (self.bulk, False)})
        want = sorted((t, c) for t, n in enumerate(self.tiles) for c in range(n))
        if sorted(self.stored) != want:
            raise ProtocolError(f"chunks stored: {sorted(self.stored)}, wanted {want}")


def _tiles(rng, chunks):
    """0 .. 6 tiles, each stored through the slots (`chunks` chunks) or, now and then, directly"""
    return [0 if rng.random() < 0.2 else chunks for _ in range(rng.randint(0, 6))]


@pytest.mark.parametrize("chunks", [2, 4, 8])
def test_slots_are_never_rewritten_under_a_bulk_store(chunks):
    """The kernel's chunk counts per tile (GLU, fp16, fp32), tile lists that mix slot-stored and directly stored tiles."""
    rng = random.Random(chunks)
    for _ in range(300):
        StoreSlots(_tiles(rng, chunks), rng).run()


def test_the_model_catches_a_reuse_without_wait_read():
    """Sanity of the checker: without the leader's wait_group.read 1, a slot is rewritten while the bulk store issued from
    it two chunks earlier has not read it yet."""
    rng = random.Random(23)
    with pytest.raises(ProtocolError, match="while a bulk store may still read it"):
        for _ in range(300):
            StoreSlots(_tiles(rng, 4), rng, wait_read=False).run()


def test_the_model_catches_a_store_issued_before_the_slot_is_complete():
    """... a bulk store issued right after the leader's own warp has written, without the second barrier: it reads rows the
    other warps have not written yet, or a late warp writes them under it."""
    rng = random.Random(29)
    with pytest.raises(ProtocolError, match="read slot|may still read it"):
        for _ in range(300):
            StoreSlots(_tiles(rng, 4), rng, second_barrier=False).run()


def test_the_model_catches_an_exit_with_stores_outstanding():
    """... and a warpgroup that leaves without wait_group 0."""
    rng = random.Random(31)
    with pytest.raises(ProtocolError, match="outstanding"):
        for _ in range(300):
            StoreSlots(_tiles(rng, 2), rng, wait_all=False).run()
