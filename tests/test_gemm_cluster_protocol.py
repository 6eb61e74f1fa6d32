"""Model check on the CPU of the GEMM's two-CTA cluster ring (gigaam_b200/csrc/gemm_sm90.cuh), restated as Python
coroutines under the random scheduler of test_attention_protocol_model.py, whose single-CTA GemmRing it extends.

Per CTA c of the cluster: full[s] expects one local arrival (the producer's arrive_expect_tx of 48 KB) and the bytes of
three loads -- its own A, its own W half and the peer's W half, both W halves multicast into the same stage of every CTA.
A load may land, and complete its bytes, before the local expect_tx.  empty[s] counts one arrival per consumer warpgroup
of every CTA, because either producer's multicast writes the stage in both.  Both CTAs walk the same tile-pair list.
The kernel ends with a cluster barrier, so no CTA exits while the peer can still write into it or arrive on its barriers.

Checked: no deadlock; no parity aliasing (every expect_tx, byte completion and arrival is tagged with the completion it
belongs to); no stage reloaded in any CTA while a wgmma group of that CTA still reads it (contents tagged per part); no
write or arrival into a CTA that has exited.  Two sanity cases show that the checker catches an empty[s] that counts
only the local warpgroups and a CTA that exits without the closing cluster barrier."""
import random

import pytest

from test_attention_protocol_model import Barrier, ProtocolError, _schedule

STAGE_BYTES = {"A": 16, "W": 16}       # KB per part of a stage


class TxBarrier:
    """mbarrier with one expected arrival per phase plus a transaction count that may go below zero (bytes that land
    before the expect_tx); every operation names the completion it belongs to."""

    def __init__(self, name):
        self.name, self.pending, self.tx, self.completions = name, 1, 0, 0

    def _check(self, j, what):
        if self.completions != j:
            raise ProtocolError(f"{self.name}: {what} for completion {j} while at completion {self.completions} (aliasing)")

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.completions += 1
            self.pending, self.tx = 1, 0

    def arrive_expect_tx(self, j, nbytes):
        self._check(j, "expect_tx")
        self.pending -= 1
        self.tx += nbytes
        self._maybe_complete()

    def complete_tx(self, j, nbytes):
        self._check(j, "complete_tx")
        self.tx -= nbytes
        self._maybe_complete()

    def ready(self, j):
        if self.completions > j + 1:
            raise ProtocolError(f"{self.name}: waiting for completion {j} but {self.completions} have happened (parity aliasing)")
        return self.completions == j + 1


class ClusterGemmRing:
    def __init__(self, n_pairs, nkb, stages, rng, C=2, empty_count=None, closing_barrier=True):
        self.n, self.nkb, self.S, self.C, self.rng, self.closing = n_pairs, nkb, stages, C, rng, closing_barrier
        cnt = 2 * C if empty_count is None else empty_count
        self.full = [[TxBarrier(f"cta{c}.full[{s}]") for s in range(stages)] for c in range(C)]
        self.empty = [[Barrier(f"cta{c}.empty[{s}]", cnt) for s in range(stages)] for c in range(C)]
        parts = ["A"] + [f"W{r}" for r in range(C)]
        self.stage = [[dict.fromkeys(parts) for _ in range(stages)] for _ in range(C)]
        self.reads = [[0] * stages for _ in range(C)]
        self.tma, self.wgmma = [], {(c, wg): [] for c in range(C) for wg in range(2)}
        self.finished = {(c, wg): [] for c in range(C) for wg in range(2)}
        self.at_end, self.exited = 0, [False] * C
        self.roles_left = [3] * C

    def _alive(self, c, what):
        if self.exited[c]:
            raise ProtocolError(f"{what} reaches CTA {c} after it exited")

    def _end(self, c):
        """the closing cluster barrier (or none): then the role is done; a CTA exits when all three of its roles are"""
        if self.closing:
            self.at_end += 1
            yield lambda: self.at_end == 3 * self.C
        self.roles_left[c] -= 1
        if self.roles_left[c] == 0:
            self.exited[c] = True

    def producer(self, c):
        stage, fills = 0, [0] * self.S
        for t in range(self.n):
            for kb in range(self.nkb):
                j = fills[stage]
                yield lambda s=stage, j=j: self.empty[c][s].ready(j - 1)              # mbar_wait(empty, phase ^ 1)
                self.full[c][stage].arrive_expect_tx(j, STAGE_BYTES["A"] + self.C * STAGE_BYTES["W"])
                # own A into this CTA, own W half multicast into every CTA
                for dst, part in [(c, "A")] + [(d, f"W{c}") for d in range(self.C)]:
                    if self.reads[dst][stage]:
                        raise ProtocolError(f"CTA {c} reloads stage {stage} of CTA {dst} under {self.reads[dst][stage]} "
                                            "pending wgmma group(s)")
                    self.stage[dst][stage][part] = "loading"

                    def landed(dst=dst, part=part, s=stage, j=j, tag=(t, kb)):
                        self._alive(dst, f"a TMA write of {part}")
                        self.stage[dst][s][part] = tag
                        self.full[dst][s].complete_tx(j, STAGE_BYTES[part[0]])
                    self.tma.append(landed)
                fills[stage] += 1
                stage = (stage + 1) % self.S
        yield from self._end(c)

    def release(self, c, wg, s):
        for d in range(self.C):
            self._alive(d, f"an empty arrival of cta{c}.wg{wg}")
            self.empty[d][s].arrive(f"cta{c}.wg{wg}")

    def consumer(self, c, wg):
        stage, uses, q = 0, [0] * self.S, self.wgmma[(c, wg)]
        for t in range(self.n):
            prev = None
            for kb in range(self.nkb):
                yield lambda s=stage, j=uses[stage]: self.full[c][s].ready(j)         # mbar_wait(full, phase)
                uses[stage] += 1
                if any(v != (t, kb) for v in self.stage[c][stage].values()):
                    raise ProtocolError(f"cta{c}.wg{wg} found {self.stage[c][stage]} in stage {stage}, wanted {(t, kb)}")
                self.reads[c][stage] += 1

                def group(s=stage, tag=(t, kb)):
                    if any(v != tag for v in self.stage[c][s].values()):
                        raise ProtocolError(f"wgmma of cta{c} read stage {s} as {self.stage[c][s]}, issued for {tag}")
                    self.reads[c][s] -= 1
                q.append(group)
                yield lambda: len(q) <= 1                                               # wgmma.wait_group 1
                if prev is not None:
                    self.release(c, wg, prev)
                prev = stage
                stage = (stage + 1) % self.S
            yield lambda: not q                                                         # wgmma.wait_group 0
            if prev is not None:
                self.release(c, wg, prev)
            self.finished[(c, wg)].append(t)
        yield from self._end(c)

    def run(self):
        roles = {f"cta{c}.producer": self.producer(c) for c in range(self.C)}
        roles.update({f"cta{c}.wg{wg}": self.consumer(c, wg) for c in range(self.C) for wg in range(2)})
        engines = {"tma": (self.tma, False)}
        engines.update({f"wgmma{c}.{wg}": (q, True) for (c, wg), q in self.wgmma.items()})
        _schedule(self.rng, roles, engines)
        if any(v != list(range(self.n)) for v in self.finished.values()):
            raise ProtocolError(f"tiles finished: {self.finished}")


@pytest.mark.parametrize("nkb", [1, 2, 3, 4, 5, 12])
@pytest.mark.parametrize("stages", [2, 4])
def test_cluster_ring_has_no_deadlock_aliasing_or_hazard(stages, nkb):
    """Pair counts 0 .. 7 per cluster (dead pairs are skipped by every role of both CTAs alike), k-blocks per tile below,
    at and above the ring depth (the kernel runs 4 stages)."""
    rng = random.Random(1000 * stages + nkb)
    for _ in range(100):
        ClusterGemmRing(rng.randint(0, 7), nkb, stages, rng).run()


def test_peer_bytes_may_land_before_the_local_expect_tx():
    """The schedules above do reach the case: some full[s] phase sees the peer's W half complete its bytes before the
    local producer's arrive_expect_tx."""
    seen = []
    orig = TxBarrier.complete_tx

    def spy(self, j, nbytes):
        if self.pending == 1 and self.completions == j:
            seen.append(self.name)
        orig(self, j, nbytes)
    TxBarrier.complete_tx = spy
    try:
        rng = random.Random(5)
        for _ in range(50):
            ClusterGemmRing(3, 6, 4, rng).run()
    finally:
        TxBarrier.complete_tx = orig
    assert seen


def test_the_model_catches_an_empty_barrier_counting_only_local_warpgroups():
    """Sanity of the checker: with empty[s] expecting only this CTA's two warpgroups, a producer's multicast can overwrite
    a stage the peer still reads (or arrivals of the peer complete a phase nobody waits for: aliasing)."""
    rng = random.Random(17)
    with pytest.raises(ProtocolError):
        for _ in range(300):
            ClusterGemmRing(3, 5, 2, rng, empty_count=2).run()


def test_the_model_catches_an_exit_without_the_closing_cluster_barrier():
    """... and a CTA that exits as soon as its own roles are done: the peer's last releases (or multicasts) then reach a
    CTA that no longer exists."""
    rng = random.Random(19)
    with pytest.raises(ProtocolError, match="after it exited"):
        for _ in range(300):
            ClusterGemmRing(2, 3, 2, rng, closing_barrier=False).run()
