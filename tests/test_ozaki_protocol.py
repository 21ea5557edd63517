"""CPU model of the stage ring of k_ozaki_gemm<S> (csrc/ozaki.cu): one producer thread and eight consumer warps
hand k-block stages back and forth through the full[] / empty[] mbarriers, with random copy and product latencies.

What the model runs, as the kernel does:
  ring       NST = min(floor(OZ_RING_BYTES / (S * 10 KB)), OZ_MAX_RING) stages of S A slices (8 KB) and S B slices (2 KB)
  producer   for every k-block of every tile of the CTA's id walk (ids without a tile are skipped): from the second round
             on, wait on empty[st] with parity (round - 1) & 1; arrive on full[st] with expect_tx of the stage's bytes;
             issue 2 S bulk copies that complete at random times
  consumers  each of the 8 warps, per k-block: wait on full[st] with parity round & 1; issue and commit the stage's
             products (a group that completes at a random later time); wait_group 1; lane 0 arrives on the previous
             stage's empty barrier (arrival count 8).  After the last k-block of a tile: wait_group 0, then release it.
  counters   st and round of both sides carry across the tiles of the walk.

Asserted: nothing deadlocks; no stage is refilled while a warp's products on it may still be in flight; every parity
wait passes on the phase it means (phases are counted, so a wait that passes on a phase two before or after is caught);
every stage a warp reads holds all 2 S slices of the k-block it expects; NST >= 2 and the shared memory fits.  The
ring constants are read from csrc/ozaki.cu."""

import os
import random
import re

import pytest

from conftest import ROOT

SMEM_LIMIT = 232448  # 227 KB of dynamic shared memory per block on sm_90
WARPS = 8


def _kernel_constants():
    src = open(os.path.join(ROOT, 'sgdml_b200', 'csrc', 'ozaki.cu')).read()
    env = {}
    for decl in re.findall(r'^constexpr int ([^;]+);', src, flags=re.M):
        for part in decl.split(','):
            name, expr = (x.strip() for x in part.split('=', 1))
            env[name] = eval(expr, {}, dict(env))  # integer expressions of earlier constants
    return env


K = _kernel_constants()
UNIT = K['OZ_A_BYTES'] + K['OZ_B_BYTES']


def stages(S):
    return min(K['OZ_RING_BYTES'] // (S * UNIT), K['OZ_MAX_RING'])


def smem_bytes():
    return K['OZ_RING_BYTES'] + 2 * K['OZ_MAX_RING'] * 8 + 1024  # ring, full[] and empty[], 1024-byte alignment


class MBar(object):
    """mbarrier: `phases` completed phases; a phase completes when its pending arrivals and transaction bytes are both
    zero.  try_wait.parity(P) passes while the current phase's parity differs from P."""

    def __init__(self, count):
        self.count, self.pending, self.tx, self.phases = count, count, 0, 0

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phases += 1
            self.pending = self.count

    def arrive(self, expect_tx=0):
        self.tx += expect_tx
        self.pending -= 1
        assert self.pending >= 0
        self._maybe_complete()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        assert self.tx >= 0
        self._maybe_complete()

    def passes(self, parity):
        return (self.phases & 1) != parity


def simulate(S, KB, walk, seed):
    """One CTA: `walk` lists, id by id, whether the id has a tile.  Returns the number of k-blocks every warp consumed."""
    NST = stages(S)
    SB = S * UNIT
    rng = random.Random(seed)
    full = [MBar(1) for _ in range(NST)]
    empty = [MBar(WARPS) for _ in range(NST)]
    content = [dict() for _ in range(NST)]  # slice index -> (tile, kb) whose bytes have landed in the stage
    copies = []  # (time, stage, slice, tag)
    tiles = [i for i, has in enumerate(walk) if has]
    now = 0

    def producer():
        st = rnd = 0
        for t in tiles:
            for kb in range(KB):
                if rnd > 0:
                    while not empty[st].passes((rnd - 1) & 1):
                        yield False
                    # the phase meant: the consumers' release of this stage's previous k-block (phase rnd - 1)
                    assert empty[st].phases == rnd, 'empty[%d] passed on phase %d, meant %d' % (st, empty[st].phases - 1, rnd - 1)
                for w in warps:
                    assert not any(g[1] == st and g[0] > now for g in w['groups']), \
                        'stage %d refilled while products on it are in flight' % st
                content[st].clear()
                full[st].arrive(expect_tx=SB)
                for sl in range(2 * S):
                    copies.append((now + rng.randint(1, 40), st, sl, (t, kb)))
                st += 1
                if st == NST:
                    st, rnd = 0, rnd + 1
                yield True

    def consumer(w):
        st = rnd = 0
        for t in tiles:
            prev = -1
            for kb in range(KB):
                while not full[st].passes(rnd & 1):
                    yield False
                assert full[st].phases == rnd + 1, 'full[%d] passed on phase %d, meant %d' % (st, full[st].phases - 1, rnd)
                assert content[st] == {sl: (t, kb) for sl in range(2 * S)}, 'stage %d does not hold k-block %d of tile %d' % (st, kb, t)
                last = max([g[0] for g in w['groups']] + [now])
                w['groups'].append((last + rng.randint(1, 12), st))  # commit: in-order completion
                while len([g for g in w['groups'] if g[0] > now]) > 1:  # wgmma.wait_group 1
                    yield False
                if prev >= 0:
                    empty[prev].arrive()
                prev = st
                w['consumed'] += 1
                st += 1
                if st == NST:
                    st, rnd = 0, rnd + 1
                yield True
            while any(g[0] > now for g in w['groups']):  # wgmma.wait_group 0
                yield False
            if prev >= 0:
                empty[prev].arrive()
            for _ in range(rng.randint(0, 30)):  # the epilogue
                yield True

    warps = [dict(groups=[], consumed=0) for _ in range(WARPS)]
    live = [producer()] + [consumer(w) for w in warps]
    while live:
        for ev in sorted(c for c in copies if c[0] <= now):
            copies.remove(ev)
            _, st, sl, tag = ev
            content[st][sl] = tag
            full[st].complete_tx(K['OZ_A_BYTES'] if sl % 2 == 0 else K['OZ_B_BYTES'])  # A and B slice sl // 2
        progressed = False
        for a in list(live):
            try:
                progressed |= bool(next(a))
            except StopIteration:
                live.remove(a)
                progressed = True
        pending = copies or any(g[0] > now for w in warps for g in w['groups'])
        assert progressed or pending or not live, 'deadlock at time %d' % now
        now += 1
    assert not copies
    return [w['consumed'] for w in warps]


WALKS = {
    'dense': [True] * 5,
    'gaps': [True, False, True, False, False, True, True],
    'leading_and_trailing_gaps': [False, False, True, True, False],
    'single': [True],
}


@pytest.mark.parametrize('walk', sorted(WALKS))
@pytest.mark.parametrize('S', [2, 3, 4, 5, 6, 7])
def test_ring_protocol(S, walk):
    tiles = sum(WALKS[walk])
    for KB in (2, 3, 16):
        for seed in range(4):
            consumed = simulate(S, KB, WALKS[walk], seed)
            assert consumed == [tiles * KB] * WARPS


@pytest.mark.parametrize('S', [2, 3, 4, 5, 6, 7])
def test_ring_fits(S):
    """3 to 8 stages by S, at least two k-blocks in flight, within the shared memory of one block."""
    assert 2 <= stages(S) <= K['OZ_MAX_RING']
    assert stages(S) * S * UNIT <= K['OZ_RING_BYTES']
    assert smem_bytes() <= SMEM_LIMIT
    assert [stages(s) for s in range(2, 8)] == [8, 7, 5, 4, 3, 3]


def stage_layout(S):
    """Byte offsets inside a stage, as the producer fills it: the S A slices (8 KB each), then the S B slices (2 KB
    each), in slice order."""
    return ([(p, p * K['OZ_A_BYTES'], K['OZ_A_BYTES']) for p in range(S)]
            + [(S + q, S * K['OZ_A_BYTES'] + q * K['OZ_B_BYTES'], K['OZ_B_BYTES']) for q in range(S)])


def issue_order(S):
    """oz_issue_kstep / oz_issue_slice: for PA = 1..S, Q = 1.. while PA + Q <= S + 1, one product into the accumulator of
    level PA + Q, reading A slice PA and B slice Q of the stage."""
    return [(pa, q, pa + q - 2) for pa in range(1, S + 1) for q in range(1, S + 2 - pa)]


def test_order_tables():
    """For S = 2..7: every kept slice pair once, in its level's accumulator; the stage's slices tile it without overlap,
    each part 1024-byte aligned (the 64-byte swizzle atoms), and the stage bytes are what expect_tx announces."""
    import ozaki_model as om

    for S in range(2, 8):
        order = issue_order(S)
        assert sorted((pa, q) for pa, q, _ in order) == sorted(pq for L in range(2, S + 2) for pq in om.level_pairs(S, L))
        assert all(acc == pa + q - 2 < S for pa, q, acc in order)
        lay = stage_layout(S)
        assert all(off % 1024 == 0 for _, off, _ in lay)
        assert all(a[1] + a[2] == b[1] for a, b in zip(lay, lay[1:]))
        assert lay[0][1] == 0 and lay[-1][1] + lay[-1][2] == S * UNIT
