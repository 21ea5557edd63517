"""CPU model of the persistent sweep loop of k_predict_main (csrc/predict.cu).  A CTA runs one sweep over its training
tiles for each of its query tiles; the model tiles stream through two stages, each with its own mbarrier, and a running
counter g over every tile the CTA consumes sets the stage (g & 1) and the phase parity ((g >> 1) & 1) of each wait.
Thread 0 (warp 0) issues tile g + 1 after the CTA-wide barrier of tile g in the one-barrier form (OB), tile g + 2
after the barrier that follows GEMM2 of tile g otherwise -- across sweep boundaries alike.  At the start of a sweep
the warps build the Q tile (one warp per row) or, on the graph path, thread 0 copies the prepared rows in through a
third mbarrier whose parity is the sweep's; a CTA-wide barrier follows.  The epilogue reads Q, and a barrier at the
end of each sweep orders those reads before the next sweep's Q is written.

The model runs 8 warps and the copy engine with random progress and checks that no buffer is overwritten while a warp
can still read it (Q by GEMM1 and the epilogue, stages by GEMM1 and GEMM2), that every wait sees the tile it expects,
and that the loop ends, also for CTAs without a query tile.  No GPU."""

import itertools
import random

import pytest

N_WARPS = 8


class Hazard(Exception):
    pass


class CTA:
    def __init__(self, n_qt, n_sweep, ob, q_copy, running=True, end_barrier=True):
        self.n_qt, self.n_sweep, self.ob, self.q_copy = n_qt, n_sweep, ob, q_copy
        self.running, self.end_barrier = running, end_barrier
        self.g_end = n_qt * n_sweep
        self.stage_tag = [None, None]  # model tile g each stage holds (None: empty or being written)
        self.stage_phases = [0, 0]  # completed phases of the two stage mbarriers
        self.q_tag = [None] * N_WARPS  # sweep whose rows of Q warp w's rows hold
        self.q_phases = 0
        self.copies = []  # in flight: ('stage', s, g) or ('q', qi)
        self.readers = {}  # buffer -> warps reading it
        self.issued = 0
        self.bar_arrived = 0
        self.bar_gen = 0

    def slot(self, g, tt):
        k = g if self.running else tt
        return k & 1, (k >> 1) & 1

    def check_free(self, buf, what):
        if self.readers.get(buf):
            raise Hazard('%s overwrites %s while warps %s read it' % (what, buf, sorted(self.readers[buf])))

    def read(self, w, buf, on):
        (self.readers.setdefault(buf, set()).add if on else self.readers[buf].discard)(w)

    def issue(self, g):
        if g >= self.g_end:
            raise Hazard('tile %d issued beyond the %d this CTA consumes' % (g, self.g_end))
        s = g & 1
        self.check_free(('stage', s), 'tile %d' % g)
        self.stage_tag[s] = None
        self.copies.append(('stage', s, g))
        self.issued += 1

    def issue_q(self, qi):
        self.check_free('Q', 'the Q copy of sweep %d' % qi)
        self.q_tag = [None] * N_WARPS
        self.copies.append(('q', qi))

    def complete(self, rng):
        c = self.copies.pop(rng.randrange(len(self.copies)))
        if c[0] == 'stage':
            self.stage_tag[c[1]] = c[2]
            self.stage_phases[c[1]] += 1
        else:
            self.q_tag = [c[1]] * N_WARPS
            self.q_phases += 1

    def barrier(self):
        gen = self.bar_gen
        self.bar_arrived += 1
        if self.bar_arrived == N_WARPS:
            self.bar_arrived = 0
            self.bar_gen += 1
        yield lambda: self.bar_gen > gen

    def check_q(self, w, qi, where):
        if any(t != qi for t in self.q_tag):
            raise Hazard('warp %d: %s of sweep %d reads Q rows of sweeps %s' % (w, where, qi, self.q_tag))

    def warp(self, w):
        work = lambda: True  # noqa: E731  (a step of work; the scheduler's random choice of warp sets its length)
        yield from self.barrier()  # mbarrier init
        if w == 0 and self.g_end > 0:
            self.issue(0)
            if not self.ob and self.g_end > 1:
                self.issue(1)
        g = 0
        for qi in range(self.n_qt):
            if self.q_copy:
                if w == 0:
                    self.issue_q(qi)
            else:
                self.check_free('Q', 'warp %d building sweep %d' % (w, qi))
                self.q_tag[w] = None
                yield work
                self.q_tag[w] = qi
            yield from self.barrier()
            if self.q_copy:
                yield lambda qi=qi: (self.q_phases & 1) != (qi & 1)
            for tt in range(self.n_sweep):
                s, par = self.slot(g, tt)
                yield lambda s=s, par=par: (self.stage_phases[s] & 1) != par
                if self.stage_tag[s] != g:
                    raise Hazard('warp %d waits for tile %d in stage %d and finds %s' % (w, g, s, self.stage_tag[s]))
                self.check_q(w, qi, 'GEMM1')
                self.read(w, 'Q', True)
                self.read(w, ('stage', s), True)
                yield work
                self.check_q(w, qi, 'GEMM1')
                self.read(w, 'Q', False)
                if self.ob:
                    yield from self.barrier()
                    if w == 0 and g + 1 < self.g_end:
                        self.issue(g + 1)
                yield work  # GEMM2
                if self.stage_tag[s] != g:
                    raise Hazard('warp %d: stage %d changed under GEMM2 of tile %d' % (w, s, g))
                self.read(w, ('stage', s), False)
                if not self.ob:
                    yield from self.barrier()
                    if w == 0 and g + 2 < self.g_end:
                        self.issue(g + 2)
                g += 1
            yield from self.barrier()  # row sums / parked partial sums
            self.check_q(w, qi, 'epilogue')
            self.read(w, 'Q', True)
            yield work
            self.check_q(w, qi, 'epilogue')
            self.read(w, 'Q', False)
            if self.end_barrier:
                yield from self.barrier()


def run(n_qt, n_sweep, ob, q_copy, seed, max_steps=200000, **kw):
    """True when every warp finished and no copy is left in flight; False on a deadlock."""
    rng = random.Random(seed)
    cta = CTA(n_qt, n_sweep, ob, q_copy, **kw)
    warps = {}
    for w in range(N_WARPS):
        gen = cta.warp(w)
        warps[w] = (gen, next(gen))
    for _ in range(max_steps):
        if not warps and not cta.copies:
            assert cta.issued == cta.g_end
            return True
        ready = [w for w, (_, cond) in warps.items() if cond()]
        if not ready and not cta.copies:
            return False
        if cta.copies and (not ready or rng.random() < 0.2):
            cta.complete(rng)
            continue
        w = rng.choice(ready)
        gen = warps[w][0]
        try:
            warps[w] = (gen, next(gen))
        except StopIteration:
            del warps[w]
    return False


SHAPES = [(n_qt, n_sweep) for n_qt, n_sweep in itertools.product((1, 2, 5), (1, 2, 3, 7))]


@pytest.mark.parametrize('ob', [True, False], ids=['one_barrier', 'two_barrier'])
@pytest.mark.parametrize('q_copy', [False, True], ids=['built', 'copied'])
@pytest.mark.parametrize('n_qt,n_sweep', SHAPES)
def test_persistent_loop_has_no_hazard_and_no_deadlock(n_qt, n_sweep, ob, q_copy):
    for seed in range(4):
        assert run(n_qt, n_sweep, ob, q_copy, seed), 'deadlock'


@pytest.mark.parametrize('ob', [True, False], ids=['one_barrier', 'two_barrier'])
def test_cta_without_query_tiles_ends(ob):
    assert all(run(0, 5, ob, q_copy, s) for q_copy in (False, True) for s in range(3))


def test_model_detects_sweep_local_phases():
    """Stages and parities counted from the start of each sweep (t - t_begin) break at the first sweep boundary
    after an odd sweep: the prefetched tile sits in the other stage, or the wait aliases an older phase."""
    for ob in (True, False):
        found = 0
        for seed in range(10):
            try:
                found += not run(3, 3, ob, False, seed, running=False)
            except Hazard:
                found += 1
        assert found == 10


def test_model_detects_a_missing_end_of_sweep_barrier():
    """Without the barrier at the end of a sweep, a warp starts the next Q tile while another still reads Q in the
    epilogue."""
    found = 0
    for seed in range(30):
        try:
            run(3, 2, True, False, seed, end_barrier=False)
        except Hazard:
            found += 1
    assert found > 0
