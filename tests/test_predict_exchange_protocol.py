"""CPU model of the k-split warp pairs of k_predict_main (PCfg XK, csrc/predict.cu: Cfg160o and Cfg224o).  The two
warps of a pair each run GEMM1 over half of k, write the row half of their partial S1 / S2 fragments that the partner
finishes into their own slot of the pair's exchange area, meet at a 64-thread named barrier, read the partner's slot,
run the Matern transform and then reach the one CTA-wide barrier of the tile.  The exchange area is single-buffered:
the CTA-wide barrier separates the reads of tile t from the writes of tile t + 1.  The model runs 8 warps with random
progress and checks that a slot is never rewritten while the partner still reads it, that every read sees the
partner's data of the same tile, and that the loop cannot deadlock.  No GPU."""

import random

import pytest


class Hazard(Exception):
    pass


def run(n_tiles, seed, cta_barrier=True, max_steps=400000):
    rng = random.Random(seed)
    n_warps = 8
    partner = [w ^ 1 for w in range(n_warps)]  # warp = 2 * pair + w1k
    # phases: 0 GEMM1, 1 write own slot, 2 named barrier, 3 read partner slot, 4 transform, 5 CTA barrier, 6 GEMM2
    tile = [0] * n_warps
    phase = [0] * n_warps
    slot_tile = [None] * n_warps  # tile whose partials warp w's slot holds
    reading = [False] * n_warps  # warp w is reading its partner's slot
    named = {}  # (pair, tile) -> arrivals at the named barrier
    cta = [0] * n_tiles  # arrivals at the CTA-wide barrier

    for _ in range(max_steps):
        if all(t >= n_tiles for t in tile):
            return True
        w = rng.randrange(n_warps)
        t = tile[w]
        if t >= n_tiles:
            continue
        q = partner[w]
        if phase[w] == 0:
            if rng.random() < 0.3:  # GEMM1 done
                phase[w] = 1
        elif phase[w] == 1:
            if reading[q]:
                raise Hazard('warp %d rewrites its slot for tile %d while warp %d still reads it' % (w, t, q))
            slot_tile[w] = t
            key = (w >> 1, t)
            named[key] = named.get(key, 0) + 1
            phase[w] = 2
        elif phase[w] == 2:
            if named[(w >> 1, t)] == 2:  # both warps of the pair arrived
                if slot_tile[q] != t:
                    raise Hazard('warp %d reads tile %s from warp %d in tile %d' % (w, slot_tile[q], q, t))
                reading[w] = True
                phase[w] = 3
        elif phase[w] == 3:
            if slot_tile[q] != t:
                raise Hazard('slot of warp %d overwritten with tile %s while warp %d reads tile %d' % (q, slot_tile[q], w, t))
            if rng.random() < 0.5:  # read done
                reading[w] = False
                phase[w] = 4
        elif phase[w] == 4:
            if rng.random() < 0.5:  # transform done
                cta[t] += 1
                phase[w] = 5
        elif phase[w] == 5:
            if not cta_barrier or cta[t] == n_warps:
                phase[w] = 6
        elif phase[w] == 6:
            if rng.random() < 0.3:  # GEMM2 done
                tile[w] = t + 1
                phase[w] = 0
    return False


@pytest.mark.parametrize('seed', range(30))
def test_exchange_has_no_reuse_hazard_and_no_deadlock(seed):
    assert run(n_tiles=9, seed=seed)


def test_exchange_single_tile():
    """A CTA whose split of the training points is one tile (small batches) runs the exchange once."""
    assert all(run(n_tiles=1, seed=s) for s in range(10))


def test_model_detects_a_missing_cta_barrier():
    """Without the CTA-wide barrier a warp can run ahead into the next tile's exchange while its partner still reads
    the current one: the single-buffered area is only safe because of that barrier, and the model sees it."""
    found = 0
    for seed in range(50):
        try:
            run(n_tiles=9, seed=seed, cta_barrier=False)
        except Hazard:
            found += 1
    assert found > 0
