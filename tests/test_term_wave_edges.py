"""The generators of term_wave16.py on the CPU, against the batch oracles: the bumps of the three term passes must reset
cells onto every edge of the 16-bit offset window that bump_edges16 claims, empty full Inflights windows and read
queues, and the frames of wave_world must cross the window both ways and free full windows in waves 2 and later --
for the GPU tests that run on them (test_gpu_term_wave_edges.py) to mean anything."""
import numpy as np
import pytest

from helpers import B, O
from oracle import control_oracle as CO
from oracle import wire_waves_oracle as WW
import hb_frames as F
import term_wave16 as W


@pytest.mark.parametrize("name", sorted(W.ROLES))
def test_bumps_reach_every_16bit_edge(name):
    rng = np.random.default_rng(0x16B0 + sorted(W.ROLES).index(name))
    s, c, vt, q, _, _ = W.bump_world(rng, name, 6000, 200)
    assert (q.count[: s.n] > 0).sum() > (500 if name == "leader_term" else 100)
    before, q0 = O.copy_columns(c), q.copy()
    blob, off = F.batch(W.bump_frames(rng, s, name))
    st = W.BATCH[name](c, q, vt, blob, off, s.table)[0]
    assert np.count_nonzero(st & B.FTERM_BUMPED) > 1000            # (VREQ_BUMPED is the same bit)
    W.check_bump_counts(W.bump_counts(before, c, W.persisted_of(s), s.n, q0, q), name)


@pytest.mark.parametrize("runs", [False, True], ids=["no_runs", "runs"])
def test_wave_world_crosses_the_16bit_window_in_later_waves(runs):
    rng = np.random.default_rng(0x16B8 + runs)
    c, rows, fill, blob, off, script = W.wave_world(rng, 4000)
    O.enable_inflights(c, W.INS_CAP)
    assert np.all(CO.arena_control(c, np.zeros((O.SLOTS, c.cap), np.uint8), fill)["status"] == 0)
    rep = (c.pflags[1:5, : c.n_groups] & O.PF_STATE_MASK) == O.STATE_REPLICATE
    full = (c.pflags[1:5, : c.n_groups] & O.PF_INS_FULL) != 0
    assert np.count_nonzero(full) > 0.6 * np.count_nonzero(rep)
    for waves in (2, 4, B.WIRE_WAVES_MAX):
        counts = W.wave_counts(c, rows if runs else None, blob, off, waves, WW.leader)
        for what, k in counts.items():
            assert k >= W.FLOOR, (waves, what, counts)
