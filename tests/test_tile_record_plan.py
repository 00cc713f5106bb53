"""The fused tile kernels' stage plan with 16-bit offset rows at their own stride and the packed kernel's record
buffers (k_tile.cuh: kFRow16, kRecCap, tile_stage_bytes, tile_stages), restated on the CPU; and the shape matrix of
test_gpu_tile_shapes.py reaching every stage count of that plan."""
import numpy as np
import pytest

from helpers import B, TILE_SHAPES, random_state, GROUPS, MAX_STAGES, ROW64, ROW8, SMEM, TILE, UNIT_CAP, plan

ROW16 = (TILE + 8) * 2
REC_CAP = 4 * TILE
REC_BYTES = GROUPS * 2 * REC_CAP * 16
KERNELS = {"packed": (0, REC_BYTES), "compact": (4 * UNIT_CAP, GROUPS * TILE * 4)}   # (payload bytes, extra bytes)
WANT_STAGES = {"packed": (8, 8, 7, 6, 5, 4, 4, 3), "compact": (8, 8, 8, 8, 7, 6, 6, 5)}

needs_256 = pytest.mark.skipif(B.tile_groups() != 256, reason="the stage table is for 256-group tiles")


def stage_bytes(h, payload):
    return h * ROW64 + 2 * h * ROW16 + 3 * ROW64 + TILE * 4 + h * ROW8 + payload


def stages(h, kernel):
    payload, extra = KERNELS[kernel]
    return min(MAX_STAGES, (SMEM - extra) // stage_bytes(h, payload))


@needs_256
def test_stage_plan_restated():
    assert ROW16 == 528 and ROW16 % 16 == 0 and (ROW16 // 4) % 32 == 4    # TMA alignment; rows 4 banks apart
    assert stage_bytes(5, 0) == 24176 and stage_bytes(5, 4 * UNIT_CAP) == 30320
    assert REC_BYTES == 96 * 1024
    for kernel, want in WANT_STAGES.items():
        assert tuple(stages(h, kernel) for h in range(1, 9)) == want, kernel
        assert min(want) >= GROUPS        # wait_stage needs a stage per consumer group
        payload, extra = KERNELS[kernel]
        assert all(stages(h, kernel) * stage_bytes(h, payload) + extra <= SMEM for h in range(1, 9))


@needs_256
def test_shape_matrix_covers_every_stage_count():
    reachable = {(k, s) for k, want in WANT_STAGES.items() for s in want}
    covered = set()
    for name, (shape, hint, force_general, seed) in TILE_SHAPES.items():
        meta = random_state(3000, shape, np.random.default_rng(seed)).meta
        for kernel in KERNELS:
            _, h, _ = plan(meta, force_general, kernel)
            covered.add((kernel, stages(bin(h).count("1"), kernel)))
    assert covered == reachable
