"""The scoring-kernel thresholds that tests/test_gpu_score_edges.py builds its cases from parse out of the sources: a renamed
or reshaped constant fails here, on the CPU suite, instead of silently moving the GPU cases off their edges."""
from tests.score_constants import score_constants


def test_score_constants_parse():
    c = score_constants()
    assert 0 < c.exc_max < c.exc_slots and c.exc_slots & (c.exc_slots - 1) == 0
    assert c.probe_unroll >= 1 and c.inline_eps >= 3 and c.lut_max >= 1 and c.narrow_counter_max >= 1
    # every geometry the ABI accepts: 1 <= max_endpoints <= 8192
    seen = set()
    for n in (1, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192):
        log_epl, J, mpad, G = c.geo(n)
        assert mpad >= n and mpad == J * (32 << log_epl) and J & (J - 1) == 0 and 1 <= G <= 32
        seen.add(G)
    assert seen == {8, 16, 32}
