"""scripts/tick_bytes.py counts the bytes a tick of the headline workload moves (no GPU needed)."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import tick_bytes as tb  # noqa: E402


def test_steady_state_tick_moves_active_planes_only():
    # 1M entities, SyncTest d=8: one image read, eight Saves, live image deferred
    assert tb.tick_bytes(1_000_000, 8, True, False) == 9 * 33 * 1_000_000 == 297_000_000


def test_a_version_bump_adds_the_passive_planes_and_an_eager_tick_the_live_image():
    assert tb.tick_bytes(1_000_000, 8, True, True) == 9 * 61 * 1_000_000
    assert tb.tick_bytes(1_000_000, 8, False, True) == 10 * 61 * 1_000_000
