"""Spawning registrations on the generated kernel, on the CPU: NVRTC compiles generic_program_jit.cuh for sm_90a with the
preludes of worlds that register spawn_particles next to other columns (the spawn spec carries Transform, Velocity and
Ttl as plane0 / plane1 / param), and both entry points (k_generic_jit, k_generic_jit_batch) compile without spills at
the two instances the engine builds by default."""
import pytest

from test_batch_sources import _compile_verbose
from test_jit_sources_compile import _prelude

# {system, plane0, plane1, need, param} / {first_plane, off, len, finite, slot, absent}
# Transform = planes 0..9, Velocity = 10..12, Ttl = 13..14 in every registration below.
SPAWN = ("BGR_SYS_PARTICLES_SPAWN", 0, 10, 0, 13)
UPDATE = ("BGR_SYS_PARTICLES_UPDATE", 0, 10, 0, 0)
DESPAWN = ("BGR_SYS_PARTICLES_DESPAWN", 13, 0, 0, 0)
REGISTRATIONS = {
    # the stress schema (15 words) with spawn_particles and the example's two checksums
    "stress_15_words_spawn": (15, [SPAWN, UPDATE, DESPAWN], [(10, 0, 12, 1, 0, 0), (0, 0, 12, 1, 1, 0)]),
    # checksum_component_with_hash::<Transform> over all 40 bytes, and an optional Score (plane 15, absent bit 2)
    "whole_transform_optional_score": (16, [SPAWN, UPDATE, DESPAWN, ("BGR_SYS_U32_ADD", 15, 0, 2, 1)],
                                       [(0, 0, 40, 0, 0, 0), (10, 0, 12, 1, 1, 0), (15, 0, 4, 0, 2, 2)]),
    # a 24-word row (the widest the generated kernel takes): a 36-byte Blob behind Ttl, checksummed
    "24_words_spawn": (24, [SPAWN, UPDATE, DESPAWN], [(10, 0, 12, 1, 0, 0), (15, 0, 36, 0, 1, 0)]),
}


def _entry_block(log, kernel):
    at = log.index(f"Compiling entry function '{kernel}'")
    end = log.find("Compiling entry function", at + 1)
    return log[at:end if end >= 0 else len(log)]


# (2, 128): quarter-tile items (small worlds, batches); (4, 512): whole tiles
@pytest.mark.parametrize("rows,item_rows", [(2, 128), (4, 512)])
@pytest.mark.parametrize("name", list(REGISTRATIONS))
def test_spawning_registration_compiles_without_spills(name, rows, item_rows):
    words, systems, hashes = REGISTRATIONS[name]
    cubin, log = _compile_verbose(_prelude(words, rows, systems, hashes, item_rows))
    assert cubin[:4] == b"\x7fELF"
    assert b"k_generic_jit\x00" in cubin and b"k_generic_jit_batch\x00" in cubin
    for kernel in ("k_generic_jit", "k_generic_jit_batch"):
        block = _entry_block(log, kernel)
        assert "0 bytes spill stores, 0 bytes spill loads" in block, block
