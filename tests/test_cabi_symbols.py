"""The C-ABI library loads on a CPU-only host and exports every symbol the header declares."""
import ctypes as C

from synergynet_b200 import _lib


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _lib.declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/synergy_b200.h but not exported'
    assert set(declared) == set(_lib.SIGNATURES), 'ctypes table and header out of sync'
    assert lib.syn_abi_version() == 1


def test_null_handle_calls_fail_cleanly():
    lib = _lib.load()
    assert lib.syn_commit(None) == 1
    assert lib.syn_forward(None, None, 1, None, None, None) == 1
    assert lib.syn_launch_count(None) == -1
    assert b'null handle' in lib.syn_last_error()
    lib.syn_destroy(None)
    h = C.c_void_p()
    rc = lib.syn_create(0, C.byref(h))      # no GPU here -> CUDA error, not a crash
    if rc != 0:
        assert rc in (1, 2, 6) and h.value is None
    else:
        lib.syn_destroy(h)


def _plan(lib, batch, sms, fpt):
    split, groups = C.c_int(-1), C.c_int(-1)
    assert lib.syn_debug_tile_plan(batch, sms, fpt, C.byref(split), C.byref(groups)) == 0
    return split.value, groups.value


def test_fused_tile_plan_covers_every_face_once():
    """Host logic of the fused engine's tile plan (kernels_fused.cuh fused_tile_plan / group_faces): every
    face belongs to exactly one group, two-face groups come first, and the single-face groups of a split
    last wave fit into one wave."""
    lib = _lib.load()
    for sms in (1, 4, 132, 148):
        for batch in list(range(1, 40)) + [147, 148, 149, 295, 296, 297, 300, 333, 592, 593, 1023, 1024, 1025, 4096]:
            split, groups = _plan(lib, batch, sms, 2)
            full = batch // 2
            assert 0 <= split <= full and groups == split + (batch - 2 * split)
            covered = []
            for fg in range(groups):                       # the kernel's group_faces()
                f0, nf = (2 * fg, 2) if fg < split else (2 * split + (fg - split), 1)
                covered.extend(range(f0, f0 + nf))
            assert covered == list(range(batch))
            singles = groups - split
            assert split % sms == 0 or split == full        # two-face groups fill whole waves, or all of them are kept
            if split < full:
                assert singles <= sms                       # the split tail is one wave
            else:
                assert singles == (batch & 1)
            for fpt in (1, 4):
                s1, g1 = _plan(lib, batch, sms, fpt)
                assert s1 == 0 and g1 == (batch + fpt - 1) // fpt
    assert lib.syn_debug_tile_plan(0, 148, 2, None, None) == 1
    split, groups = C.c_int(), C.c_int()
    assert lib.syn_debug_tile_plan(8, 148, 3, C.byref(split), C.byref(groups)) == 1
