"""CPU: the oracle restatement and the product's device functions against the compiled, unmodified
reference (oracle/_ref) on seeded synthetic captures and on randomised slicer inputs."""
import numpy as np
import pytest

import helpers
from oracle import orc, refh
from rtl_433_b200 import lib, synth

pytestmark = pytest.mark.skipif(not refh.available(), reason="oracle/_ref/libr433ref.so not built")


@pytest.fixture(scope="module")
def ref():
    r = refh.Ref(store_bitbuffers=False, store_stages=True)
    r.register_defaults()
    yield r
    r.close()


def test_device_table_matches_reference(ref):
    table = lib.default_device_table()
    live = ref.registered()
    assert len(table) == len(live) == 335
    for a, b in zip(table, live):
        for k in ("protocol_num", "modulation", "short_width", "long_width", "reset_limit", "gap_limit", "sync_width",
                  "tolerance", "priority"):
            assert a[k] == b[k], (a["name"], k)


@pytest.mark.parametrize("seed", [0, 1])
def test_ook_stream_all_devices(ref, seed):
    devs = ref.registered()
    x = synth.ook_stream(seed, n_samples=1 << 19, n_bursts=4)
    want = ref.run(x, 2)
    assert len(want["packages"]) >= 4 and len(want["events"]) > 1000
    o = orc.Oracle(store_bitbuffers=False, store_stages=True)
    o.add_devices(devs)
    assert not helpers.compare_results(want, o.run(x, 2), "oracle")
    hc = helpers.HostCore(store_bitbuffers=False, store_stages=True)
    hc.add_devices(devs)
    assert not helpers.compare_results(want, hc.run(x, 2), "device functions", floats=False)


@pytest.mark.parametrize("seed", range(4))
def test_full_scale_samples_at_block_starts(ref, seed):
    """The hostile-IQ fuzz's (255, 255) family (tests/hostile_iq.py): the reference's int16 x[-1] across block calls
    drives AM below zero behind a spike on the last sample of a block.  The oracle must follow it exactly."""
    import hostile_iq
    devs = ref.registered()
    x = hostile_iq.spikes(seed)[0].iq
    o = orc.Oracle(store_bitbuffers=False, store_stages=True)
    o.add_devices(devs)
    for bb, block in ((0, hostile_iq.DEFAULT_BLOCK), (32768, hostile_iq.SMALL_BLOCK)):
        want = ref.run(x, 2, block_bytes=bb)
        assert hostile_iq.block_start_dips(want["am"], block).min() < 0
        d = helpers.compare_results(want, o.run(x, 2, block_bytes=bb), f"oracle, block_bytes {bb}")
        assert not d, "\n".join(d[:12])


@pytest.mark.parametrize("fpdm,freq", [(2, 868000000), (0, 433920000)])
def test_fsk_stream_all_devices(ref, fpdm, freq):
    devs = ref.registered()
    x = synth.fsk_stream(1, n_samples=1 << 18, n_bursts=2)
    want = ref.run(x, 4, 1024000, freq, fpdm)
    assert any(p["type"] == 2 for p in want["packages"])
    o = orc.Oracle(store_bitbuffers=False, store_stages=True)
    o.add_devices(devs)
    assert not helpers.compare_results(want, o.run(x, 4, 1024000, freq, fpdm), "oracle")
    hc = helpers.HostCore(store_bitbuffers=False, store_stages=True)
    hc.add_devices(devs)
    assert not helpers.compare_results(want, hc.run(x, 4, 1024000, freq, fpdm), "device functions", floats=False)


def test_small_blocks_and_silence(ref):
    """32 KiB blocks (block-call semantics: eop flag, start_ago/end_ago, x[-1] int16 wrap) and a
    file that is constant 128/128 except for its bursts."""
    devs = ref.registered()
    for x in (synth.ook_stream(9, n_samples=1 << 18, n_bursts=3), synth.nice_flor_s_file()[: 46752 // 16 * 16]):
        for bb in (32768, 0):
            want = ref.run(x, 2, block_bytes=bb)
            o = orc.Oracle(store_bitbuffers=False, store_stages=True)
            o.add_devices(devs)
            assert not helpers.compare_results(want, o.run(x, 2, block_bytes=bb), "oracle")
            hc = helpers.HostCore(store_bitbuffers=False, store_stages=True)
            hc.add_devices(devs)
            assert not helpers.compare_results(want, hc.run(x, 2, block_bytes=bb), "device functions", floats=False)


def test_saturated_input_wraps_like_reference(ref):
    """I = Q = 255 gives an envelope of 32768, which the reference stores as int16 between
    blocks (src/baseband.c:167); a block boundary inside a saturated stretch exercises it."""
    devs = ref.registered()
    x = synth.ook_stream(4, n_samples=1 << 16, n_bursts=0)
    x[2 * 16300:2 * 16500] = 255
    want = ref.run(x, 2, block_bytes=32768)
    hc = helpers.HostCore(store_bitbuffers=False, store_stages=True)
    hc.add_devices(devs)
    assert not helpers.compare_results(want, hc.run(x, 2, block_bytes=32768), "device functions", floats=False)
    o = orc.Oracle(store_bitbuffers=False, store_stages=True)
    o.add_devices(devs)
    assert not helpers.compare_results(want, o.run(x, 2, block_bytes=32768), "oracle")


def random_train(rng, kind):
    """Pulse trains that stress the slicers: nominal symbol mixes, long runs (row spill past
    1024 bits), many short rows (50-row overflow), zero widths, huge pulses."""
    n = int(rng.integers(1, 400))
    unit = int(rng.choice([12, 25, 50, 62, 100, 125, 250]))
    if kind == 0:
        pulse = rng.choice([unit, 2 * unit, 3 * unit], n) + rng.integers(-3, 4, n)
        gap = rng.choice([unit, 2 * unit, 4 * unit, 8 * unit], n) + rng.integers(-3, 4, n)
    elif kind == 1:  # long NRZ-like runs -> thousands of bits per row
        pulse = rng.integers(1, 40, n) * unit
        gap = rng.integers(1, 40, n) * unit
    elif kind == 2:  # many row breaks
        pulse = rng.choice([unit, 2 * unit], n)
        gap = rng.choice([unit, 20 * unit, 45 * unit], n, p=[0.5, 0.3, 0.2])
    else:
        pulse = rng.integers(0, 3000, n)
        gap = rng.integers(0, 30000, n)
        pulse[rng.integers(0, n)] = 400000
    gap[-1] = int(rng.integers(2500, 30000))
    return np.maximum(pulse, 0).astype(np.int32), np.maximum(gap, 0).astype(np.int32)


def test_slicers_on_random_pulse_trains(ref):
    """Every default device's slicer (all ten modulations + the FSK three) on random trains:
    device index order, event count and every bitbuffer byte must match the reference."""
    devs = ref.registered()
    hc = helpers.HostCore(store_bitbuffers=True)
    hc.add_devices(devs)
    ref.L.refh_set_capture(ref.h, 0, 1, 0)
    rng = np.random.default_rng(1234)
    try:
        total = 0
        for it in range(60):
            pulse, gap = random_train(rng, it % 4)
            for fsk, rate in ((0, 250000), (1, 1024000), (0, 1000000)):
                want = ref.slice_all(fsk, rate, pulse, gap)
                got = hc.slice(2 if fsk else 1, rate, pulse, gap)
                assert len(want) == len(got), (it, fsk, len(want), len(got))
                for (wd, wb), (gd, gb) in zip(want, got):
                    assert wd == gd
                    assert wb.tobytes() == gb.tobytes(), (it, fsk, devs[wd]["name"], devs[wd]["modulation"])
                total += len(want)
        assert total > 50000
    finally:
        ref.L.refh_set_capture(ref.h, 0, 0, 1)


def test_per_stage_functions(ref):
    rng = np.random.default_rng(7)
    L, O = refh.lib(), orc.lib()
    iq8 = rng.integers(0, 256, 2 * 5000, dtype=np.uint8)
    iq16 = rng.integers(-32767, 32768, 2 * 5000).astype(np.int16)
    for rf, of, src in (("refh_envelope_detect", "orc_envelope_cu8", iq8), ("refh_magnitude_est_cu8", "orc_magnitude_cu8", iq8),
                        ("refh_magnitude_est_cs16", "orc_magnitude_cs16", iq16)):
        a = np.zeros(5000, np.uint16)
        b = np.zeros(5000, np.uint16)
        getattr(L, rf)(src.ctypes.data, a.ctypes.data, 5000)
        getattr(O, of)(src.ctypes.data, b.ctypes.data, 5000)
        assert np.array_equal(a, b)
    for cs16, src, lp in ((0, iq8, 0.1), (0, iq8, 0.2), (1, iq16, 0.2), (1, iq16, 0.1), (0, iq8, 25000.0), (1, iq16, 12.0)):
        a = np.zeros(5000, np.int16)
        b = np.zeros(5000, np.int16)
        ca = np.zeros(2, np.int32)
        cb = np.zeros(2, np.int32)
        L.refh_demod_fm(cs16, src.ctypes.data, a.ctypes.data, 5000, 1024000 if cs16 else 250000, lp, ca.ctypes.data)
        O.orc_demod_fm(cs16, src.ctypes.data, b.ctypes.data, 5000, 1024000 if cs16 else 250000, lp, cb.ctypes.data)
        assert np.array_equal(ca, cb) and np.array_equal(a, b)


def _level_grid():
    import test_level_fuzz
    return test_level_fuzz.GRID


@pytest.mark.parametrize("levels", _level_grid(), ids=lambda g: ",".join(f"{k}={v:g}" for k, v in g.items()))
def test_level_grid_on_hostile_iq(ref, levels):
    """The level fuzz's grid (tests/test_level_fuzz.py: level_limit, min_level, min_snr one at a time, in envelope and
    magnitude mode, and three combined points) on every hostile-IQ family: the GPU suite judges the kernels by the
    oracle alone there, so the oracle must equal the reference at every point -- packages, widths, events, stages."""
    import hostile_iq
    import test_front_fuzz
    devs = ref.registered()
    o = orc.Oracle(store_bitbuffers=False, store_stages=True)
    o.add_devices(devs)
    ref.set_levels(**levels)
    o.set_levels(**levels)
    try:
        for name in hostile_iq.FAMILIES:
            for c in test_front_fuzz.family_cases(name, 0):
                want = ref.run(c.iq, c.fmt, c.rate, c.freq, c.fpdm)
                d = helpers.compare_results(want, o.run(c.iq, c.fmt, c.rate, c.freq, c.fpdm), f"oracle, {c}, {levels}")
                assert not d, "\n".join(d[:12])
    finally:
        ref.set_levels()
        o.close()
