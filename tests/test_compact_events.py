"""-m gpu: the one-word forms of the event wire format (r433b_slice.cuh) on caller-built packages.

A row of <= 16 bits is stored in one word, and so is an event of one such row.  Hand-made devices and pulse trains put
rows of 0, 1, 15, 16, 17, 31, 32 and 33 bits, sync counts at and one past the limits of both forms, empty events
(NRZS), mixed short and long rows, the 50-row overflow path, a spilled row followed by short rows and PCM clears of an
event longer than the write-combining window into k_slice2, next to one package whose output is over 4 KiB, so that
its warp takes the second pass.  Every event must equal the oracle's (the default devices on the same packages: the
reference's, where it is built), gates on and off; r433b_stream_digest must hash the long form of the events, and
an event of one short row must take one word.  tests/test_emu_compact_events.py runs the same bodies under the
SIMT emulator."""
import ctypes as C

import numpy as np
import pytest

import helpers
from oracle import orc
from rtl_433_b200 import lib
from test_parity_holes import MOD
from test_slice_fuzz import _pd, expected_events

RATE = 1000000  # one sample per microsecond: the widths below are samples


def dev(mod, short, long_, reset, gap=0.0, sync=0.0, tol=0.0):
    return dict(modulation=MOD[mod], short_width=float(short), long_width=float(long_), reset_limit=float(reset),
                gap_limit=float(gap), sync_width=float(sync), tolerance=float(tol), priority=0)


# PWM with syncs: one 100, zero 200, sync 400; a gap over 1000 ends a row, over 5000 the event
PWM = dev("OOK_PWM", 100, 200, 5000, gap=1000, sync=400, tol=30)
# PCM NRZ of 50-sample bits whose every gap ends a row: a pulse of k bits is a row of k ones
PCM = dev("OOK_PCM", 50, 50, 5000, gap=20)
# PCM RZ: a pulse off the 50-sample short width clears the event
PCM_RZ = dev("OOK_PCM", 50, 100, 5000, gap=1000, tol=10)
NRZS = dev("OOK_NRZS", 100, 100, 2000)
DEVICES = [PWM, PCM, PCM_RZ, NRZS]
GATES = [(17, -2, -2), (17, -2, -2), (0, 0, 0), (0, 0, 0)]  # gated: events whose rows are all <= 16 bits


def pwm_event(rng, rows):
    """rows = [(syncs, bits)] -> pulse / gap widths of one PWM event."""
    pulse, gap = [], []
    for syncs, bits in rows:
        pulse += [400] * syncs
        gap += [100] * syncs
        pulse += [int(w) for w in rng.choice([100, 200], bits)]
        gap += [100] * bits
        if gap:
            gap[-1] = 2000
    if not gap:  # no rows: a sync alone
        pulse, gap = [400], [0]
    gap[-1] = 9000
    return pulse, gap


def pcm_event(row_bits):
    """A row of k ones per pulse (k = 0: a pulse too short for a bit, an empty row)."""
    return [max(10, 50 * k) for k in row_bits], [100] * (len(row_bits) - 1) + [9000]


def rz_cleared(rng, n_before, n_after):
    """A PCM RZ row of n_before bits (well over the 16-word window), a cleared event, then n_after bits."""
    g = [int(x) for x in rng.choice([50, 150], n_before)]
    return [50] * n_before + [200] + [50] * n_after, g + [150] + [150] * (n_after - 1) + [9000]


def packages(seed):
    """-> [pulse_data_t record]: the edge cases, then random short packages of the same devices."""
    rng = np.random.default_rng(seed)
    trains = []
    for bits in (0, 1, 15, 16, 17, 31, 32, 33):
        trains.append(pwm_event(rng, [(0 if bits else 1, bits)]))
        trains.append(pwm_event(rng, [(1, bits), (0, 3), (2, bits)]))
        trains.append(pcm_event([bits]))
    for syncs in (7, 8, 9, 1023, 1024):
        trains.append(pwm_event(rng, [(syncs, 16)]))
        trains.append(pwm_event(rng, [(syncs, 5), (1, 40)]))
    trains.append(pwm_event(rng, [(0, 0)] + [(1, 0)]))  # syncs only: one row of 0 bits
    trains.append(pcm_event([3, 40, 0, 16, 17, 1, 33, 2]))  # mixed short and long rows
    trains.append(pcm_event([2] * 49 + [70, 5]))  # 50 rows: the last one goes dirty, then gets 5 bits
    trains.append(pcm_event([1] * 60))  # 50-row path with a dirty row of 0 bits
    trains.append(pcm_event([1100, 3, 16, 1, 0, 9]))  # a spilled row, then short rows
    trains.append(pcm_event([2200, 7]))  # two rows of spill
    trains.append(rz_cleared(rng, 700, 5))
    trains.append(rz_cleared(rng, 300, 40))
    trains.append(([50 * 36000], [9000]))  # 4.5 KiB from one device: its warp slices again into the arena
    trains.append(([100, 150, 100, 100], [2500, 100, 2500, 2500]))  # NRZS: empty events
    for _ in range(150):
        kind = int(rng.integers(0, 3))
        if kind == 0:
            rows = [(int(rng.integers(0, 3)), int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 5)))]
            trains.append(pwm_event(rng, rows))
        elif kind == 1:
            trains.append(pcm_event([int(rng.integers(0, 40)) for _ in range(int(rng.integers(1, 12)))]))
        else:
            trains.append(rz_cleared(rng, int(rng.integers(1, 80)), int(rng.integers(1, 30))))
    return [_pd(RATE, p, g) for p, g in trains]


def run(ctx, pds):
    ps = lib.Pulses()
    for pd in pds:
        ps.add(pd, stream=0)
    ctx.process_pulses(ps)
    res = ctx.fetch()
    return ps, res


def oracle_events(devices, pds):
    """[[(dev, bitbuffer bytes)] per package] in r433b_dispatch's order: priority class, then registration order."""
    o = orc.Oracle(store_bitbuffers=True)
    o.add_devices(devices)
    order = sorted(range(len(devices)), key=lambda dv: devices[dv]["priority"])
    try:
        return [[(dv, bb.tobytes()) for dv in order if devices[dv]["modulation"] < 16
                 for bb in o.slice(dv, RATE, pd["pulse"][:int(pd["num_pulses"])], pd["gap"][:int(pd["num_pulses"])])]
                for pd in pds]
    finally:
        o.close()


def by_package(got, n):
    out = [[] for _ in range(n)]
    for e in got["events"]:
        out[e["package"]].append(e)
    return out


def gated_out(bb, t):
    nr = int(bb["num_rows"])
    return t > 0 and nr >= 1 and int(bb["bits_per_row"][:nr].max()) < t


def custom_devices_match_the_oracle():
    pds = packages(5)
    want = oracle_events(DEVICES, pds)
    ctx = lib.Context(0)
    try:
        ctx.set_devices(DEVICES)
        ps, res = run(ctx, pds)
        got = by_package(helpers.gpu_stream_results(ctx, 0, store_bitbuffers=True), len(pds))
        n_events = 0
        for i in range(len(pds)):
            mine = [(e["dev"], e["bitbuffer"].tobytes()) for e in got[i]]
            assert mine == want[i], f"package {i}: {len(mine)} vs {len(want[i])} events"
            n_events += len(mine)
        assert n_events == res["n_events"] > 600
        nb = res["pairs"]["bytes"]
        assert nb.max() > 4096 and ((nb > 0) & (nb <= 4096)).sum() > 100
        # gates on: the same events without the gated ones
        ctx.set_gates(GATES)
        ps2, res = run(ctx, pds)
        got = by_package(helpers.gpu_stream_results(ctx, 0, store_bitbuffers=True), len(pds))
        for i in range(len(pds)):
            keep = [(dv, bb) for dv, bb in want[i]
                    if not gated_out(np.frombuffer(bb, lib.BITBUFFER_DTYPE)[0], GATES[dv][0])]
            assert [(e["dev"], e["bitbuffer"].tobytes()) for e in got[i]] == keep, f"gated package {i}"
        assert res["n_gated"] > 100
        ps.close()
        ps2.close()
    finally:
        ctx.close()


def default_devices_match():
    """The 335 default devices on the same packages, against the reference where it is built."""
    devices = lib.default_device_table()
    pds = packages(6)
    want = expected_events([pds], devices)
    ctx = lib.Context(0)
    try:
        ctx.set_devices(devices)
        ps, res = run(ctx, pds)
        got = by_package(helpers.gpu_stream_results(ctx, 0, store_bitbuffers=want is None), len(pds))
        if want is None:
            want_bb = oracle_events(devices, pds)
            for i in range(len(pds)):
                assert [(e["dev"], e["bitbuffer"].tobytes()) for e in got[i]] == want_bb[i], f"package {i}"
        else:
            for i in range(len(pds)):
                assert [(e["dev"], e["hash"]) for e in got[i]] == want[0][i], f"package {i}"
        ps.close()
    finally:
        ctx.close()


def fnv1a(h, words):
    for w in words:
        h = ((h ^ int(w)) * 1099511628211) & 0xffffffffffffffff
    return h


def long_form(bb, header, trailer):
    """An event in the long form of the wire format, from its bitbuffer; `header` is its first stored word, `trailer`
    its last (the word count of a dirty last row)."""
    nr, free_row = int(bb["num_rows"]), int(bb["free_row"])
    dirty = (header & 0xff) != 0xff and (header >> 7) & 1
    flat = bb["bb"].reshape(-1)
    words = []
    for r in range(nr):
        bits, syncs = int(bb["bits_per_row"][r]), int(bb["syncs_before_row"][r])
        words.append(bits | (syncs << 16))
        n = trailer if dirty and r + 1 == nr else (bits + 31) // 32
        words += list(np.frombuffer(flat[r * 128:r * 128 + 4 * n].tobytes(), "<u4"))
    if dirty:
        words.append(trailer)
    return [nr | (dirty << 7) | (free_row << 8) | ((len(words) + 1) << 16)] + words


def stream_digest_hashes_the_long_form():
    ctx = lib.Context(0)
    try:
        ctx.set_devices(DEVICES)
        pds = packages(7)
        ps, res = run(ctx, pds)
        arena = res["events"]
        bb = np.zeros(1, lib.BITBUFFER_DTYPE)
        h = 1469598103934665603
        n_events = 0
        for k in res["packages"]:  # fetched in (stream, seq) order
            off, cnt = int(k["pulse_off"]), int(k["pulse_count"])
            h = fnv1a(h, [int(k["seq"]), int(k["type"]) & 0xffffffff, int(k["block"]) & 0xffffffff,
                          int(k["offset"]) & 0xffffffff, int(k["offset"]) >> 32, 0, 0, int(k["start_ago"]),
                          int(k["end_ago"]), int(k["num_pulses"]), cnt, int(k["ook_low_estimate"]) & 0xffffffff,
                          int(k["ook_high_estimate"]) & 0xffffffff, int(k["fsk_f1_est"]) & 0xffffffff,
                          int(k["fsk_f2_est"]) & 0xffffffff])
            h = fnv1a(h, res["pulse_pool"][off:off + cnt].view(np.uint32))
            h = fnv1a(h, res["gap_pool"][off:off + cnt].view(np.uint32))
            for pr in res["pairs"][int(k["first_pair"]) // res["n_devices"]]:
                words, at = [], 0
                base = arena.ctypes.data + int(pr["offset"])
                for _ in range(int(pr["events"])):
                    used = C.c_uint32()
                    assert ctx.L.r433b_event_to_bitbuffer(base + at, int(pr["bytes"]) - at, 0, bb.ctypes.data, C.byref(used)) == 0
                    ev = arena[int(pr["offset"]) + at:int(pr["offset"]) + at + used.value].view("<u4")
                    words += long_form(bb[0], int(ev[0]), int(ev[-1]))
                    at += used.value
                assert at == int(pr["bytes"])
                n_events += int(pr["events"])
                h = fnv1a(h, [4 * len(words), int(pr["events"]), int(pr["gated_single"]), int(pr["gated_multi"])] + words)
        assert n_events > 600 and ctx.stream_digest(0) == h
        ps.close()
        # the one-word forms are used: a one-row event of <= 16 bits (and < 8 syncs) took three words, now one
        rng = np.random.default_rng(8)
        for device, short in ((PWM, [pwm_event(rng, [(int(rng.integers(0, 3)), int(rng.integers(1, 17)))]) for _ in range(200)]),
                              (PCM, [pcm_event([int(rng.integers(1, 17))]) for _ in range(200)])):
            ctx.set_devices([device])
            ps, res = run(ctx, [_pd(RATE, p, g) for p, g in short])
            assert res["n_events"] == 200 and res["event_bytes"] == 4 * 200
            ps.close()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_custom_devices_match_the_oracle():
    custom_devices_match_the_oracle()


@pytest.mark.gpu
def test_default_devices_on_the_edge_cases():
    default_devices_match()


@pytest.mark.gpu
def test_stream_digest_hashes_the_long_form():
    stream_digest_hashes_the_long_form()
