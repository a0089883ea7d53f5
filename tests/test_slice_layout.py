"""-m gpu: k_slice2 on packages that stress its exact-length sort and the lane-interleaved copy of the widths.

k_bucket sorts a range's packages by type and descending length, gives every group of 32 as many rows as its first
(longest) package has pool entries, and copies the widths there lane by lane (r433b_kernels.cuh).  The set here has:
a group of one 1200-pulse package and 31 one-pulse packages (the most padding a group can have); per type and rate a
number of packages that is a multiple of 32, or one more; OSV1 packages whose sync is the entry after their last pulse
(the slicer reads pulse[num_pulses]) on the last lane of one group and the first lane of the next, next to OSV1
packages with data; DMC and PIWM packages of odd lengths, which read the widths at data-dependent positions; and OOK
and FSK packages at two sample rates in one r433b_process_pulses call.  Every package's events must equal the
oracle's slicers, device by device.  tests/test_emu_slice_layout.py runs the same body under the SIMT emulator, with
every device buffer, the copy included, ending at its computed size in front of a guard page."""
import numpy as np
import pytest

import helpers
from oracle import orc
from rtl_433_b200 import lib
from test_slice_fuzz import _pd, check_pairs

RATE_A, RATE_B = 250000, 1024000
MODULATIONS = (6, 9, 10, 11, 16)  # PWM, DMC, OSV1, PIWM_DC; FSK PCM


def devices():
    """The first default device of each modulation above, and an OSV1 device at the default one's timing."""
    table = lib.default_device_table()
    devs = [next(d for d in table if d["modulation"] == m) for m in MODULATIONS]
    osv1 = dict(devs[2])
    osv1["name"] = "OSV1 at 1.5 x"
    osv1["short_width"] = devs[2]["short_width"] * 1.5
    return devs + [osv1]


def osv1_train(rng, rate, short_us, data_pulses):
    """Twelve preamble pulses, the sync, then `data_pulses` Manchester widths; with none, the sync is the entry
    after the last pulse (num_pulses = 12)."""
    s = int(short_us * rate / 1e6)
    pulse, gap = [s] * 12, [s] * 11 + [2 * s]
    sync = (4 * s, 4 * s + s // 2)
    if data_pulses == 0:
        return pulse, gap, sync
    pulse.append(sync[0])
    gap.append(sync[1])
    for _ in range(data_pulses):
        pulse.append(s * int(rng.integers(1, 3)))
        gap.append(s * int(rng.integers(1, 3)))
    gap[-1] = int(rate * 0.02)
    return pulse, gap, None


def symbol_train(rng, rate, short_us, n):
    """n pulses of one and two short widths, the odd symbol (gap) now and then far off, the last gap a reset."""
    s = int(short_us * rate / 1e6)
    pulse = [s * int(rng.integers(1, 3)) for _ in range(n)]
    gap = [s * int(rng.integers(1, 3)) if rng.random() > 0.1 else s * 7 for _ in range(n)]
    gap[-1] = int(rate * 0.03)
    return pulse, gap


def make_set(seed):
    """-> [[pulse_data_t record] per stream]: stream 0 rate A, stream 1 rate B."""
    rng = np.random.default_rng(seed)
    devs = devices()
    osv1_us = devs[2]["short_width"]
    a, b = [], []
    # rate A, OOK: 64 packages, group 0 = one 1200-pulse package and 31 one-pulse ones
    pulse, gap = symbol_train(rng, RATE_A, devs[0]["short_width"], 1200)
    a.append(_pd(RATE_A, pulse, gap))
    a += [_pd(RATE_A, [int(rng.integers(20, 400))], [int(RATE_A * 0.02)]) for _ in range(63)]
    # rate A, FSK: 33 packages of odd lengths
    for _ in range(33):
        n = int(rng.integers(0, 40)) * 2 + 1
        pulse, gap = symbol_train(rng, RATE_A, devs[4]["short_width"] * 2, n)
        a.append(_pd(RATE_A, pulse, gap, fsk_f2=int(rng.integers(1, 9000)), fsk_f1=int(rng.integers(-9000, 9000))))
    # rate B, OOK: 20 packages longer than 12 pulses, 24 of 12 (sorted positions 20 .. 43: lane 31 of group 0 and
    # lane 0 of group 1), 21 shorter ones -- 65 in all
    for k in range(20):
        if k % 2:
            pulse, gap, _ = osv1_train(rng, RATE_B, osv1_us, int(rng.integers(1, 40)))
        else:
            pulse, gap = symbol_train(rng, RATE_B, devs[1 if k % 4 else 3]["short_width"], 2 * int(rng.integers(7, 60)) + 1)
        b.append(_pd(RATE_B, pulse, gap))
    for _ in range(24):
        pulse, gap, sync = osv1_train(rng, RATE_B, osv1_us, 0)
        pd = _pd(RATE_B, pulse, gap)
        pd["pulse"][12], pd["gap"][12] = sync
        b.append(pd)
    for _ in range(21):
        pulse, gap = symbol_train(rng, RATE_B, devs[1 if rng.random() < 0.5 else 3]["short_width"], 2 * int(rng.integers(1, 6)) + 1)
        b.append(_pd(RATE_B, pulse, gap))
    # rate B, FSK: 32 packages
    for _ in range(32):
        pulse, gap = symbol_train(rng, RATE_B, devs[4]["short_width"] * 2, int(rng.integers(1, 90)))
        b.append(_pd(RATE_B, pulse, gap, fsk_f2=int(rng.integers(1, 9000)), fsk_f1=int(rng.integers(-9000, 9000))))
    rng.shuffle(a)
    rng.shuffle(b)
    return [a, b]


def slice_layout(seed):
    devs = devices()
    runs = make_set(seed)
    counts = {}
    for r in runs:
        for pd in r:
            key = (int(pd["sample_rate"]), bool(pd["fsk_f2_est"]))
            counts[key] = counts.get(key, 0) + 1
    assert counts == {(RATE_A, False): 64, (RATE_A, True): 33, (RATE_B, False): 65, (RATE_B, True): 32}
    ps = lib.Pulses()
    for s, r in enumerate(runs):
        for pd in r:
            ps.add(pd, stream=s)
    ctx = lib.Context(0)
    oracle = orc.Oracle(store_bitbuffers=True)
    oracle.add_devices(devs)
    try:
        ctx.set_devices(devs)
        ctx.process_pulses(ps)
        res = ctx.fetch()
        check_pairs(ctx, res, 2)
        seen = set()
        total = 0
        for s, r in enumerate(runs):
            got = helpers.gpu_stream_results(ctx, s, store_bitbuffers=True)
            assert len(got["packages"]) == len(r)
            per_pkg = [[] for _ in r]
            for e in got["events"]:
                per_pkg[e["package"]].append(e)
            for li, pd in enumerate(r):
                n = int(pd["num_pulses"])
                fsk = bool(pd["fsk_f2_est"])
                theirs = []
                for dv, d in enumerate(devs):
                    if (d["modulation"] >= 16) == fsk:
                        bbs = oracle.slice(dv, int(pd["sample_rate"]), pd["pulse"][:n], pd["gap"][:n])
                        theirs += [(dv, bb.tobytes()) for bb in bbs]
                mine = [(e["dev"], e["bitbuffer"].tobytes()) for e in per_pkg[li]]
                assert mine == theirs, f"stream {s} package {li} ({n} pulses)"
                seen |= {devs[dv]["modulation"] for dv, _ in mine}
                total += len(mine)
        assert total == res["n_events"]
        # the slicers this set is for all produced events
        assert {6, 9, 10, 11, 16} <= seen, seen
    finally:
        ps.close()
        ctx.close()


@pytest.mark.gpu
def test_sorted_groups_and_interleaved_widths():
    slice_layout(11)
