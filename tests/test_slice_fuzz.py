"""-m gpu: k_slice2 on random packages through r433b_process_pulses.

The slicers themselves are fuzzed against the reference one (package, device) at a time on the CPU
(test_oracle_vs_ref.test_slicers_on_random_pulse_trains).  What only the kernel does is checked here: the (type,
length class) sort of k_bucket, the item -> (device, class, group of 32) decode with the idle lanes of a partial group,
the warp's arena reservation and its line-by-line copy out of window and scratch, the second pass of a warp with a
lane over kStageWords (4 KiB), the pair table, and one range per sample rate with its own slicer table.  The generator
puts package lengths on both sides of every class boundary, gives every (rate, type, class) segment a size that is not
a multiple of 32, mixes OOK and FSK packages and interleaves three sample rates; PCM packages with one long pulse give
one device outputs just under, at and just over 4096 bytes in the same segment as short packages, and gaps above every
device's reset limit make several events per (package, device), some of them gated.

Every package's events (device order, bitbuffer hash) must equal the reference's run_ook_demods / run_fsk_demods on
the same pulse_data_t (or, without the compiled reference, the oracle's slicers device by device); the fetched pair
table must be consistent with the event arena, and a gated run must be the ungated run filtered by the gate
predicate.  tests/test_emu_slice_fuzz.py runs the same body, smaller, under the SIMT emulator."""
import numpy as np
import pytest

import helpers
from oracle import orc, refh
from rtl_433_b200 import lib
from test_oracle_vs_ref import random_train

# input order of the packages: 250 k appears in two runs, so a rate's range gathers packages from both
RATE_RUNS = [250000, 1024000, 250000, 48000]
# pulse counts on both sides of the class boundaries of k_bucket (len_bucket: < 64, < 160, < 400, longer)
CLASS_BOUNDS = [(1, 64), (64, 160), (160, 400), (400, 1201)]
FORCED = [[1, 31, 32, 33, 63], [64, 65, 159], [160, 161, 399], [400, 401, 1199, 1200]]
STAGE_BYTES = 4096  # kStageWords * 4: a warp with a larger pair takes k_slice2's second pass
# one pulse of W samples at 250 k through the PCM device with 30 us bits (7.5 samples): about W / 60 bytes, so this
# sweep in steps of 16 bits gives that device every output size from 4096 - 28 to 4096 + 28 bytes
LONG_PCM_WIDTHS = [245300 + 120 * k for k in range(-7, 8)]


def len_class(n):
    return 0 if n < 64 else 1 if n < 160 else 2 if n < 400 else 3


def _train(rng, n, rate):
    """n pulses of one of random_train's four kinds (its pattern repeated), with some gaps above every device's
    reset limit (102.4 ms at most) so that a device emits several events for the package."""
    pulse, gap = random_train(rng, int(rng.integers(0, 4)))
    reps = -(-n // len(pulse))
    pulse, gap = np.tile(pulse, reps)[:n].copy(), np.tile(gap, reps)[:n].copy()
    if n > 4 and rng.random() < 0.4:
        for at in rng.integers(0, n - 1, int(rng.integers(1, 4))):
            gap[at] = int(rate * 0.11) + int(rng.integers(0, 5000))
    return pulse, gap


def _pd(rate, pulse, gap, fsk_f2=0, fsk_f1=0):
    pd = np.zeros(1, lib.PULSE_DATA_DTYPE)[0]  # pulse[num_pulses] / gap[num_pulses] stay 0 on every side
    n = len(pulse)
    pd["sample_rate"] = rate
    pd["num_pulses"] = n
    pd["pulse"][:n] = pulse
    pd["gap"][:n] = gap
    pd["fsk_f2_est"] = fsk_f2
    pd["fsk_f1_est"] = fsk_f1
    pd["freq1_hz"] = np.float32(433.92e6)
    pd["freq2_hz"] = np.float32(433.92e6)
    return pd


def make_set(seed, short_sizes, long_sizes):
    """-> [[pulse_data_t record] per stream], stream i = the packages of RATE_RUNS[i] in input order.
    Segment sizes (none a multiple of 32) are drawn from `short_sizes` for the < 64 class, from `long_sizes` for the
    others: a pulse of a random train makes an event for about one device in four, so long packages are few."""
    assert all(s % 32 for s in short_sizes + long_sizes)
    rng = np.random.default_rng(seed)
    runs = [[] for _ in RATE_RUNS]
    next_forced = [0] * len(FORCED)  # per class: the forced lengths go round over its segments
    for rate in sorted(set(RATE_RUNS)):
        run_ids = [i for i, r in enumerate(RATE_RUNS) if r == rate]
        for fsk in (0, 1):
            for b, (lo, hi) in enumerate(CLASS_BOUNDS):
                pds = []
                if rate == 250000 and not fsk and b == 0:
                    # long PCM pulses next to short packages: one device's pairs around the staging size; and
                    # long_pd of test_pulse_io (row spill over the whole bitbuffer for several devices)
                    pds += [_pd(rate, [w], [250000]) for w in LONG_PCM_WIDTHS]
                    pds += [_pd(rate, [20000] * 40, [100] * 39 + [250000])]
                count = int(rng.choice(long_sizes if b else short_sizes))
                while count <= len(pds) or count % 32 == 0:
                    count += 1
                for k in range(count - len(pds)):
                    # the forced lengths first, then lengths near the class's lower bound
                    if k < len(FORCED[b]):
                        n = FORCED[b][next_forced[b] % len(FORCED[b])]
                        next_forced[b] += 1
                    else:
                        n = int(rng.integers(lo, lo + 12))
                    pulse, gap = _train(rng, n, rate)
                    f2 = int(rng.integers(1, 9000)) if fsk else 0
                    pds.append(_pd(rate, pulse, gap, f2, int(rng.integers(-9000, 9000))))
                for pd in pds:
                    runs[run_ids[int(rng.integers(0, len(run_ids)))]].append(pd)
    for r in runs:
        rng.shuffle(r)
    return runs


def segments(runs):
    """(rate, type, class) -> number of packages: k_slice2's segments, one set per rate range."""
    out = {}
    for r in runs:
        for pd in r:
            key = (int(pd["sample_rate"]), 2 if pd["fsk_f2_est"] else 1, len_class(int(pd["num_pulses"])))
            out[key] = out.get(key, 0) + 1
    return out


def gated_out(ev, gates):
    """test_gates.gate_predicate from the collector's row count and longest row."""
    t = gates[ev["dev"]][0]
    return ev["num_rows"] >= 1 and ev["max_bits"] < t


def expected_events(runs, devices):
    """[[[(dev, hash)] per package] per stream] from the compiled reference, or None without it."""
    if not refh.available():
        return None
    ref = refh.Ref(store_bitbuffers=False)
    ref.register_defaults()
    try:
        assert len(ref.registered()) == len(devices)
        return [[[(dev, h) for dev, h, _bb in ref.slice_pulse_data(pd)] for pd in r] for r in runs]
    finally:
        ref.close()


def check_pairs(ctx, res, n_ranges):
    """The fetched pair table against the event arena."""
    pairs = res["pairs"]
    ev, nb = pairs["events"].astype(np.int64), pairs["bytes"].astype(np.int64)
    assert int(ev.sum()) == ctx.counts()["events"] == res["n_events"]
    assert np.array_equal(nb == 0, ev == 0), "a pair with bytes but no events, or events without bytes"
    used = nb > 0
    off = pairs["offset"].astype(np.int64)[used]
    end = off + nb[used]
    order = np.argsort(off)
    assert off.min() >= 0 and end.max() <= res["event_bytes"]
    assert (off[order][1:] >= end[order][:-1]).all(), "pair ranges overlap"
    assert int(nb.sum()) == res["event_bytes"], "the arena holds bytes that belong to no pair"
    # once per range; twice where the event arena of a new context (1 MiB) had to grow
    assert ctx.timing()["slice_launches"] in (n_ranges, 2 * n_ranges)


def slice_fuzz(seed, short_sizes, long_sizes, min_packages, min_events):
    devices = lib.default_device_table()
    gates = lib.default_gates(devices)
    runs = make_set(seed, short_sizes, long_sizes)
    segs = segments(runs)
    n_pkgs = sum(len(r) for r in runs)
    rates = sorted({r for r, _t, _b in segs})
    # the cases the generator is for
    assert len(rates) >= 3 and len(segs) == 8 * len(rates), segs
    assert all(v % 32 for v in segs.values()), segs
    lengths = {int(pd["num_pulses"]) for r in runs for pd in r}
    assert set(sum(FORCED, [])) <= lengths
    assert n_pkgs >= min_packages
    ps = lib.Pulses()
    for s, r in enumerate(runs):
        for pd in r:
            ps.add(pd, stream=s)
    ctx = lib.Context(0)
    try:
        ctx.set_devices(devices)
        ctx.process_pulses(ps)
        res = ctx.fetch()
        check_pairs(ctx, res, len(rates))
        pk = res["packages"]
        pairs = res["pairs"][pk["first_pair"] // res["n_devices"]]  # rows in fetched package order
        # one device with pairs over and at most kStageWords in the same class: warps of first- and second-pass lanes
        nb = pairs["bytes"].astype(np.int64)
        cls = np.array([len_class(int(n)) for n in pk["num_pulses"]])
        mixed = []
        for dv in range(len(devices)):
            for b in range(4):
                col = nb[cls == b, dv]
                if (col > STAGE_BYTES).any() and ((col > 0) & (col <= STAGE_BYTES)).any():
                    mixed.append((dv, b))
        assert mixed, "no device has pairs on both sides of the staging size in one class"
        near = nb[(nb > STAGE_BYTES - 32) & (nb <= STAGE_BYTES + 32)]
        assert (near == STAGE_BYTES).any() and (near < STAGE_BYTES).any() and (near > STAGE_BYTES).any(), sorted(set(near))

        want = expected_events(runs, devices)
        oracle = None
        if want is None:
            oracle = orc.Oracle(store_bitbuffers=True)
            oracle.add_devices(devices)
        plain = []
        total = 0
        for s, r in enumerate(runs):
            got = helpers.gpu_stream_results(ctx, s, store_bitbuffers=oracle is not None)
            assert len(got["packages"]) == len(r)
            per_pkg = [[] for _ in r]
            for e in got["events"]:
                per_pkg[e["package"]].append(e)
            for li, pd in enumerate(r):
                gp = got["packages"][li]
                n = int(pd["num_pulses"])
                assert gp["num_pulses"] == n and gp["sample_rate"] == int(pd["sample_rate"])
                assert np.array_equal(gp["pulse"][:n], pd["pulse"][:n]) and np.array_equal(gp["gap"][:n], pd["gap"][:n])
                mine = [(e["dev"], e["hash"]) for e in per_pkg[li]]
                if want is not None:
                    assert mine == want[s][li], f"stream {s} package {li} ({n} pulses): {len(mine)} vs {len(want[s][li])} events"
                else:
                    theirs = []
                    for dv, d in enumerate(devices):
                        if (d["modulation"] >= 16) == bool(pd["fsk_f2_est"]):
                            theirs += [(dv, bb.tobytes()) for bb in oracle.slice(dv, int(pd["sample_rate"]), pd["pulse"][:n], pd["gap"][:n])]
                    assert [(e["dev"], e["bitbuffer"].tobytes()) for e in per_pkg[li]] == theirs, f"stream {s} package {li}"
                total += len(mine)
            plain.append([(e["package"], e["dev"], e["hash"], gated_out(e, gates), e["num_rows"]) for e in got["events"]])
        assert total == ctx.counts()["events"] >= min_events

        # gates on: the ungated run filtered by the gate predicate, the dropped ones counted per pair and row class
        full_bytes = res["event_bytes"]
        ctx.set_gates(gates)
        ctx.process_pulses(ps)
        res = ctx.fetch()
        check_pairs(ctx, res, len(rates))
        pk = res["packages"]
        dropped_total = 0
        for s, r in enumerate(runs):
            got = helpers.gpu_stream_results(ctx, s)
            keep = [(p, d, h) for p, d, h, out, _rows in plain[s] if not out]
            assert [(e["package"], e["dev"], e["hash"]) for e in got["events"]] == keep, f"gated stream {s}"
            count1, countn = {}, {}
            for p, d, _h, out, rows in plain[s]:
                if out:
                    tgt = count1 if rows == 1 else countn
                    tgt[(p, d)] = tgt.get((p, d), 0) + 1
                    dropped_total += 1
            _, index = ctx.packages_of(s)
            for li, gi in enumerate(index):
                row = res["pairs"][int(pk["first_pair"][gi]) // res["n_devices"]]
                for dv in np.nonzero(row["gated_single"] | row["gated_multi"] | row["events"])[0]:
                    assert int(row["gated_single"][dv]) == count1.get((li, int(dv)), 0), (s, li, dv)
                    assert int(row["gated_multi"][dv]) == countn.get((li, int(dv)), 0), (s, li, dv)
                assert int(row["gated_single"].sum()) == sum(v for (q, _d), v in count1.items() if q == li)
                assert int(row["gated_multi"].sum()) == sum(v for (q, _d), v in countn.items() if q == li)
        assert res["n_gated"] == dropped_total == ctx.gated() > 0
        assert res["n_events"] + res["n_gated"] == total
        assert res["event_bytes"] < full_bytes
        ps.close()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_random_packages_through_k_slice2():
    """About 2,100 packages and 300 k events."""
    slice_fuzz(2024, [289, 321, 353, 385], [1, 3, 5, 7], 2000, 300000)
