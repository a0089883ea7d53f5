"""Capture-file ingest: the part of `rtl_433 -r FILE ...` in front of the hot path.

* `parse_capture_name()` restates file_info_parse_filename() / file_type() (src/fileformat.c:173-328):
  sample rate, centre frequency and sample format are read from tags in the file NAME
  ("g001_433.92M_250k.cu8", "am:s16:path", "868M_1024k.cs16", ...).
* `load_batches()` groups files by (format, rate, frequency) -- one r433b batch each -- and packs
  them at 16-byte aligned starts with their true lengths (r433b_batch.lengths).
* `python -m rtl_433_b200.captures FILES...` replays capture files through the GPU path and
  prints, per file, the detected packages and the bitbuffer rows every requested device's slicer
  produced, in rtl_433's "{len}hex" notation (what `rtl_433 -R n:vv` logs before decoding).
* `--chunk-mb N` streams every group through a chain (r433b_process_chained): each call reads the next N MiB of
  whole blocks of every file at an offset, so host memory is about (files in the group) x N MiB; the printed
  output is that of the plain run.  It does not combine with `-S`.
* `--split [N|auto]` walks long files in segments of N blocks on separate warps (r433b_set_split; `auto` sizes them
  from the batch); the printed output, and the files `-S all` writes, are those of the plain run.  It does not
  combine with `--chunk-mb`.
* `-S all [--grab-dir DIR]` is the signal grabber (src/samp_grab.c): every frame's IQ is written to
  `g%03u_%gM_%gk.cu8|.cs16` files as `rtl_433 -S all -r FILES...` writes them.  The grabber's ring runs
  across the files in processing order, which is group order: the files of each (format, rate,
  frequency) group in command-line order, groups in the order their first file appears.  That is the
  command-line order unless groups interleave.  The modes unknown / known / undecoded depend on what the
  decoders return, so they live behind r433b_dispatch (INTEGRATION.md), not here.
* `--one-batch` replays every file in one mixed batch (r433b_process_mixed), each with its own format, rate and
  frequency, in command-line order: the report is the same, and the files `-S all` writes are those of
  `rtl_433 -S all -r f1 -r f2 ...` whatever the groups.  It does not combine with `--chunk-mb` or `--split`.

Decoding itself stays with the reference's decoders (INTEGRATION.md); this module stops at the
bitbuffer like the rest of the package.
"""
import argparse
import os
import re
import sys

import numpy as np

from . import lib

DEFAULT_RATE = 250000        # include/rtl_433.h:13
DEFAULT_FREQ = 433920000     # include/rtl_433.h:14

# format tags of file_type(), src/fileformat.c:222-252 (only what the hot path can take is mapped)
_FORMAT_TAGS = {"cu8": "cu8", "data": "cu8", "complex16u": "cu8", "cs8": "cs8", "complex16s": "cs8", "cs16": "cs16",
                "cf32": "cf32", "cfile": "cf32", "complex": "cf32", "s16": "s16", "u8": "u8", "s8": "s8", "u16": "u16",
                "u32": "u32", "s32": "s32", "f32": "f32", "cs32": "cs32"}
_CONTENT_TAGS = {"i", "q", "iq", "am", "fm", "vcd", "ook", "logic", "sigmf"}


def _scan(text, info):
    """One pass of file_type() over `text`, updating info in place (later tags win)."""
    p, n = 0, len(text)
    while p < n:
        ch = text[p]
        if ch.isdigit() and ch.isascii():
            start = p
            while p < n and text[p] in "0123456789":
                p += 1
            if p < n and text[p] == ".":
                p += 1
                if not (p < n and text[p] in "0123456789"):
                    continue  # "if not [0-9] after '.' abort": the number is dropped
                while p < n and text[p] in "0123456789":
                    p += 1
            s = p
            while p < n and text[p].isascii() and text[p].isalpha():
                p += 1
            num = float(text[start:s])
            unit = text[s:p]
            scale = {"k": 1e3, "m": 1e6, "g": 1e9}.get(unit[:1].lower(), 1.0) if unit else 1.0
            low = unit.lower()
            if low == "m":
                info["center_frequency"] = int(num * 1e6)
            elif low == "k":
                info["sample_rate"] = int(num * 1e3)
            elif low == "hz":
                info["center_frequency"] = int(num)
            elif low == "sps":
                info["sample_rate"] = int(num)
            elif len(unit) == 3 and low[1:] == "hz" and scale > 1.0:
                info["center_frequency"] = int(num * scale)
            elif len(unit) == 4 and low[1:] == "sps" and scale > 1.0:
                info["sample_rate"] = int(num * scale)
        elif ch.isascii() and ch.isalpha():
            start = p
            while p < n and text[p].isascii() and text[p].isalnum():
                p += 1
            tag = text[start:p].lower()
            if tag in _FORMAT_TAGS:
                info["format"] = _FORMAT_TAGS[tag]
            elif tag in _CONTENT_TAGS:
                info["content"] = tag
        else:
            p += 1


def parse_capture_name(spec):
    """-> dict(path, format, content, sample_rate, center_frequency); 0 = not given in the name.
    A prefix up to the last ':' (not followed by a backslash) is an override, parsed last."""
    info = {"format": None, "content": None, "sample_rate": 0, "center_frequency": 0}
    cut = None
    for m in re.finditer(":", spec):
        if spec[m.start() + 1:m.start() + 2] == "\\":
            break
        cut = m.start()
    if cut is not None and cut < 64:
        path = spec[cut + 1:]
        _scan(path, info)
        _scan(spec[:cut], info)
    else:
        path = spec
        _scan(spec, info)
    # file_type_guess_auto_format(): nothing (or just "iq") means cu8
    if info["format"] is None and info["content"] in (None, "iq"):
        info["format"] = "cu8"
    info["path"] = path
    return info


def read_sigmf(path):
    """A SigMF archive as `rtl_433 -r x.sigmf` reads it (sigmf_reader_open(), src/sigmf.c:336-434, and the file loop
    of src/rtl_433.c:1712-1723) -> dict(data, sample_rate, center_frequency, datatype, data_offset).

    The first `.sigmf-meta` member names the stream; `global."core:sample_rate"` and the LAST capture's
    `"core:frequency"` (src/sigmf.c:127-287 overwrites first_frequency per capture) become rate and centre
    frequency; the samples are the member named like the meta file with `-data`.  Two properties of the reference
    are kept because results depend on them: the payload is demodulated as cu8 whatever "core:datatype" says
    (src/rtl_433.c:1719), and the block loop reads from the start of the data member to the END OF THE ARCHIVE,
    i.e. including the tar padding and end-of-archive blocks behind the samples."""
    import json

    def members(raw):
        # ustar walk like microtar's: 512-byte headers, octal size at 124, type flag at 156, all-zero block ends
        pos = 0
        while pos + 512 <= len(raw):
            h = raw[pos:pos + 512]
            if h[0] == 0:
                break
            name = h[:100].split(b"\0", 1)[0].decode("latin-1")
            size = int(h[124:136].split(b"\0", 1)[0].strip() or b"0", 8)
            kind = h[156:157]
            yield name, size, kind, pos + 512
            pos += 512 + (size + 511) // 512 * 512

    raw = np.fromfile(path, dtype=np.uint8).tobytes()
    stream, meta = None, None
    for name, size, kind, at in members(raw):
        if kind not in (b"0", b"\0"):
            continue
        if name.lower().endswith(".sigmf-meta"):
            if stream is not None and name != stream:  # "updated meta file": the later stream name wins
                stream, meta = None, None
            if stream is None:
                stream, meta = name, json.loads(raw[at:at + size].decode("utf-8", "replace") or "{}")
    if stream is None:
        raise ValueError(f"{path}: SigMF input file with no streams")
    info = {"sample_rate": 0, "center_frequency": 0, "datatype": None}
    g = meta.get("global", {}) if isinstance(meta, dict) else {}
    if "core:sample_rate" in g:
        info["sample_rate"] = int(float(g["core:sample_rate"])) & 0xffffffff
    info["datatype"] = g.get("core:datatype")
    for cap in meta.get("captures", []) if isinstance(meta, dict) else []:
        if "core:frequency" in cap:
            info["center_frequency"] = int(float(cap["core:frequency"])) & 0xffffffff
    want = stream[:-4] + "data"
    for name, size, kind, at in members(raw):
        if name == want:
            info["data_offset"] = at
            info["data"] = np.frombuffer(raw, dtype=np.uint8)[at:].copy()
            return info
    raise ValueError(f"{path}: SigMF input file with no stream data")


_ABI_FORMAT = {"cu8": lib.FMT_CU8, "cs8": lib.FMT_CS8, "cs16": lib.FMT_CS16, "cf32": lib.FMT_CF32}


def load_batches(specs, default_rate=DEFAULT_RATE, default_freq=DEFAULT_FREQ, uniform="auto", one_batch=False):
    """-> list of dict(format, sample_rate, center_frequency, files, data, offsets, lengths), one per
    (format, rate, frequency) group, files in command-line order inside a group.

    `uniform`: put the files of a group on ONE stride (the longest file, rounded up) so that r433b_process() can
    overlap the host-to-device copy with the kernels, time slice by time slice (one strided copy per slice);
    "auto" does it when the padding costs less than half again the bytes, False packs the files back to back.

    one_batch: ONE batch of every file in command-line order, packed back to back at 32-byte aligned starts, for
    r433b_process_mixed: format "mixed", and per file "formats" (names), "abi_formats", "rates" and "freqs"."""
    if one_batch:
        return [_mixed_batch(specs, default_rate, default_freq)]
    groups = {}
    preloaded = {}
    for spec in specs:
        info = parse_capture_name(spec)
        if info["content"] == "sigmf":
            # container: format, rate and frequency come from the archive's metadata, not from the name
            sm = read_sigmf(info["path"])
            preloaded[info["path"]] = sm["data"]
            groups.setdefault(("cu8", sm["sample_rate"], sm["center_frequency"]), []).append(info["path"])
            continue
        if info["format"] not in _ABI_FORMAT:
            raise ValueError(f"{spec}: format {info['format']!r} is not on the GPU path (cu8, cs8, cs16, cf32 are)")
        key = (info["format"], info["sample_rate"] or default_rate, info["center_frequency"] or default_freq)
        groups.setdefault(key, []).append(info["path"])
    out = []
    for (fmt, rate, freq), paths in groups.items():
        ss = {"cu8": 2, "cs8": 2, "cs16": 4, "cf32": 8}[fmt]
        align = 32 if fmt == "cf32" else 16
        bufs = [preloaded[p] if p in preloaded else np.fromfile(p, dtype=np.uint8) for p in paths]
        lengths = np.array([len(b) // ss * ss for b in bufs], np.uint64)  # a trailing partial sample is dropped
        offsets = np.zeros(len(bufs) + 1, np.uint64)
        longest = (int(lengths.max()) + 4095) // 4096 * 4096 if len(bufs) else 0
        if uniform is True or (uniform == "auto" and len(bufs) > 1 and longest * len(bufs) <= 1.5 * float(lengths.sum())):
            offsets = np.arange(len(bufs) + 1, dtype=np.uint64) * np.uint64(longest)
        else:
            for i, n in enumerate(lengths):
                offsets[i + 1] = offsets[i] + (int(n) + align - 1) // align * align
        data = np.zeros(int(offsets[-1]), np.uint8)
        for i, b in enumerate(bufs):
            data[int(offsets[i]):int(offsets[i]) + int(lengths[i])] = b[:int(lengths[i])]
        out.append({"format": fmt, "abi_format": _ABI_FORMAT[fmt], "sample_rate": rate, "center_frequency": freq,
                    "files": paths, "data": data, "offsets": offsets, "lengths": lengths})
    return out


def _mixed_batch(specs, default_rate=DEFAULT_RATE, default_freq=DEFAULT_FREQ):
    files, fmts, rates, freqs, bufs = [], [], [], [], []
    for spec in specs:
        info = parse_capture_name(spec)
        if info["content"] == "sigmf":
            sm = read_sigmf(info["path"])
            fmt, rate, freq, buf = "cu8", sm["sample_rate"], sm["center_frequency"], sm["data"]
        else:
            if info["format"] not in _ABI_FORMAT:
                raise ValueError(f"{spec}: format {info['format']!r} is not on the GPU path (cu8, cs8, cs16, cf32 are)")
            fmt, rate = info["format"], info["sample_rate"] or default_rate
            freq, buf = info["center_frequency"] or default_freq, np.fromfile(info["path"], dtype=np.uint8)
        files.append(info["path"])
        fmts.append(fmt)
        rates.append(rate)
        freqs.append(freq)
        bufs.append(buf)
    lengths = np.array([len(b) // _IN_BYTES[_ABI_FORMAT[f]] * _IN_BYTES[_ABI_FORMAT[f]] for b, f in zip(bufs, fmts)], np.uint64)
    offsets = np.zeros(len(bufs) + 1, np.uint64)
    for i, n in enumerate(lengths):
        offsets[i + 1] = offsets[i] + (int(n) + 31) // 32 * 32
    data = np.zeros(int(offsets[-1]), np.uint8)
    for i, b in enumerate(bufs):
        data[int(offsets[i]):int(offsets[i]) + int(lengths[i])] = b[:int(lengths[i])]
    return {"format": "mixed", "files": files, "formats": fmts, "abi_formats": [_ABI_FORMAT[f] for f in fmts],
            "rates": rates, "freqs": freqs, "data": data, "offsets": offsets, "lengths": lengths}


def row_code(bb, row):
    """rtl_433's '{len}hex' row notation (src/decoder_util.c:61-90) of a re-inflated bitbuffer record."""
    n = int(bb["bits_per_row"][row])
    nbytes = (n + 7) // 8
    flat = bb["bb"].reshape(-1)
    data = bytes(flat[row * 128:row * 128 + nbytes])
    return "{%d}%s" % (n, data.hex()[:(n + 3) // 4])


def grab_name(counter, center_frequency, samp_rate, sample_size):
    """samp_grab_write()'s file name, src/samp_grab.c:139 (cs8 is grabbed as cu8, cf32 as cs16)."""
    return "g%03u_%gM_%gk.%s" % (counter, center_frequency / 1e6, samp_rate / 1e3, "cu8" if sample_size == 2 else "cs16")


class Grabber:
    """The run-wide state of `rtl_433 -S`: the ring tail carried from batch to batch, the file counter and the
    directory the files go to.  Call write() once per batch, in processing order, after ctx.fetch() (and, for the
    modes that need decoder results, after the dispatch and r433b_analyze)."""

    BLOCK = 128 * 1024

    def __init__(self, directory=".", err=None, page_bytes=256 << 20):
        self.dir = directory
        self.err = err if err is not None else sys.stderr
        self.page = page_bytes
        self.counter = 1  # samp_grab_create()
        self.ring = None  # (bytes pushed, tail)

    def write(self, ctx, mode, center_frequency, samp_rate, sample_size, per_stream=None):
        """Write the batch's files; -> their names.  per_stream: (center_frequency, samp_rate, sample_size) of every
        stream of a mixed batch, which then name each grab from the stream whose block call ended its frame."""
        prior = None if self.ring is None else (self.ring[0], self.ring[1], self.counter)
        plan = ctx.grab_plan(mode, prior)
        names = []
        i = 0
        while i < len(plan):
            j, total = i, 0
            while j < len(plan) and (j == i or total + int(plan["bytes"][j]) <= self.page):
                total += int(plan["bytes"][j])
                j += 1
            data = ctx.grab_copy(i, j - i, total)
            at = 0
            for g in plan[i:j]:
                n = int(g["bytes"])
                fmt = (center_frequency, samp_rate, sample_size) if per_stream is None else per_stream[int(g["stream"])]
                names.append(self._file(data[at:at + n], int(g["grab_len"]), *fmt))
                at += n
            i = j
        self.ring = ctx.grab_tail()
        return names

    def _file(self, data, grab_len, center_frequency, samp_rate, sample_size):
        wanted = (sample_size * grab_len) & 0xffffffff
        wanted = (wanted + self.BLOCK - wanted % self.BLOCK) & 0xffffffff
        if wanted > len(data):
            self.err.write("Signal bigger than buffer, signal = %u > buffer %u !!\n" % (wanted, len(data)))
        while True:  # names that exist are skipped, the counter runs on
            name = grab_name(self.counter, center_frequency, samp_rate, sample_size)
            self.counter += 1
            if not os.path.exists(os.path.join(self.dir, name)):
                break
        self.err.write("*** Saving signal to file %s (%u samples, %u bytes)\n" % (name, grab_len, len(data)))
        with open(os.path.join(self.dir, name), "wb") as f:
            f.write(data.tobytes())
        return name


def _file_rows(ctx, res, i, devs, protocols, max_rows):
    """What one stream of a fetched batch adds to its file's report: package lines, every event's row text (None when
    the event is not shown) in dispatch order."""
    pk = res["packages"][res["packages"]["stream"] == i]
    events = []

    def on_event(pkg, dev, pd, bb, events=events):
        events.append((pkg, dev, bb.copy()))
        return 0

    ctx.dispatch(i, on_event)
    lines = []
    for k in pk:
        kind = "OOK" if k["type"] == lib.PACKAGE_OOK else "FSK"
        lines.append(f"  {kind} package @{int(k['offset'])}: {int(k['num_pulses'])} pulses, "
                     f"levels low {int(k['ook_low_estimate'])} high {int(k['ook_high_estimate'])}")
    rows = []
    for pkg, dev, bb in events:
        shown = protocols or any(int(b) > 16 for b in bb["bits_per_row"][:int(bb["num_rows"])])
        rows.append(f"    [{devs[dev]['protocol_num']}] {devs[dev]['name']}: "
                    + " ".join(row_code(bb, r) for r in range(min(int(bb["num_rows"]), max_rows))) if shown else None)
    return len(pk), lines, rows


def _print_file(out, path, batch, n_samples, rep):
    n_pk, lines, rows = rep
    out(f"{path}: {batch['format']} {batch['sample_rate']} S/s {batch['center_frequency']} Hz, "
        f"{n_samples} samples, {n_pk} package(s)")
    for line in lines:
        out(line)
    for line in [r for r in rows if r is not None][:40]:
        out(line)
    return {"file": path, "packages": n_pk, "events": len(rows)}


_IN_BYTES = {lib.FMT_CU8: 2, lib.FMT_CS8: 2, lib.FMT_CS16: 4, lib.FMT_CF32: 8}


def _chunked_groups(specs, default_rate=DEFAULT_RATE, default_freq=DEFAULT_FREQ):
    """The groups of load_batches() without their data: per file a reader of (offset, count) bytes and its length."""
    groups = {}
    for spec in specs:
        info = parse_capture_name(spec)
        if info["content"] == "sigmf":
            sm = read_sigmf(info["path"])
            key, src = ("cu8", sm["sample_rate"], sm["center_frequency"]), sm["data"]
        else:
            if info["format"] not in _ABI_FORMAT:
                raise ValueError(f"{spec}: format {info['format']!r} is not on the GPU path (cu8, cs8, cs16, cf32 are)")
            key, src = (info["format"], info["sample_rate"] or default_rate, info["center_frequency"] or default_freq), None
        groups.setdefault(key, []).append((info["path"], src))
    out = []
    for (fmt, rate, freq), files in groups.items():
        ss = _IN_BYTES[_ABI_FORMAT[fmt]]
        sizes = [len(src) if src is not None else os.path.getsize(p) for p, src in files]
        out.append({"format": fmt, "abi_format": _ABI_FORMAT[fmt], "sample_rate": rate, "center_frequency": freq,
                    "files": [p for p, _ in files], "sources": [src for _, src in files],
                    "lengths": np.array([n // ss * ss for n in sizes], np.uint64)})
    return out


def _replay_chunked(ctx, batch, chunk_mb, report):
    """One group through a chain: every round reads the next `chunk_mb` MiB of whole blocks of every file at an
    offset, so host memory is about (files in the group) x chunk_mb MiB.  -> per file the merged report."""
    block = 262144 * (2 if batch["abi_format"] == lib.FMT_CF32 else 1)  # DEFAULT_BUF_LENGTH, of cs16 for cf32
    step = max(1, (chunk_mb << 20) // block) * block
    n = len(batch["files"])
    lengths = [int(v) for v in batch["lengths"]]
    reps = [(0, [], []) for _ in range(n)]
    chain = lib.Chain(ctx, n)
    try:
        for r in range((max(lengths) + step - 1) // step if max(lengths) else 1):
            at = r * step
            data = np.zeros(n * step, np.uint8)
            lens, last, live = [], [], []
            for i, (path, src) in enumerate(zip(batch["files"], batch["sources"])):
                take = max(0, min(step, lengths[i] - at))
                if take:
                    data[i * step:i * step + take] = (src[at:at + take] if src is not None
                                                       else np.fromfile(path, dtype=np.uint8, count=take, offset=at))
                live.append(at < lengths[i] or (at == 0 and lengths[i] == 0))
                lens.append(take)
                last.append(1 if at + take >= lengths[i] else 0)
            offsets = np.arange(n + 1, dtype=np.uint64) * np.uint64(step)
            ctx.process(data, offsets, batch["abi_format"], batch["sample_rate"], batch["center_frequency"],
                        lengths=lens, chain=chain, last=last)
            res = ctx.fetch()
            for i in range(n):
                if live[i]:
                    k, lines, rows = report(res, i)
                    reps[i] = (reps[i][0] + k, reps[i][1] + lines, reps[i][2] + rows)
    finally:
        chain.close()
    return reps


def _replay_mixed(ctx, grabber, grab_mode, batch, report, out):
    """Every file in one mixed batch; the report in command-line order."""
    ctx.process_mixed(batch["data"], batch["offsets"], batch["abi_formats"], batch["rates"], batch["freqs"],
                      lengths=batch["lengths"])
    res = ctx.fetch()
    if grabber:
        ss = {"cu8": 2, "cs8": 2, "cs16": 4, "cf32": 4}
        grabber.write(ctx, grab_mode, None, None, None,
                      per_stream=[(f, r, ss[t]) for f, r, t in zip(batch["freqs"], batch["rates"], batch["formats"])])
    summary = []
    for i, path in enumerate(batch["files"]):
        one = {"format": batch["formats"][i], "sample_rate": batch["rates"][i], "center_frequency": batch["freqs"][i]}
        n_samples = int(batch["lengths"][i]) // _IN_BYTES[batch["abi_formats"][i]]
        summary.append(_print_file(out, path, one, n_samples, report(res, i)))
    return summary


def replay(specs, protocols=None, cuda_device=0, max_rows=8, out=print, grab_mode=0, grab_dir=".", chunk_mb=0, split=0,
           one_batch=False):
    """Run capture files through the GPU path; report packages and slicer output per file.  grab_mode 1 writes
    every frame's IQ to grab_dir (`-S all`).  chunk_mb > 0 streams every group through a chain, chunk_mb MiB of every
    file per call: the report is the same, host memory stays bounded.  split (blocks per segment, or lib.SPLIT_AUTO)
    walks long files in segments on separate warps: the report is the same, long files finish sooner.  one_batch
    replays every file in one mixed batch in command-line order (r433b_process_mixed): the report is the same, and
    -S all writes what the reference writes for the files in that order."""
    table = lib.default_device_table(include_disabled=True)
    if protocols:
        devs = [d for d in table if d["protocol_num"] in set(protocols)]
    else:
        devs = [d for d in table if d["disabled"] == 0]
    if grab_mode not in (0, lib.GRAB_ALL):
        raise ValueError("grab modes unknown / known / undecoded need decoder results: use r433b_grab_plan after r433b_dispatch")
    if grab_mode and chunk_mb:
        raise ValueError("the signal grabber does not run on chained batches (-S with --chunk-mb)")
    if split and chunk_mb:
        raise ValueError("segmented replay does not run on chained batches (--split with --chunk-mb)")
    if one_batch and (chunk_mb or split):
        raise ValueError("a mixed batch runs neither chained (--chunk-mb) nor split (--split)")
    ctx = lib.Context(cuda_device)
    ctx.set_devices(devs)
    if split:
        ctx.set_split(split)
    grabber = Grabber(grab_dir) if grab_mode else None
    summary = []
    try:
        if one_batch:
            return _replay_mixed(ctx, grabber, grab_mode, load_batches(specs, one_batch=True)[0],
                                 lambda res, i: _file_rows(ctx, res, i, devs, protocols, max_rows), out)
        groups = _chunked_groups(specs) if chunk_mb else load_batches(specs)
        for batch in groups:
            if chunk_mb:
                reps = _replay_chunked(ctx, batch, chunk_mb,
                                       lambda res, i: _file_rows(ctx, res, i, devs, protocols, max_rows))
            else:
                ctx.process(batch["data"], batch["offsets"], batch["abi_format"], batch["sample_rate"],
                            batch["center_frequency"], lengths=batch["lengths"])
                res = ctx.fetch()
                if grabber:
                    ss = {"cu8": 2, "cs8": 2, "cs16": 4, "cf32": 4}[batch["format"]]
                    grabber.write(ctx, grab_mode, batch["center_frequency"], batch["sample_rate"], ss)
                reps = [_file_rows(ctx, res, i, devs, protocols, max_rows) for i in range(len(batch["files"]))]
            for i, path in enumerate(batch["files"]):
                n_samples = int(batch["lengths"][i]) // _IN_BYTES[batch["abi_format"]]
                summary.append(_print_file(out, path, batch, n_samples, reps[i]))
    finally:
        ctx.close()
    return summary


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("files", nargs="+", help="capture files; rate/frequency/format come from the name as in rtl_433 -r")
    ap.add_argument("-R", dest="protocols", type=int, action="append", help="protocol number(s); default: all enabled")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("-S", dest="grab", choices=["all"], help="signal grabber: write every frame's IQ (rtl_433 -S all)")
    ap.add_argument("--grab-dir", default=".", help="directory for the grabbed files (default: the current one)")
    ap.add_argument("--chunk-mb", type=int, default=0, metavar="N",
                    help="stream every file through a chain, N MiB of whole blocks per call (bounded host memory)")
    ap.add_argument("--split", nargs="?", const="auto", default=None, metavar="N|auto",
                    help="walk long files in segments of N blocks on separate warps (auto: sized from the batch)")
    ap.add_argument("--one-batch", action="store_true",
                    help="every file in one mixed batch, each with its own format, rate and frequency, in command-line order")
    a = ap.parse_args(argv)
    split = 0
    if a.split is not None:
        if a.split == "auto":
            split = lib.SPLIT_AUTO
        elif a.split.isdigit() and int(a.split) > 0:
            split = int(a.split)
        else:
            ap.error("--split takes a positive number of blocks or 'auto'")
    if a.split is not None and a.chunk_mb:
        ap.error("--split does not run with --chunk-mb: segmented replay does not run on chained batches")
    if a.chunk_mb < 0:
        ap.error("--chunk-mb must be positive")
    if a.grab and a.chunk_mb:
        ap.error("-S does not run with --chunk-mb: the signal grabber does not run on chained batches")
    if a.one_batch and (a.chunk_mb or a.split is not None):
        ap.error("--one-batch does not run with --chunk-mb or --split: a mixed batch runs neither chained nor split")
    replay(a.files, a.protocols, a.device, grab_mode=lib.GRAB_ALL if a.grab else 0, grab_dir=a.grab_dir,
           chunk_mb=a.chunk_mb, split=split, one_batch=a.one_batch)


if __name__ == "__main__":
    main()
