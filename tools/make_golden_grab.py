"""Write tests/golden/grab.json: what the stock reference program writes with `-S MODE` for the capture runs of
tests/test_grab.py (file names, sizes and a sha256 prefix of each file), so that the GPU tests can check the
signal grabber where oracle/_ref is not built.  `--mixed` writes tests/golden/grab_mixed.json instead: `-S all` over
the interleaved files of different formats, rates and frequencies of tests/test_mixed.py, in command-line order.  Needs oracle/_ref/rtl_433 (build() makes it when the reference's
sources are present)."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import test_grab  # noqa: E402


def main_mixed():
    import test_mixed
    with tempfile.TemporaryDirectory() as d:
        paths = test_grab.write_case(test_mixed.grab_case(), d)
        got, _ = test_grab.reference_grabs(paths, "all")
    with open(test_mixed.GOLDEN, "w") as f:
        json.dump({"all": test_grab.fingerprint(got)}, f, indent=1)
        f.write("\n")
    print("mixed all", len(got), "files", file=sys.stderr)


def main():
    out = {}
    for case, files in test_grab.cases().items():
        modes = list(test_grab.MODES) if case == "ook_cu8" else ["all"]
        with tempfile.TemporaryDirectory() as d:
            paths = test_grab.write_case(files, d)
            out[case] = {}
            for mode in modes:
                got, lines = test_grab.reference_grabs(paths, mode)
                out[case][mode] = test_grab.fingerprint(got)
                print(case, mode, len(got), "files", file=sys.stderr)
    with open(test_grab.GOLDEN, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main_mixed() if "--mixed" in sys.argv[1:] else main()
