"""e64(oracle), e64(engine) and their ratio for every form x signal class of tests/test_conv_precision.py, on either
library: the emulation build (--lib emu, no GPU needed) or the product library (--lib cuda, the tensor-core forms
included).  e64 is the max error against the float64 convolution over the peak of the float64 output, maximised over
channels and segments; the ratio is the largest per channel / segment ratio where the engine's error is above the
2^-23 floor of the test's criterion (cells at the floor print '-'); bias is |mean signed error| / peak64.

Run: python tools/conv_precision_table.py --lib emu [--forms k0-M16-C1x1,...] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import test_conv_precision as tcp  # noqa: E402
from tests.backends import get_lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", choices=["emu", "cuda"], default="emu")
    ap.add_argument("--forms", default="", help="comma-separated form names (default: all the library can run)")
    ap.add_argument("--json", default="", help="also write the rows as JSON to this path")
    a = ap.parse_args()
    lib = get_lib(a.lib)
    forms = tcp.FORMS + (tcp.FORMS_TC if a.lib == "cuda" else [])
    if a.forms:
        want = set(a.forms.split(","))
        forms = [f for f in forms if f.name in want]
    if a.lib == "cuda":
        import torch
        print("#", torch.cuda.get_device_name(0))
    print("| form | signal | e64 oracle | e64 engine | ratio | k_form | bias oracle | bias engine |")
    print("|---|---|---|---|---|---|---|---|")
    out, worst = [], {}
    for f in forms:
        for s in tcp.signals(f):
            t0 = time.time()
            rows, calls, stages = tcp.measure(f, s, lib)
            f.check_selection(calls, stages)
            e_o = max(r[2] for r in rows)
            e_e = max(r[3] for r in rows)
            ratios = [r[3] / r[2] for r in rows if r[3] > tcp.FLOOR]
            ratio = max(ratios) if ratios else None
            if ratio is not None:
                worst[f.family] = max(worst.get(f.family, 0.0), ratio)
            print(f"| {f.name} | {s} | {e_o:.2g} | {e_e:.2g} | {'-' if ratio is None else f'{ratio:.2f}'} | "
                  f"{tcp.K_FORM[f.family]} | {max(r[5] for r in rows):.2g} | {max(r[6] for r in rows):.2g} |"
                  f"  <!-- {time.time() - t0:.1f} s -->", flush=True)
            out.append(dict(form=f.name, family=f.family, signal=s, e64_oracle=e_o, e64_engine=e_e, ratio=ratio,
                            rows=rows))
    print("\nworst ratio per family:", {k: round(v, 2) for k, v in sorted(worst.items())})
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(lib=a.lib, rows=out, worst=worst), fh, indent=1)


if __name__ == "__main__":
    main()
