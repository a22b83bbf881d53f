"""Compare the SASS of the kernels two builds of one .cu file have in common.

    python tools/sass_compare.py OLD.o NEW.o [--match sdf_fused_kernel]

Both objects are disassembled with `cuobjdump -sass`.  A kernel is keyed by its mangled name with the file's anonymous
namespace tag removed (it changes with the file's contents) and with a trailing template argument equal to 0 dropped, so
that `f<..., Src>` of OLD and `f<..., Src, 0>` of NEW (a new last template parameter whose default is 0) are the same
kernel.  Prints one line per kernel of OLD: identical, differs (with the first differing instruction) or missing in NEW;
exits 1 unless every kernel of OLD is identical in NEW.  Needs no GPU.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys

_ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]{8}")


def kernels(obj: str) -> dict[str, list[str]]:
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = re.sub(r"ELi0EEEv", "EEEv", _ANON.sub("ANON", m.group(1)))
            out[name] = []
        elif name is not None and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            out[name].append(line.split(";")[0].strip())
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--match", default="", help="only kernels whose name contains this string")
    args = ap.parse_args(argv)
    old, new = kernels(args.old), kernels(args.new)
    bad = 0
    for name, body in old.items():
        if args.match not in name:
            continue
        if name not in new:
            print(f"missing  {name}")
            bad += 1
        elif new[name] != body:
            i = next((k for k, (a, b) in enumerate(zip(body, new[name])) if a != b), min(len(body), len(new[name])))
            print(f"differs  {name}: {len(body)} vs {len(new[name])} instructions, first at {i}")
            bad += 1
        else:
            print(f"same     {name} ({len(body)} instructions)")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
