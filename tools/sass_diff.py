"""Compare the machine code of two libbevk.so builds function by function.

    python tools/sass_diff.py OLD.so NEW.so [--show NAME]

Runs cuobjdump -sass on both, drops the per-instruction address and encoding comments, and reports functions present
in one build only and functions whose instruction text differs.  Build both libraries with the same flags (build.py's
defaults, e.g. `nvcc` with build.FLAGS on a checkout of each commit) so that only the source change can differ.
Exit status 0 when every function is identical.
"""
from __future__ import annotations

import argparse
import difflib
import os
import re
import subprocess
import sys

CUOBJDUMP = os.environ.get("CUOBJDUMP", "/usr/local/cuda/bin/cuobjdump")
_FUNC = re.compile(r"^\s*Function : (\S+)")
_ADDR = re.compile(r"/\*[0-9a-f]{4,}\*/")            # /*0a30*/ instruction address
_ENC = re.compile(r"/\* 0x[0-9a-f]{16} \*/")          # /* 0x... */ encoding words


def functions(lib: str) -> dict[str, list[str]]:
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs: dict[str, list[str]] = {}
    cur = None
    for line in out.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        if cur is None:
            continue
        text = _ENC.sub("", _ADDR.sub("", line)).strip()
        if text:
            cur.append(text)
    return funcs


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--show", help="print the instruction diff of this mangled name")
    args = ap.parse_args()
    old, new = functions(args.old), functions(args.new)
    only_old, only_new = sorted(set(old) - set(new)), sorted(set(new) - set(old))
    changed = sorted(f for f in set(old) & set(new) if old[f] != new[f])
    print(f"functions: {len(old)} old, {len(new)} new, {len(changed)} changed, "
          f"{len(only_old)} only in old, {len(only_new)} only in new")
    for title, names in (("only in old", only_old), ("only in new", only_new), ("changed", changed)):
        for f in names:
            extra = f" ({len(old[f])} -> {len(new[f])} instructions)" if title == "changed" else ""
            print(f"{title}: {f}{extra}")
    if args.show:
        sys.stdout.writelines(difflib.unified_diff([l + "\n" for l in old.get(args.show, [])],
                                                   [l + "\n" for l in new.get(args.show, [])], "old", "new"))
    return 1 if only_old or only_new or changed else 0


if __name__ == "__main__":
    sys.exit(main())
