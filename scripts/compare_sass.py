#!/usr/bin/env python3
"""Compare the device code of two builds of libkvquant_b200.so, kernel by kernel.

    python scripts/compare_sass.py OLD.so NEW.so

Runs `cuobjdump -sass` on both, splits the listing by function and compares the instruction text with what moves when
code moves stripped: addresses, encodings and branch targets.  Prints the kernels that were added, removed or differ
and exits 1 if there are any, 0 if the two builds hold the same kernels with the same instructions.  CPU only.
"""
import os
import re
import subprocess
import sys

_COMMENT = re.compile(r"/\*.*?\*/")          # /*0010*/ addresses and /* 0x... */ encodings
_TARGET = re.compile(r"\b0x[0-9a-f]+\b")     # branch / call targets of control-flow instructions
_FLOW = re.compile(r"\b(BRA|BRX|JMP|JMX|CALL|BSSY|BSYNC|BREAK|WARPSYNC|RET|EXIT)\b")


def _cuobjdump():
    return os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def kernels(path):
    """{mangled function name: [normalised instruction lines]}"""
    text = subprocess.run([_cuobjdump(), "-sass", path], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        s = line.strip()
        if s.startswith("Function :"):
            cur = out.setdefault(s.split(":", 1)[1].strip(), [])
            continue
        if s.startswith("Fatbin"):       # header of the next translation unit (it names the source path)
            cur = None
        if cur is None or s.startswith("."):
            continue
        s = _COMMENT.sub("", s).strip()
        if not s:
            continue
        if _FLOW.search(s):
            s = _TARGET.sub("<target>", s)
        cur.append(s)
    return out


def main(argv):
    if len(argv) != 3:
        print(__doc__)
        return 2
    old, new = kernels(argv[1]), kernels(argv[2])
    removed = sorted(set(old) - set(new))
    added = sorted(set(new) - set(old))
    differ = sorted(k for k in set(old) & set(new) if old[k] != new[k])
    for tag, names in (("removed", removed), ("added", added), ("differs", differ)):
        for k in names:
            print("%-8s %s" % (tag, k))
    print("%d kernels in %s, %d in %s: %d removed, %d added, %d differ" %
          (len(old), argv[1], len(new), argv[2], len(removed), len(added), len(differ)))
    return 1 if (removed or added or differ) else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
