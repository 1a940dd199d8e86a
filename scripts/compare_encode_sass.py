#!/usr/bin/env python3
"""Checks that two builds compiled every batch encode_kernel instantiation to the same SASS, instruction for
instruction (cuobjdump -sass; addresses and encodings dropped).  The encoder sets added a fourth template
argument, APPEND, to encode_kernel: an old build's <INT_OPT, PACKED, IN> is compared with a new build's
<INT_OPT, PACKED, IN, false>.  Instantiations only one build has (the append mode) are listed, not compared.

    python scripts/compare_encode_sass.py OLD.(o|so) NEW.(o|so)     # exit code 1 on any difference
"""
import re
import subprocess
import sys


def kernels(path):
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            cur = None
            if "encode_kernel" in name:
                cur = re.sub(r"(encode_kernelILb[01]ELb[01]ELi[0-9]+E)Lb0E", r"\1", name)
                out[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?)\s*;", line)
        if m and cur:
            out[cur].append(m.group(1))
    return out


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    bad = 0
    for name in sorted(old):
        if name not in new:
            print("MISSING in new build:", name)
            bad += 1
        elif old[name] != new[name]:
            diff = next(i for i, (a, b) in enumerate(zip(old[name] + [""], new[name] + [""])) if a != b)
            print("DIFFERENT: %s (%d vs %d instructions, first difference at %d)" %
                  (name, len(old[name]), len(new[name]), diff))
            bad += 1
        else:
            print("identical: %s (%d instructions)" % (name, len(old[name])))
    for name in sorted(set(new) - set(old)):
        print("new only:  %s (%d instructions)" % (name, len(new[name])))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
