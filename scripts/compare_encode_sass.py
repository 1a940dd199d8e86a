#!/usr/bin/env python3
"""Checks that two builds compiled every batch encode_kernel and every decode_kernel instantiation to the same SASS,
instruction for instruction (cuobjdump -sass; addresses and encodings dropped).  The encoder sets added a fourth
template argument, APPEND, to encode_kernel: an old build's <INT_OPT, PACKED, IN> is compared with a new build's
<INT_OPT, PACKED, IN, false>.  decode_kernel<INT_OPT, MODE> is compared by name; the source-block loop added a third
argument, BLK, so an old build's <INT_OPT, MODE> is compared with a new build's <INT_OPT, MODE, false>.  The rollup's
rollup_forward_kernel and rollup_fold_kernel are compared too; the annotated rollup made them templates over ANN, so an
old build's untemplated kernel is compared with a new build's <false>.  The element sets' element_add_kernel<CTR> and
element_consume_kernel<CTR> are compared too; the annotated element sets added a second argument, ANN, so an old
build's <CTR> is compared with a new build's <CTR, false>.  The element rollup's element_forward_kernel,
element_fold_kernel and element_commit_kernel are compared too; the annotated element rollup added a second argument,
ANN, to the first two, so an old build's <CTR> is compared with a new build's <CTR, false>.  The Timer element sets'
element_timer_{add,consume,forward,fold}_kernel are compared too; the annotated Timer element sets made them templates
over ANN, so an old build's untemplated kernel is compared with a new build's <false>.  The cross-shard rollup's
forward_write_{count_,}kernel and add_forwarded_{prep_,timer_,}kernel are compared too.  Instantiations only one
build has (the append mode, new decode modes, the annotated element kernels) are listed, not compared.

    python scripts/compare_encode_sass.py OLD.(o|so) NEW.(o|so)     # exit code 1 on any difference

--allow NAME_SUBSTRING (repeatable) reports a difference in matching kernels without failing: the instantiations a
change is meant to alter.
"""
import argparse
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
            elif "decode_kernel" in name:
                cur = re.sub(r"(decode_kernelILb[01]ELi[0-9]+E)Lb0E", r"\1", name)
                out[cur] = []
            elif "element_add_kernel" in name or "element_consume_kernel" in name:
                cur = re.sub(r"(element_(?:add|consume)_kernelILb[01]E)Lb0E", r"\1", name)
                out[cur] = []
            elif "element_timer_" in name:  # (Timer element sets)
                cur = re.sub(r"(element_timer_(?:add|consume|forward|fold)_kernel)ILb0EEEvNS_", r"\1ENS_", name)
                out[cur] = []
            elif re.search(r"element_(forward|fold|commit)_kernel", name):  # (element sets through a rollup)
                cur = re.sub(r"(element_(?:forward|fold)_kernelILb[01]E)Lb0E", r"\1", name)
                out[cur] = []
            elif re.search(r"(forward_write|add_forwarded)", name):  # (element-set rollups across shards, Timer too)
                cur = name
                out[cur] = []
            elif "rollup_forward_kernel" in name or "rollup_fold_kernel" in name:
                cur = re.sub(r"(rollup_(?:forward|fold)_kernel)ILb0EEEvNS_", r"\1ENS_", name)
                out[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur:
            out[cur].append(m.group(1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--allow", action="append", default=[])
    a = ap.parse_args()
    old, new = kernels(a.old), kernels(a.new)
    bad = 0
    for name in sorted(old):
        if name not in new:
            print("MISSING in new build:", name)
            bad += 1
        elif old[name] != new[name]:
            diff = next(i for i, (x, y) in enumerate(zip(old[name] + [""], new[name] + [""])) if x != y)
            allowed = any(s in name for s in a.allow)
            print("DIFFERENT%s: %s (%d vs %d instructions, first difference at %d)" %
                  (" (allowed)" if allowed else "", name, len(old[name]), len(new[name]), diff))
            bad += 0 if allowed else 1
        else:
            print("identical: %s (%d instructions)" % (name, len(old[name])))
    for name in sorted(set(new) - set(old)):
        print("new only:  %s (%d instructions)" % (name, len(new[name])))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
