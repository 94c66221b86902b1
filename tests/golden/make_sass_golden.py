"""Fingerprints of the machine code of every kernel of every object (tests/test_train_cpu.py checks that the kernels
stay unchanged).  Run on a build of the commit whose kernels the golden should pin:

    make -C luciddreamer_b200/csrc && python tests/golden/make_sass_golden.py luciddreamer_b200/csrc
"""
import glob
import hashlib
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def kernel_fingerprints(obj: str) -> dict:
    """{function name: sha256 of its SASS listing}.  The listing is the function name line and the instructions, with
    the encodings dropped and the anonymous-namespace tags replaced (in the name too): nvcc derives one from the
    source path and one from the file's contents, so neither says anything about the kernel's machine code."""
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    per, fn = {}, None
    for line in out.splitlines():
        if "Function :" in line or re.search(r"/\*[0-9a-f]{4}\*/", line):
            line = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_", "_GLOBAL__N__X_", line)
            line = re.sub(r"(_GLOBAL__N__X_\d+_\w+?_cu)_[0-9a-f]{8}", r"\1_X", line)
            line = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", line).strip()
            if "Function :" in line:
                fn = line.split("Function :", 1)[1].strip()
                per[fn] = []
            per[fn].append(line)
    return {fn: hashlib.sha256("\n".join(lines).encode()).hexdigest() for fn, lines in per.items()}


if __name__ == "__main__":
    objs = sorted(glob.glob(os.path.join(sys.argv[1], "*.o")))
    gold = {os.path.basename(o): kernel_fingerprints(o) for o in objs}
    json.dump(gold, open(os.path.join(HERE, "sass_kernels.json"), "w"), indent=1, sort_keys=True)
    print(f"{len(gold)} objects, {sum(len(k) for k in gold.values())} kernels")
