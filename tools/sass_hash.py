#!/usr/bin/env python
"""Per-kernel hash of the product library's SASS (instruction text without addresses / encodings):

    python tools/sass_hash.py            # print
    python tools/sass_hash.py --write    # refresh tests/golden/product_sass.json

tests/test_abi.py compares the built libpgemb_b200.so with the recorded hashes: the recorded set is the build whose numbers
are in profiles/ and DESIGN.md section 9 -- a kernel that changes (on purpose or by accident) has to be re-measured, and the
file refreshed together with the numbers."""
import hashlib
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sass_hashes(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    cur, fns = None, {}
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fns[cur] = hashlib.sha1()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if cur and m:
            fns[cur].update((re.sub(r"0x[0-9a-f]{8,}", "ADDR", m.group(1).strip()) + "\n").encode())   # absolute branch targets vary with the load address
    return {k: v.hexdigest() for k, v in fns.items() if k.startswith("_ZN5pgemb")}


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from pg_embedding_b200 import build
    h = sass_hashes(build.build())
    if "--write" in sys.argv:
        json.dump({"_comment": "SASS hashes of the kernels of libpgemb_b200.so that the numbers in DESIGN.md section 9 were measured with "
                               "(tools/sass_hash.py --write)", "nvcc": subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-2],
                   "kernels": h}, open(os.path.join(ROOT, "tests", "golden", "product_sass.json"), "w"), indent=1, sort_keys=True)
    print(json.dumps(h, indent=1, sort_keys=True))
