"""The kernels the multi-GPU slot exchange must not touch keep their SASS: every kernel listed in tests/golden/sass_kernels.json (a
digest per kernel of `cuobjdump -sass` of the build before the exchange carried policy slots) is in the library with the same
instructions.  The only kernels of the library not listed are the pack kernel, which gained the slot stamp and one argument, and
the three slot-filtered intake kernels of the gathered blocks.  Instructions are compared without addresses and encodings, and with
the per-file hash of anonymous namespaces removed from the names."""
import hashlib
import json
import os
import re
import subprocess

import deepterrainrl_b200 as trl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
NEW = {"_ZN10trl_comm_k13k_pack_tuplesEN3trl7BuffersEPhiiixPdPjPiS5_PKi",
       "_ZN9trl_train16k_addg_copy_slotENS_3DevENS_7GBlocksE",
       "_ZN9trl_train17k_addg_order_slotENS_3DevENS_7GBlocksEi",
       "_ZN9trl_train18k_addg_assign_slotENS_3DevENS_7GBlocksEi"}


def sass_digests(lib):
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    ks, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_", "_GLOBAL__N_", m.group(1))
            ks.setdefault(cur, [])
            continue
        if cur and ";" in line and "/*" in line:
            txt = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line.split(";")[0]).strip()
            if txt:
                ks[cur].append(txt)
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in ks.items()}


def test_kernels_keep_their_sass():
    lib = trl.build_library()
    got = sass_digests(lib)
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_kernels.json")))
    changed = sorted(k for k, d in want.items() if got.get(k) != d)
    assert not changed, changed
    assert set(got) - set(want) == NEW, sorted(set(got) - set(want))
