#!/usr/bin/env python
"""TEST / BASELINE INFRASTRUCTURE — stages the UNMODIFIED reference mergeGeno.py under the git-ignored oracle/_ref/ (it
imports nothing from genomics.py), so that tools/merge_timing.py can run it as a subprocess where the reference tree is
absent.  A manifest with its sha256 is written next to it."""
import hashlib
import json
import os
import shutil
import sys

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
SRC = "mergeGeno.py"


def stage(verbose=True):
    src = os.path.join(REF, SRC)
    if not os.path.exists(src):
        return False
    os.makedirs(DST, exist_ok=True)
    shutil.copyfile(src, os.path.join(DST, "mergeGeno.py"))
    with open(os.path.join(DST, "MANIFEST_merge.json"), "wt") as m:
        json.dump(dict(source=src, sha256={"mergeGeno.py": hashlib.sha256(open(src, "rb").read()).hexdigest()}), m, indent=1)
    if verbose:
        print("staged %s under %s" % (SRC, DST))
    return True


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
