"""Regenerates tests/golden/js_patch_targets.json from a manatee checkout:

    python tests/golden/make_js_patch_golden.py /path/to/manatee

For each upstream file js/patches/*.patch edits, it records the line count, a short SHA-1 of every
line and the bracket skeleton of every line (no code), the same for the file as patch(1) leaves
it, and how often each seam of tests/test_js_patches.py occurs in the patched file.  The patches
are applied with patch(1) in a scratch copy; the upstream files are only read.
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
import test_js_patches as T  # noqa: E402


def main():
    ref = sys.argv[1]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "lib"))
        for f in T.FILES:
            shutil.copy(os.path.join(ref, f), os.path.join(tmp, f))
            p = os.path.join(ROOT, "js", "patches", os.path.basename(f) + ".patch")
            r = subprocess.run(["patch", "-p1", "--no-backup-if-mismatch", "-i", p], cwd=tmp,
                               stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
            assert r.returncode == 0 and "fuzz" not in r.stdout, r.stdout + r.stderr
            a = open(os.path.join(ref, f)).read()
            b = open(os.path.join(tmp, f)).read()
            al, bl = a.splitlines(True), b.splitlines(True)
            out[f] = {"lines": len(al), "line_sha1": [T.line_key(x) for x in al],
                      "skeleton": T.skeleton(a)[:len(al)],
                      "patched_line_sha1": [T.line_key(x) for x in bl],
                      "patched_counts": {nd: b.count(nd) for nd in T.NEEDLES}}
    with open(os.path.join(HERE, "js_patch_targets.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
