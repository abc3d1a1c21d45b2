"""Stage the UNMODIFIED original tutorial (seba-1511/dist_tuto.pth) into ``oracle/_ref/`` for the reference arm of bench.py.

The original is a handful of flat scripts (no setup.py / pyproject), so staging is a byte-for-byte copy, checked file by file
against the SHA-256 list committed next to this recipe (``REF_SHA256.json``).  ``__graft_entry__.build()`` runs it; the source
is the original project's checkout, ``$DIST_TUTO_REFERENCE`` (default ``/root/reference``).  ``oracle/_ref/`` is git-ignored
and nothing else in the project reads the original: when it is not available the reference arm reports itself unavailable.

    python oracle/stage_reference.py [SRC]
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
SHA_FILE = os.path.join(HERE, "REF_SHA256.json")


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def verify(dst=DST):
    """(ok, why): every file of REF_SHA256.json is present in ``dst`` with the recorded hash."""
    want = json.load(open(SHA_FILE))
    for name, h in sorted(want.items()):
        p = os.path.join(dst, name)
        if not os.path.isfile(p):
            return False, f"{name} missing from {dst} (run build() where the original project is available)"
        if _sha(p) != h:
            return False, f"{name} differs from the original (sha256 mismatch)"
    return True, "ok"


def stage(src=None, dst=DST):
    """Copy the original's files into ``dst`` if they are not there yet; (ok, why)."""
    ok, why = verify(dst)
    if ok:
        return ok, why
    src = src or os.environ.get("DIST_TUTO_REFERENCE", "/root/reference")
    want = json.load(open(SHA_FILE))
    if not all(os.access(os.path.join(src, n), os.R_OK) for n in want):
        return False, f"original project not readable at {src}"
    for name, h in want.items():
        if _sha(os.path.join(src, name)) != h:
            return False, f"{src}/{name} is not the recorded original (sha256 mismatch)"
    tmp = f"{dst}.tmp{os.getpid()}"
    shutil.rmtree(tmp, ignore_errors=True)
    os.makedirs(tmp)
    for name in want:
        shutil.copyfile(os.path.join(src, name), os.path.join(tmp, name))
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return verify(dst)


if __name__ == "__main__":
    ok, why = stage(sys.argv[1] if len(sys.argv) > 1 else None)
    print("reference staging:", "OK" if ok else "not staged:", why)
    sys.exit(0 if ok else 1)
