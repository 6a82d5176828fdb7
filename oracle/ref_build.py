"""Stage the unmodified reference ``sbi`` package under ``oracle/_ref/`` (git-ignored).

TEST INFRASTRUCTURE.  ``oracle.ref_shim`` imports the reference from there, so the copy goes
wherever the built tree goes.  Source: ``$SBI_REFERENCE_SRC``, else ``/root/reference`` (a checkout
of sbi-dev/sbi).  The copy is refreshed whenever the source's files differ from the recorded stamp.
"""
import hashlib
import os
import shutil

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(_REPO, "oracle", "_ref")
STAMP = os.path.join(DEST, "source.sha256")


def _fingerprint(pkg):
    h = hashlib.sha256()
    for root, dirs, files in os.walk(pkg):
        dirs[:] = sorted(d for d in dirs if d != "__pycache__")
        for f in sorted(files):
            if f.endswith(".pyc"):
                continue
            p = os.path.join(root, f)
            h.update(os.path.relpath(p, pkg).encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    return h.hexdigest()


def stage():
    """Copy the reference package to oracle/_ref/sbi unless an identical copy is there; returns the
    destination, or None (with a message) when no reference source exists."""
    src = os.environ.get("SBI_REFERENCE_SRC") or "/root/reference"
    pkg = os.path.join(src, "sbi")
    if not os.path.isdir(pkg):
        have = os.path.isdir(os.path.join(DEST, "sbi"))
        print(f"no reference source at {src}: " + ("keeping the staged copy in oracle/_ref" if have else
              "the reference-comparison tests will skip"))
        return DEST if have else None
    fp = _fingerprint(pkg)
    if os.path.isfile(STAMP) and open(STAMP).read().strip() == fp:
        return DEST
    tmp = DEST + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(pkg, os.path.join(tmp, "sbi"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    with open(os.path.join(tmp, "source.sha256"), "w") as fh:
        fh.write(fp)
    shutil.rmtree(DEST, ignore_errors=True)
    os.replace(tmp, DEST)
    print("staged the reference package in", DEST)
    return DEST
