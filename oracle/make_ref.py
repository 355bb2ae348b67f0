#!/usr/bin/env python
"""Install the UNMODIFIED reference (OpenRL) into oracle/_ref (git-ignored; bench.py's reference arm
imports it from there).

The reference source is taken from $OPENRL_REFERENCE_SRC, else from a checkout named `reference` next
to this repository; without either, nothing is installed and the reference arm is skipped.

TEST / BENCH INFRASTRUCTURE.  The reference is pure Python (`setup.py` installs `find_packages()`
and no package data), so the install is what pip would lay down for it: the `openrl` package tree,
byte for byte, plus a minimal `.dist-info` with its name and version.  No pip is needed.  Its
third-party imports (gymnasium / treevalue / jsonargparse / ...) are not installed: the stand-ins
under oracle/refstubs replace them at run time (oracle/run_reference.py).  No reference source file
is copied into the tracked tree.
"""
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_SRC = os.environ.get("OPENRL_REFERENCE_SRC", os.path.join(os.path.dirname(ROOT), "reference"))
TARGET = os.path.join(HERE, "_ref")


def installed():
    return os.path.isfile(os.path.join(TARGET, "openrl", "__init__.py"))


def source_present():
    return os.path.isfile(os.path.join(REF_SRC, "openrl", "__init__.py"))


def _version(pkg_dir):
    with open(os.path.join(pkg_dir, "__init__.py")) as f:
        m = re.search(r'__VERSION__\s*=\s*"v?([^"]+)"', f.read())
    return m.group(1) if m else "0"


def main(force=False):
    """True when oracle/_ref holds the reference afterwards.  Raises when the source is present but the
    install fails, so that a build never silently loses the reference arm."""
    if installed() and not force:
        print("oracle/_ref already holds the reference install")
        return True
    if not source_present():
        print("no reference source here: using the prebuilt oracle/_ref" if installed() else "reference source absent")
        return installed()
    src = os.path.join(REF_SRC, "openrl")
    tmp = tempfile.mkdtemp(prefix="_ref_", dir=HERE)   # assembled beside the target, then moved into place
    try:
        shutil.copytree(src, os.path.join(tmp, "openrl"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        version = _version(src)
        info = os.path.join(tmp, f"openrl-{version}.dist-info")
        os.makedirs(info)
        with open(os.path.join(info, "METADATA"), "w") as f:
            f.write(f"Metadata-Version: 2.1\nName: openrl\nVersion: {version}\n")
        if os.path.isdir(TARGET):
            shutil.rmtree(TARGET)
        os.replace(tmp, TARGET)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if not installed():
        raise RuntimeError(f"installing the reference from {REF_SRC} into {TARGET} failed")
    print("installed the reference into", TARGET)
    return True


if __name__ == "__main__":
    sys.exit(0 if main(force="--force" in sys.argv) else 1)
