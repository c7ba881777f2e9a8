"""Installs the reference (evfro/polara, pure Python) into ``oracle/_ref`` -- TEST INFRASTRUCTURE.

``__graft_entry__.build()`` calls :func:`install`.  The comparison legs that drive the reference itself read that
directory through :mod:`oracle.ref_driver`: the drop-in test grafts the device mixins onto polara's own classes, and
``bench.py --impl reference`` and its ``cpu_baseline`` leg time polara's own code.  ``oracle/_ref`` is git-ignored and
needs nothing at run time but the Python packages the reference imports, so it can be built next to the sources and
shipped with the tree to a GPU machine that has no reference checkout.

The checkout is looked for in ``$POLARA_REFERENCE_ROOT``, in a ``reference`` directory beside this repository, and in
``/root/reference``.  Without one nothing is installed, and those legs skip or say that they ran the oracle port.
The checkout itself is only read, never written.

    python -m oracle.install_ref
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "_ref")
_STAMP = ".source"


def reference_source():
    """The reference checkout to install from, or None."""
    repo = os.path.dirname(HERE)
    for root in (os.environ.get("POLARA_REFERENCE_ROOT", ""), os.path.join(os.path.dirname(repo), "reference"),
                 "/root/reference"):
        if root and os.path.isfile(os.path.join(root, "polara", "__init__.py")):
            return os.path.abspath(root)
    return None


def _newest_mtime(tree):
    newest = 0.0
    for dirpath, _, files in os.walk(tree):
        for f in files:
            if f.endswith(".py"):
                newest = max(newest, os.path.getmtime(os.path.join(dirpath, f)))
    return newest


def install():
    """Copies the ``polara`` package of the reference checkout into ``oracle/_ref`` (what ``pip install --target`` makes
    of a pure-Python package, without building inside the read-only checkout).  Returns the target directory, or None
    when no checkout is available.  A copy that is already up to date is left alone."""
    src = reference_source()
    if src is None:
        return None
    pkg = os.path.join(src, "polara")
    stamp = "%s %r" % (src, _newest_mtime(pkg))
    stamp_path = os.path.join(TARGET, _STAMP)
    if os.path.isfile(stamp_path) and os.path.isdir(os.path.join(TARGET, "polara")):
        with open(stamp_path) as f:
            if f.read() == stamp:
                return TARGET
    tmp = TARGET + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(pkg, os.path.join(tmp, "polara"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    with open(os.path.join(tmp, _STAMP), "w") as f:
        f.write(stamp)
    shutil.rmtree(TARGET, ignore_errors=True)
    os.replace(tmp, TARGET)
    return TARGET


if __name__ == "__main__":
    print(install())
