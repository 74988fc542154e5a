"""Stage the UNMODIFIED reference for the CPU arm of bench.py (``--impl reference`` / ``cpu_baseline``).

The reference is Python, so there is nothing to compile: the python files of its ``models/`` and ``util/`` packages are
copied verbatim into ``oracle/_ref/`` (kept out of git), where ``baseline/ref_runner.py`` imports them in a process of
their own. Nothing of the reference enters the repository.
"""
import os
import shutil

DEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def stage(reference):
    """Copy <reference>/{models,util}/**/*.py into oracle/_ref/. Returns whether a staged copy exists afterwards."""
    if reference and os.path.isdir(os.path.join(reference, "models")):
        for pkg in ("models", "util"):
            for d, _, files in os.walk(os.path.join(reference, pkg)):
                for f in files:
                    if f.endswith(".py"):
                        rel = os.path.relpath(os.path.join(d, f), reference)
                        os.makedirs(os.path.dirname(os.path.join(DEST, rel)), exist_ok=True)
                        shutil.copyfile(os.path.join(d, f), os.path.join(DEST, rel))
    return os.path.isfile(os.path.join(DEST, "models", "editline2_model.py"))
