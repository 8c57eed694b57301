"""Import the reference's *Python half* in place.  TEST INFRASTRUCTURE ONLY.

Works only where a bytewax v0.21.1 source checkout is present (``$BYTEWAX_SRC``, else
``REFERENCE``).  Used by ``oracle/gen_golden.py`` to produce ``tests/golden/*.json``.
``stage()`` (called by ``build()``) copies the parts of the checkout that
``tests/test_reference_pytests.py`` executes into ``oracle/_ref/`` (out of git), so
that those tests also run on machines without the checkout.

The reference's engine is Rust (``bytewax._bytewax``, src/lib.rs:24-32) and
cannot be built here (no cargo, un-vendored timely; SURVEY.md section 8c).  Its
Python operator logic imports fine once a stub ``bytewax._bytewax`` with the
13 names of ``pysrc/bytewax/_bytewax.pyi`` is registered first.
"""

import os
import shutil
import sys
import types

# the bytewax v0.21.1 checkout: $BYTEWAX_SRC, else where the build environment keeps it
REFERENCE = os.environ.get("BYTEWAX_SRC") or "/root/reference"
REFERENCE_PYSRC = os.path.join(REFERENCE, "pysrc")
STAGED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "bytewax")
STAGED_PARTS = ("pysrc", "pytests", "examples", "docs")


def stage() -> bool:
    """Copy ``STAGED_PARTS`` of the checkout into ``STAGED`` (replacing an earlier copy; files only, writable, no
    ``__pycache__``).  Without a readable checkout nothing changes and the result is False."""
    if not all(os.access(os.path.join(REFERENCE, p), os.R_OK | os.X_OK) for p in STAGED_PARTS):
        return False
    tmp = STAGED + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    for part in STAGED_PARTS:
        src = os.path.join(REFERENCE, part)
        for d, dirs, files in os.walk(src):
            dirs[:] = [x for x in dirs if x != "__pycache__"]
            out = os.path.join(tmp, part, os.path.relpath(d, src))
            os.makedirs(out, exist_ok=True)
            for f in files:
                shutil.copyfile(os.path.join(d, f), os.path.join(out, f))
    shutil.rmtree(STAGED, ignore_errors=True)
    os.replace(tmp, STAGED)
    return True


def available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_PYSRC, "bytewax"))


def load():
    """Return the reference's ``bytewax.operators.windowing`` module."""
    if not available():
        raise RuntimeError("reference tree not present")
    if "bytewax" in sys.modules and not getattr(sys.modules["bytewax"], "__file__", "").startswith(
        REFERENCE_PYSRC
    ):
        raise RuntimeError("a different `bytewax` is already imported")
    if "bytewax._bytewax" not in sys.modules:
        stub = types.ModuleType("bytewax._bytewax")

        class AbortExecution(RuntimeError):
            pass

        class InconsistentPartitionsError(ValueError):
            pass

        class MissingPartitionsError(FileNotFoundError):
            pass

        class NoPartitionsError(FileNotFoundError):
            pass

        class RecoveryConfig:
            def __init__(self, db_dir, backup_interval=None):
                self.db_dir, self.backup_interval = db_dir, backup_interval

        class TracingConfig:
            pass

        class JaegerConfig(TracingConfig):
            pass

        class OtlpTracingConfig(TracingConfig):
            pass

        def _unavailable(*_a, **_k):
            raise RuntimeError("the reference's Rust engine is not built here")

        for name, obj in dict(
            AbortExecution=AbortExecution,
            InconsistentPartitionsError=InconsistentPartitionsError,
            MissingPartitionsError=MissingPartitionsError,
            NoPartitionsError=NoPartitionsError,
            RecoveryConfig=RecoveryConfig,
            TracingConfig=TracingConfig,
            JaegerConfig=JaegerConfig,
            OtlpTracingConfig=OtlpTracingConfig,
            init_db_dir=_unavailable,
            setup_tracing=_unavailable,
            run_main=_unavailable,
            cluster_main=_unavailable,
            cli_main=_unavailable,
        ).items():
            setattr(stub, name, obj)
        sys.modules["bytewax._bytewax"] = stub
    if REFERENCE_PYSRC not in sys.path:
        sys.path.insert(0, REFERENCE_PYSRC)
    import bytewax.operators.windowing as win  # noqa: E402

    return win


def find_stateful_batch(flow):
    """Depth-first search of ``flow.substeps`` for the ``stateful_batch`` core step
    (src/worker.rs:289-293, 447-461)."""
    stack = list(flow.substeps)
    while stack:
        step = stack.pop(0)
        if type(step).__name__ == "stateful_batch":
            return step
        stack = list(getattr(step, "substeps", [])) + stack
    raise LookupError("no stateful_batch step")
