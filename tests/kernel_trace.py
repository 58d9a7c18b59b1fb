"""The kernels the library launched, read from its DFGPU_TRACE output: under DFGPU_TRACE it names every kernel it launches
on stderr as `[dfgpu trace] launch <name>`, template arguments included."""
import os
import re
import sys
import tempfile

LAUNCH = re.compile(r"\[dfgpu trace\] launch (k_\w+(?:<[^>]*>)?)")


def canon(name):
    """`k_hash_agg<8, false, true>` -> `k_hash_agg<8,0,1>`."""
    return re.sub(r"\s", "", name).replace("true", "1").replace("false", "0")


def traced(fn):
    """(fn(), names of the kernels launched while it ran, in launch order).  File descriptor 2 goes to a temporary file
    meanwhile."""
    sys.stderr.flush()
    saved = os.dup(2)
    old = os.environ.get("DFGPU_TRACE")
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        os.environ["DFGPU_TRACE"] = "1"
        try:
            out = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            if old is None:
                del os.environ["DFGPU_TRACE"]
            else:
                os.environ["DFGPU_TRACE"] = old
        f.seek(0)
        text = f.read().decode(errors="replace")
    return out, LAUNCH.findall(text)


def traced_set(fn):
    """(fn(), set of canonical names of the kernels launched while it ran)."""
    out, names = traced(fn)
    return out, {canon(n) for n in names}


def capfd_launched(monkeypatch, capfd):
    """For a pytest fixture: sets DFGPU_TRACE and returns a function that yields the set of canonical names of the
    kernels launched since its last call, read from pytest's captured stderr."""
    monkeypatch.setenv("DFGPU_TRACE", "1")
    capfd.readouterr()
    return lambda: {canon(n) for n in LAUNCH.findall(capfd.readouterr().err)}
