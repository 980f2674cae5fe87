"""
Runs a scripts/sptk/*.py command line in a fresh interpreter, the way the tests drive every script.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_script(name, argv, library=None, cwd=ROOT, seed=None):
    """
    scripts/sptk/<name> with argv.  `library` binds that shared object in the child; when it is the
    CPU execution model, setk_b200.libs.utils' default device becomes the CPU.  `seed` seeds Python's
    random.  Returns the completed process (stdout and stderr as text); a non-zero exit fails with
    the end of stderr.
    """
    code = ["import random, runpy, sys", "sys.argv = sys.argv[1:]"]
    if library:
        code += ["from setk_b200 import _lib",
                 f"_lib.use_library({os.fspath(library)!r})",
                 "if _lib.emulated(): from setk_b200.libs import utils; utils.set_default_device('cpu')"]
    if seed is not None:
        code.append(f"random.seed({seed!r})")
    code.append("runpy.run_path(sys.argv[0], run_name='__main__')")
    script = os.path.join(ROOT, "scripts", "sptk", name)
    r = subprocess.run([sys.executable, "-c", "\n".join(code), script, *argv], cwd=cwd,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True)
    assert r.returncode == 0, f"{name} exited with {r.returncode}:\n{r.stderr[-3000:]}"
    return r
