"""TEST INFRASTRUCTURE -- install the UNMODIFIED reference package into oracle/_ref/reference (git-ignored) so that
`bench.py --impl reference` and bench.py's `cpu_baseline` can time the reference's own CPU implementation.

Runs only where the environment variable REFERENCE_SRC names a checkout of facebookresearch/differentiable-robot-model;
elsewhere bench.py falls back to the torch port (oracle/drm_oracle.py) and says so.  The reference's setup.py derives its
version from `git describe`, so the install runs from a temporary copy that is given a throw-away git tag; package
sources are not touched, and dependencies are skipped (--no-deps: the reference's XML parser dependency is replaced by
oracle/refshim)."""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "_ref", "reference")


def install(ref_src=None) -> str:
    ref_src = ref_src or os.environ.get("REFERENCE_SRC", "")
    if os.path.isdir(os.path.join(TARGET, "differentiable_robot_model")):
        return "present"
    if not ref_src or not os.path.isdir(os.path.join(ref_src, "differentiable_robot_model")):
        return f"reference sources not found (REFERENCE_SRC={ref_src!r}): bench.py's reference arm will use the torch port"
    tmp = tempfile.mkdtemp(prefix="drm_ref_")
    try:
        copy = os.path.join(tmp, "reference")
        shutil.copytree(ref_src, copy, symlinks=True)
        git = ["git", "-c", "user.email=build@localhost", "-c", "user.name=build"]
        subprocess.run(["git", "init", "-q", "."], cwd=copy, check=True)
        subprocess.run(["git", "add", "-A"], cwd=copy, check=True, stdout=subprocess.DEVNULL)
        subprocess.run(git + ["commit", "-q", "-m", "snapshot of the reference"], cwd=copy, check=True)
        subprocess.run(["git", "tag", "v0.2.1"], cwd=copy, check=True)
        subprocess.run([sys.executable, "-m", "pip", "install", "-q", "--no-index", "--no-build-isolation", "--no-deps",
                        "--target", TARGET, copy], check=True)
        return "installed"
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    print(install(sys.argv[1] if len(sys.argv) > 1 else None))
