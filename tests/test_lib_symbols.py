"""libbgs.so resolves every C++ symbol of its own: a kernel launcher whose definition drifted from the declaration
its callers use (csrc/launch.cuh) would leave an undefined bgs:: symbol, found only when the library is loaded."""
import shutil
import subprocess

import pytest

from bevy_gaussian_splatting_b200 import abi


def test_no_undefined_symbols_in_namespace_bgs():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm (binutils) is not installed")
    out = subprocess.run([nm, "-D", "--undefined-only", "--demangle", abi.LIB_PATH], check=True,
                         capture_output=True, text=True).stdout
    assert out.strip(), "nm listed no undefined symbols at all (libcudart / libc imports are expected)"
    undefined = [line for line in out.splitlines() if "bgs::" in line]
    assert not undefined, "libbgs.so leaves bgs:: symbols undefined:\n" + "\n".join(undefined)
