"""The copies of the drop-in class (include/patchwork/patchworkpp.h) compile as reference code writes them: tests/pwpp_copy_driver.cpp
(copy construction, copy assignment over a used instance, self-assignment, a copy of a never-run instance) built without linking.
tests/test_gpu_state_copy.py runs it against the real engine."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def test_copy_driver_compiles(tmp_path):
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-c", "-I" + os.path.join(REPO, "include"),
                           os.path.join(HERE, "pwpp_copy_driver.cpp"), "-o", str(tmp_path / "pwpp_copy_driver.o")])
