"""The per-channel lookup tables of a solid batch (csrc/fold.cuh) must equal sequential premultiplied-over
blending for every input value and channel: seeded random stacks of 1 to 1000 layers, valid and over-range
colours, alpha 0 and 255, empty commands, on the host build of the same header."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_fold_tables_equal_sequential_blending():
    exe = os.path.join(HERE, "_build", "fold_check")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-w", "-o", exe, os.path.join(HERE, "fold_check.cpp")],
                   check=True, cwd=HERE)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout[-2000:]
    assert "bad 0" in out.stdout
