"""build.py refuses a library in which ptxas serialised the wgmma instructions of a kernel."""
import os
import stat
import sys

import pytest

from frame_interpolation_b200 import build

REMARK = ("ptxas info    : (C7520) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
          "program dependence on compiler-inserted WG.AR in divergent path in the function 'k'")


def test_build_fails_on_serialized_wgmma(tmp_path, monkeypatch):
    # a stand-in nvcc that compiles nothing and prints the ptxas remark; the build writes under tmp_path only
    nvcc = tmp_path / "nvcc"
    nvcc.write_text(f"#!{sys.executable}\nprint({REMARK!r})\n")
    nvcc.chmod(nvcc.stat().st_mode | stat.S_IXUSR)
    monkeypatch.setenv("NVCC", str(nvcc))
    monkeypatch.setattr(build, "HERE", str(tmp_path))
    monkeypatch.setattr(build, "LIB", str(tmp_path / "libfilm_b200.so"))
    monkeypatch.setattr(build, "STAMP", str(tmp_path / "_build" / "stamp"))
    with pytest.raises(RuntimeError, match="serialised wgmma") as e:
        build.build(force=True)
    assert REMARK in str(e.value)
    assert not os.path.exists(build.STAMP)
