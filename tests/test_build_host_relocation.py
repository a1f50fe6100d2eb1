"""The C++ host build (kuiperllama_b200/kuiper/build_host.py) in a tree that was copied or moved after it was built:
CMake refuses a cache configured at another path, so the build directory must be configured afresh."""
import sys

from conftest import ROOT as REPO

sys.path.insert(0, str(REPO / "kuiperllama_b200" / "kuiper"))
import build_host  # noqa: E402


def write_cache(out, made_in, source):
    out.mkdir(parents=True, exist_ok=True)
    (out / "CMakeCache.txt").write_text(
        "# This is the CMakeCache file.\n"
        f"CMAKE_CACHEFILE_DIR:INTERNAL={made_in}\n"
        "CMAKE_BUILD_TYPE:STRING=Release\n"
        f"CMAKE_HOME_DIRECTORY:INTERNAL={source}\n")


def test_a_cache_made_here_is_kept(tmp_path):
    out = tmp_path / "llama2"
    assert not build_host._made_elsewhere(out)  # nothing configured yet
    write_cache(out, out, build_host.HERE)
    assert not build_host._made_elsewhere(out)


def test_a_cache_made_at_another_path_is_detected(tmp_path):
    out = tmp_path / "now" / "llama2"
    write_cache(out, tmp_path / "before" / "llama2", build_host.HERE)
    assert build_host._made_elsewhere(out)
    write_cache(out, out, tmp_path / "before" / "kuiper")  # the sources moved
    assert build_host._made_elsewhere(out)
    (out / "CMakeCache.txt").write_text("CMAKE_BUILD_TYPE:STRING=Release\n")  # no paths recorded
    assert build_host._made_elsewhere(out)
