"""The C++ mirror's submap overload of BatchRegistration::align (registration_batch.hpp) compiles for ICP and GICP and refuses
point-to-plane at compile time, with the reason in the message (its residual n o r is not invariant under the map poses)."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SNIPPET = """
#include <small_gicp_b200/registration_batch.hpp>
using namespace small_gicp_b200;
std::vector<RegistrationResult> f(const std::vector<PointCloud>& maps, const std::vector<PointCloud>& scans) {
  BatchRegistration<%s> reg;
  std::vector<std::vector<std::pair<size_t, Isometry3d>>> submaps(1);
  submaps[0].emplace_back(0, Isometry3d::Identity());
  return reg.align(maps, scans, std::vector<size_t>{0}, submaps, std::vector<Isometry3d>{Isometry3d::Identity()});
}
"""


def _compile(factor):
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "t.cpp")
        with open(src, "w") as f:
            f.write(SNIPPET % factor)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        return subprocess.run([cxx, "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "small_gicp_b200", "host", "include"), src],
                              capture_output=True, text=True)


@pytest.mark.parametrize("factor", ["ICPFactor", "GICPFactor", "RobustFactor<Huber, GICPFactor>"])
def test_submap_overload_compiles(factor):
    r = _compile(factor)
    assert r.returncode == 0, r.stderr[-2000:]


@pytest.mark.parametrize("factor", ["PointToPlaneICPFactor", "RobustFactor<Cauchy, PointToPlaneICPFactor>"])
def test_point_to_plane_is_refused_at_compile_time(factor):
    r = _compile(factor)
    assert r.returncode != 0 and "point-to-plane is not available against submaps" in r.stderr
