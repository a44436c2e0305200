"""Workspace sizes of the soft-projection backward and of approxmatch, without a GPU.  The expected values were recorded before the
host code that carves these workspaces was restructured and must not drift: callers size their buffers with these numbers."""
import pytest


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


# (b, n, m, k, f) -> snb200_soft_project_backward_workspace_bytes
EXPECTED_SOFTPROJ_BWD = {
    (0, 1024, 64, 8, 0): 0,
    (1, 1, 1, 1, 0): 512,
    (1, 1024, 64, 32, 0): 24832,
    (3, 333, 77, 7, 64): 20480,
    (5, 2048, 64, 32, 64): 124160,
    (32, 1024, 64, 8, 0): 204800,
    (32, 1024, 64, 8, 64): 204800,
    (50, 2048, 205, 32, 0): 3977216,
}

# (b, n, m) -> snb200_approxmatch_workspace_bytes
EXPECTED_APPROXMATCH = {
    (0, 1024, 64): 256,
    (1, 1, 1): 344,
    (1, 333, 77): 18296,
    (3, 7, 5): 1840,
    (32, 1024, 64): 1532160,
    (32, 64, 1024): 1532160,
    (50, 2048, 2048): 9011456,
    (7, 1000, 250): 385256,
}


def test_soft_project_backward_workspace_bytes(lib):
    for shape, want in EXPECTED_SOFTPROJ_BWD.items():
        assert lib.snb200_soft_project_backward_workspace_bytes(*shape) == want, shape


def test_approxmatch_workspace_bytes(lib):
    for shape, want in EXPECTED_APPROXMATCH.items():
        assert lib.snb200_approxmatch_workspace_bytes(*shape) == want, shape
