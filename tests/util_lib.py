"""The library module as the test modules take it, and the small calls many of them make on it.

A test module imports one of the two fixtures below; each registers as `m`, one library module per test module:
`gpu_library` for tests that need a device, `host_library` for those that build the library and stay on the host."""
import pytest

import _pkg


@pytest.fixture(scope="module", name="m")
def gpu_library():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


@pytest.fixture(scope="module", name="m")
def host_library():
    mod = _pkg.load()
    mod.build_library()
    mod.load_library()
    return mod


def set_options(ix, **opts):
    for name, value in opts.items():
        ix.set_option(name, value)


def refused(m, fn):
    with pytest.raises(m.Bm25xError) as e:
        fn()
    return e.value.code, str(e.value)
