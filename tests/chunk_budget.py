"""The device-path chunk budget of the default renderer, set for one test and put back afterwards.  A test module
that needs it imports the fixture: `from chunk_budget import chunk_budget`."""
import pytest

DEFAULT_CHUNK_BYTES = 32 << 20      # ss_ctx::chunk_bytes in sonicsim_b200/csrc/ss_internal.h


@pytest.fixture
def chunk_budget():
    """`R = chunk_budget(8 << 20)` sets the budget and returns the default renderer; the library default is restored
    afterwards, so that later tests run with the budget users get."""
    from sonicsim_b200 import render
    R = render.default_renderer()

    def set_budget(nbytes):
        R.set_chunk_bytes(nbytes)
        return R
    yield set_budget
    R.set_chunk_bytes(DEFAULT_CHUNK_BYTES)
