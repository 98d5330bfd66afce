"""CPU: every C entry point that takes a dk_ctx refuses a null one, and its error message names that entry point."""
import os

import pytest

from diffusionkit_b200 import _lib

# no ctx argument, or a null ctx is a valid no-op
NO_CTX = {"dk_version", "dk_last_error", "dk_ctx_create", "dk_ctx_destroy", "dk_ctx_launch_count",
          "dk_comm_unique_id", "dk_comm_destroy", "dk_groupnorm_ws_floats", "dk_conv_fused_supported"}


@pytest.mark.parametrize("name", sorted(set(_lib.SIGNATURES) - NO_CTX))
def test_null_ctx_is_refused_by_name(name):
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__

        __graft_entry__.build()
    lib = _lib.load()
    _, argtypes = _lib.SIGNATURES[name]
    rc = getattr(lib, name)(*[t() for t in argtypes])   # null ctx, every other argument zero or null
    msg = lib.dk_last_error().decode()
    assert rc == -1 and msg.startswith(name + ":"), (rc, msg)
