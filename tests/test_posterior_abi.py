"""C ABI argument checks of posterior decoding that need no device: a NULL tokenizer or result is refused with
VBT_ERR_INVALID_ARGUMENT and a message naming it, whatever the other arguments."""
import ctypes as C

import pytest

from vibrato_b200 import _native

INVALID_ARGUMENT = 1


def call(name, *args):
    L = _native.lib()
    rc = getattr(L, name)(*args)
    return rc, L.vbt_last_error().decode()


@pytest.mark.parametrize("on,gamma", [(1, 1.0), (0, 0.0), (1, -1.0), (1, float("nan"))])
def test_set_posterior_null_tokenizer(on, gamma):
    rc, msg = call("vbt_tokenizer_set_posterior", None, on, gamma)
    assert rc == INVALID_ARGUMENT and "t must not be NULL" in msg


def test_result_posterior_null_result():
    p = [C.c_void_p() for _ in range(4)]
    n = C.c_uint64()
    rc, msg = call("vbt_result_posterior", None, *[C.byref(x) for x in p], C.byref(n))
    assert rc == INVALID_ARGUMENT and "r must not be NULL" in msg


def test_last_device_posterior_null_tokenizer():
    v = [C.c_uint64() for _ in range(5)]
    rc, msg = call("vbt_last_device_posterior", None, *[C.byref(x) for x in v])
    assert rc == INVALID_ARGUMENT and "t must not be NULL" in msg


def test_posterior_text_option_null_tokenizer():
    rc, msg = call("vbt_tokenizer_set_option", None, b"posterior_text", 1)
    assert rc == INVALID_ARGUMENT and "t must not be NULL" in msg
