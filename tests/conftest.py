import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


# ---- every -m gpu test runs under BOTH 16-bit operand types (HAIRFAST_DTYPE is read at call time by
# hairfastgan_b200.model.default_dtype / nn16.default_dtype).  Setting HAIRFAST_DTYPE in the environment restricts the
# run to that type; HAIRFAST_TEST_DTYPES=default additionally keeps the un-set default (generator bf16, encoders fp16).
def _gpu_dtypes():
    if os.environ.get("HAIRFAST_TEST_DTYPES"):
        return os.environ["HAIRFAST_TEST_DTYPES"].split(",")
    if os.environ.get("HAIRFAST_DTYPE"):
        return [os.environ["HAIRFAST_DTYPE"]]
    return ["bf16", "fp16"]


def pytest_generate_tests(metafunc):
    if "hf_dtype" in metafunc.fixturenames and metafunc.definition.get_closest_marker("gpu") is not None:
        dtypes = getattr(metafunc.module, "HF_DTYPES", None) or _gpu_dtypes()     # a module may choose its own set
        metafunc.parametrize("hf_dtype", dtypes, indirect=True, scope="module")


@pytest.fixture(scope="module", autouse=True)
def hf_dtype(request):
    want = getattr(request, "param", None)
    if want is None or want == "default":
        yield want
        return
    old = os.environ.get("HAIRFAST_DTYPE")
    os.environ["HAIRFAST_DTYPE"] = want
    try:
        yield want
    finally:
        if old is None:
            os.environ.pop("HAIRFAST_DTYPE", None)
        else:
            os.environ["HAIRFAST_DTYPE"] = old
