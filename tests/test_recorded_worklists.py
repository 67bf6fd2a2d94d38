"""Recorded work lists of the committed streams (golden/worklists/) on the oracle and the CUDA path == the reference's MD5s."""
import os

import pytest

import oracle_lib

STREAMS = oracle_lib.recorded_streams()


def check(stream, gpu):
    want = open(stream[:-5] + ".md5").read().splitlines()
    got = oracle_lib.replay_worklists(oracle_lib.recorded_worklists(stream), gpu)
    for k, line in sorted(got.items()):
        assert line == want[k], f"picture {k} of {os.path.basename(stream)}"


def test_fixtures_exist():
    assert len(STREAMS) >= 40


@pytest.mark.parametrize("stream", STREAMS, ids=os.path.basename)
def test_oracle_reproduces_reference_decoder(stream):
    check(stream, gpu=False)


@pytest.mark.gpu
@pytest.mark.parametrize("stream", STREAMS, ids=os.path.basename)
def test_cuda_reproduces_reference_decoder(stream):
    check(stream, gpu=True)
