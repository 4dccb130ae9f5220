"""The oracle chain that test_gpu_bench_workload.py holds the GPU to, pinned to the reference on bench.py's own records: step 0
of the headline workload (main_ra_4k, 3840x2160: 3 P, 28 B and the I picture at index 24) decoded by the oracle and by the
reference's own reconstruction functions (oracle/_ref/libref_replay.so, SIMD table) must agree on every picture.  Without
oracle/_ref the oracle must reproduce the stored digests of what the replay returned (tests/golden/ref_pins.json).

The records themselves are pinned too, so that a change of the workload (synth, bench.build_workload) fails as such, apart
from a change of what the oracle computes."""
import json
import os

import numpy as np
import pytest

import bench_workloads as bw
import oracle_lib
import ref_pins
from test_cpu_ref_replay import same

HAVE_REF = oracle_lib.ref_replay_lib() is not None
pins = ref_pins.make_fixture(HAVE_REF)
RECORDS_KEY = "test_cpu_bench_workload_oracle::test_headline_records_are_the_pinned_workload"


@pytest.fixture(scope="module")
def headline():
    return bw.build("main_ra_4k")


def records_pin(seq):
    """The records of one step as a ref_pins digest (one record digest per picture)."""
    p = ref_pins.Pins(RECORDS_KEY, HAVE_REF)
    for pic in seq:
        d = np.frombuffer(bytes.fromhex(bw.records_digest([pic])), np.uint8)
        p.check(d, d)
    return p


def test_headline_records_are_the_pinned_workload(headline):
    p = records_pin(headline.seq[:bw.PER_STEP])
    try:
        p.finish()
    except AssertionError as e:
        raise AssertionError(f"the bench workload changed (synth.make_picture or bench.build_workload): {e}") from None


def test_headline_step0_oracle_matches_reference(pins, headline):
    want = json.load(open(ref_pins.PINS_FILE)).get(RECORDS_KEY)
    got = records_pin(headline.seq[:bw.PER_STEP]).md.hexdigest() + f":{bw.PER_STEP}"
    if got != want and not os.environ.get("REF_PINS_RECORD"):
        pytest.fail("the bench workload changed (synth.make_picture or bench.build_workload): the stored picture digests are of other records")
    kinds = [bw.describe(headline, 1, n).split("(")[1].split(",")[1].strip() for n in range(bw.PER_STEP)]
    assert kinds.count("I") == 1 and kinds[24] == "I" and kinds.count("P") == 3, kinds
    orc, ref = oracle_lib.Oracle(), oracle_lib.RefReplay(simd=True) if HAVE_REF else None
    for e in (orc, ref):
        if e is not None:
            e.upload_slot(headline.key_slot, headline.seq[0].params, headline.ref0)
    for n, (_, _, j) in enumerate(bw.schedule(headline, 1)):
        p = headline.seq[j]
        orc.reconstruct(p)
        if ref is not None:
            ref.reconstruct(p)
        same(pins, ref and ref.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), bw.describe(headline, 1, n))
    orc.close()
    if ref is not None:
        ref.close()
