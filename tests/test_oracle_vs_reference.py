"""Pin the oracle on the reference: the golden vectors under tests/golden/ are the reference's own outputs
(tests/golden/make_golden.py runs it), and the port must reproduce them bit for bit."""
import numpy as np
import pytest

from tests.golden import cases as G
from tests import util


@pytest.mark.parametrize("name", ["sins_b2_f24_h128", "sins_b1_f7_h33", "sins_b1_f12_h40_m65_initphase",
                                  "combsub_b2_f24", "superfast_b2_f24", "superfast_b1_f2_constpad",
                                  "sinegen_b2_f12", "csfast_b2_f24", "csfast_b1_f9_initphase", "srcmod_b2_f10"])
def test_port_bit_identical_to_live_reference(name):
    inp = G.build_inputs(name)
    ref = util.load_golden(name)
    util.check_inputs_match_golden(name, inp, ref)
    out = util.port_outputs(name, inp)
    for key in inp["case"]["store"]:
        got = out[key].numpy()
        assert np.array_equal(got, ref[key]), (name, key, np.abs(got - ref[key]).max())
