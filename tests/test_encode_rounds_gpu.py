"""The fast encoder's rounds on the H100: the constructed blocks of tests/encround.py (same-hash sharers planted at chosen
iterations of chosen rounds) as one batch through the library, under both forms of the round and at the extremes of
the path-selection options, against the oracle."""
import pytest

import oracle
from tests import encround

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(scope="module")
def catalogue():
    return encround.catalogue()


@pytest.mark.parametrize("variant,probe_max,wide_min", [(2, 8, 24), (1, 8, 24), (2, 0, 0), (2, 1000, 1000),
                                                        (1, 1000, 0)])
def test_constructed_rounds_byte_identical(ctx, catalogue, variant, probe_max, wide_min):
    opts = {"encode_variant": variant, "encode_probe_max": probe_max, "encode_wide_min": wide_min}
    prev = {"encode_variant": ctx.get_option("encode_variant"),            # (the tune options have no getter:
            "encode_probe_max": 8, "encode_wide_min": 24}                   # back to EncTune's defaults)
    for k, v in opts.items():
        ctx.set_option(k, v)
    try:
        blocks = [c.data for c in catalogue]
        res, outs = ctx.encode_blocks(blocks)
    finally:
        for k, v in prev.items():
            ctx.set_option(k, v)
    for c, r, o in zip(catalogue, res, outs):
        assert (r, o) == oracle.encode(c.data), (c.name, opts)
