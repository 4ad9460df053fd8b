"""The NK, ANK and ANK-turbulence matrix-free operators share one set of device vectors: the last set_base owns them.
On one long-lived context, every ownership change among the three operators leaves the other two products refused, the
owner's product equal bit for bit to the same call on a fresh context, and adfb_mffd_last_h on the h of the last NK or ANK
product."""
import numpy as np
import pytest

from adflow_b200._lib import AdflowB200Error
from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_UPDATE_INTERMED

from util import FLOW, TURB, case

pytestmark = pytest.mark.gpu

SET_BASE = {"NK": "adfb_mffd_set_base", "ANK": "adfb_ank_mffd_set_base", "TURB": "adfb_ank_mffd_turb_set_base"}
APPLY = {"NK": "adfb_mffd_apply", "ANK": "adfb_ank_mffd_apply", "TURB": "adfb_ank_mffd_turb_apply"}
H = {"NK": -1.0, "ANK": -1.0, "TURB": 1e-6}   # Walker-Pernice h for NK and ANK; the turbulence product needs h > 0


def _vectors(U):
    """base and direction of each operator: the full state, its five flow variables, its turbulence variable"""
    rng = np.random.default_rng(11)
    cells = U.reshape(-1, 6)
    base = {"NK": U, "ANK": np.ascontiguousarray(cells[:, :5]).reshape(-1), "TURB": np.ascontiguousarray(cells[:, 5])}
    return base, {k: rng.standard_normal(v.size) * np.abs(v).clip(1e-6) for k, v in base.items()}


def _prepare(s, U):
    """the state U, its residual (dtl, p, ...) and the ANK time-step matrix: what every product starts from"""
    s.setStates(U)
    s.residual(FLOW | TURB | RES_UPDATE_INTERMED)
    s.ankTimeStepMat()


def _set_base(s, op, U):
    {"NK": s.mffdSetBase, "ANK": s.ankMffdSetBase, "TURB": s.ankMffdTurbSetBase}[op](U)


def _apply(s, op, a):
    if op == "NK":
        return s.mffdApply(a, H[op])
    if op == "ANK":
        return s.ankMffdApply(a, H[op])
    return s.ankMffdTurbApply(a, H[op])


def test_matrix_free_owner(cuda_lib):
    prm, hb = case(12, 9, 8)
    ank = make_ank_params(cfl=5.0, coupled=False)

    def context():
        s = ADFLOW_B200(prm)
        s.addBlock(hb)
        s.ankSetParams(ank)
        return s

    # each operator's product (and the h it reports) on a fresh context
    ref, ref_h = {}, {}
    s = context()
    try:
        U = s.getStates()
    finally:
        s.close()
    base, a = _vectors(U)
    for op in ("NK", "ANK", "TURB"):
        s = context()
        try:
            _prepare(s, U)
            _set_base(s, op, base[op])
            ref[op] = _apply(s, op, a[op])
            ref_h[op] = s.mffdLastH()
        finally:
            s.close()
    assert ref_h["NK"] > 0 and ref_h["ANK"] > 0 and np.abs(ref["TURB"]).max() > 0

    s = context()
    try:
        last_h = s.mffdLastH()
        # every change of owner: NK -> ANK -> TURB -> NK -> TURB -> ANK -> NK
        for op in ("NK", "ANK", "TURB", "NK", "TURB", "ANK", "NK"):
            _prepare(s, U)
            _set_base(s, op, base[op])
            for other in ("NK", "ANK", "TURB"):
                if other != op:
                    with pytest.raises(AdflowB200Error, match="%s: %s has not been called" % (APPLY[other], SET_BASE[other])):
                        _apply(s, other, a[other])
            for gop in ("NK", "ANK"):
                if gop != op:
                    with pytest.raises(AdflowB200Error, match="adfb_gmres_solve: %s has not been called" % SET_BASE[gop]):
                        s.gmresSolve(base[gop], gop, restart=4, max_its=4)
            assert s.mffdLastH() == last_h   # refused products leave it alone
            y = _apply(s, op, a[op])
            assert np.array_equal(y, ref[op]), op
            if op != "TURB":
                last_h = ref_h[op]
            assert s.mffdLastH() == last_h, op   # the turbulence product leaves the h of the last NK / ANK product

        # the turbulence product refuses h <= 0
        _prepare(s, U)
        _set_base(s, "TURB", base["TURB"])
        for h in (0.0, -1.0):
            with pytest.raises(AdflowB200Error, match="adfb_ank_mffd_turb_apply: h must be positive"):
                s.ankMffdTurbApply(a["TURB"], h)
        # new ANK parameters drop an ANK base only: the turbulence base survives them
        s.ankSetParams(ank)
        assert np.array_equal(_apply(s, "TURB", a["TURB"]), ref["TURB"])
        _prepare(s, U)
        _set_base(s, "ANK", base["ANK"])
        s.ankSetParams(ank)
        s.ankTimeStepMat()
        with pytest.raises(AdflowB200Error, match="adfb_ank_mffd_apply: adfb_ank_mffd_set_base has not been called"):
            _apply(s, "ANK", a["ANK"])
    finally:
        s.close()
