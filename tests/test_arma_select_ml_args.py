"""CPU: the argument checks of the selection's ML refit and its Kalman predictor (DESIGN.md section 2 item 21) in
ForecastEngine.fit_select_arma and the frame layer, and the frames forwarding refit="ml" / predictor="kalman" to the
engine (a recorder engine answering with the selection oracle stands in for the GPU)."""
import numpy as np
import pytest

from test_arma_select_css_oracle import _SelectRecorder


class _MlRecorder(_SelectRecorder):
    """_SelectRecorder that also takes predictor= and records it"""

    def fit_select_arma(self, y, n_hold, orders, diffs, mas, ps, npred, refit=None, joint_beta=False, predictor=None,
                        want_se=False):
        res = super().fit_select_arma(y, n_hold, orders, diffs, mas, ps, npred, refit=refit, joint_beta=joint_beta)
        self.calls[-1] = self.calls[-1] + (predictor,)
        if want_se:
            res["se"] = np.ones_like(res["pred"])
        return res


def test_engine_argument_checks():
    import mmf
    eng = mmf.ForecastEngine.__new__(mmf.ForecastEngine)
    for kw, msg in ((dict(refit="mle"), r"refit must be None or 'css' \(or 'ml' for the exact likelihood\), got 'mle'"),
                    (dict(refit="ml", joint_beta=True), "joint_beta=True needs refit='css'"),
                    (dict(refit="ml", predictor="kf"), "predictor must be 'recursion' or 'kalman'"),
                    (dict(refit="css", predictor="kalman"), "predictor='kalman' needs estimator='ml'"),
                    (dict(predictor="kalman"), r"predictor='kalman' needs estimator='ml' \(or refit='ml'"),
                    (dict(max_iter=3), "max_iter= is the pass budget of refit='css'")):
        with pytest.raises(ValueError, match=msg):
            eng.fit_select_arma(None, 8, **kw)


def test_frames_forward_refit_ml_and_the_kalman_predictor():
    import mmf
    from test_arima_oracle import _frame
    pdf = _frame()
    eng = _MlRecorder()
    kw = dict(freq="D", horizon=14, mode="holdout", engine=eng, ar=(0, 1), diff=(0, 1), ma=(0, 1))
    mmf.forecast_groups(pdf, refit="ml", **kw)
    mmf.forecast_groups(pdf, refit="ml", predictor="kalman", **kw)
    mmf.forecast_groups(pdf, refit="ml", predictor="kalman", conf_int=0.9, **kw)
    mmf.forecast_groups(pdf, refit="css", **kw)
    nb = len(eng.calls) // 4
    assert eng.calls == ([("ml", False, None)] * nb + [("ml", False, "kalman")] * 2 * nb
                         + [("css", False, None)] * nb), eng.calls


def test_frame_refusals():
    import mmf
    pdf = mmf.synth.reference_weekly_demand(2)
    for fg in (mmf.frames.forecast_groups, mmf.frames.forecast_table):
        for kw, msg in ((dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), refit="css", predictor="kalman"),
                         "predictor='kalman' needs estimator='ml'"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), predictor="kalman"),
                         "predictor='kalman' needs estimator='ml'"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), refit="ml", predictor="kf"),
                         "predictor must be 'recursion' or 'kalman'"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), refit="ml", joint_beta=True),
                         "joint_beta=True needs estimator='css' or refit='css'"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), refit="mle"),
                         r"refit must be None or 'css' \(or 'ml' for the exact likelihood\)"),
                        (dict(ar=1, ma=1, refit="ml", predictor="kalman"), "refit= needs candidate MA orders"),
                        (dict(ar=1, ma=1, estimator="ml", refit="ml"), "refit= is not offered with estimator="),
                        (dict(ar=(0, 1), ma=(0, 1), refit="ml", select=(1, 3)), "is not offered with select=")):
            with pytest.raises(ValueError, match=msg):
                fg(pdf, freq="W-MON", horizon=40, mode="holdout", engine=object(), **kw)
