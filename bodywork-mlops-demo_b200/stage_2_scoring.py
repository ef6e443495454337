"""Batch scoring companion of the reference's scoring service (SURVEY.md section 8f rank 3).

``score_data_instance`` (stage_2_serve_model.py:73-80) answers one row per HTTP request --
``model.predict(np.array(features, ndmin=2))`` and returns ``prediction[0]`` -- and the service test
(stage_4_test_model_scoring_service.py:66-98) therefore spends 8 ms per row.  The same ``predict`` contract
on a (B, D) batch is one pass of the fused scoring kernel (b2_score):

* ``score_batch(model, X)``       -> all B predictions (what ``model.predict(X)`` returns)
* ``score_payload(model, json)``  -> the service's response for a JSON payload ``{"X": ...}`` with the same
  ``np.array(features, ndmin=2)`` shape rules (scalar -> (1,1), list of D -> (1,D), list of lists -> (B,D)),
  returning every prediction instead of only the first
* ``service_test(model, X, y)``   -> stage_4's test-metrics record with its own definitions
  (APE = |score/label - 1|, "r_squared" = Pearson correlation, "max_residual" = max APE;
  stage_4_test_model_scoring_service.py:89,101-113), reduced on the device.
"""
from __future__ import annotations

import time
from datetime import date
from typing import Dict, Optional

import numpy as np
import pandas as pd

from . import _native as native
from .estimator import default_context


def _coef_intercept(model):
    coef = np.asarray(model.coef_, dtype=np.float64).ravel()
    return coef, float(np.asarray(model.intercept_).ravel()[0]) if np.ndim(model.intercept_) else float(model.intercept_)


def score_batch(model, X, ctx: Optional[native.Context] = None) -> np.ndarray:
    """``model.predict(X)`` for a fitted (sklearn or B200LinearRegression) linear model on the GPU; X is (B, D) or a DeviceArray."""
    ctx = ctx or default_context()
    coef, b0 = _coef_intercept(model)
    if isinstance(X, native.DeviceArray):
        yhat, _ = ctx.score(X, coef, b0)
        return yhat
    Xh = np.ascontiguousarray(np.array(X, ndmin=2), dtype=np.float32)
    if Xh.shape[1] != coef.size:
        raise ValueError(f"X has {Xh.shape[1]} features, but the model is expecting {coef.size} features as input.")
    yhat, _ = ctx.score(Xh, coef, b0)
    return yhat.astype(np.float64)


def score_payload(model, payload: Dict, ctx: Optional[native.Context] = None) -> Dict:
    """The scoring endpoint's response (stage_2_serve_model.py:76-79) for a whole batch."""
    features = payload["X"]
    pred = score_batch(model, np.array(features, ndmin=2), ctx)
    return {"prediction": float(pred[0]), "predictions": [float(v) for v in pred], "model_info": str(model)}


def test_metrics_from_stats(stats: np.ndarray, results_date: date, mean_response_time: float) -> pd.DataFrame:
    """stage_4's ``compute_test_metrics`` record from the ten device reductions (b2_score)."""
    s = np.asarray(stats, dtype=np.float64)
    n = s[5]
    if n < 1:
        raise RuntimeError("no rows were scored")
    mape = s[0] / n                                # == mean |score/label - 1| whenever no label is exactly 0
    cov = s[8] - s[2] * s[6] / n
    var_y = s[3] - s[2] * s[2] / n
    var_p = s[7] - s[6] * s[6] / n
    corr = cov / np.sqrt(var_y * var_p) if var_y > 0 and var_p > 0 else float("nan")
    return pd.DataFrame({"date": [results_date], "MAPE": [mape], "r_squared": [corr], "max_residual": [s[9]],
                         "mean_response_time": [mean_response_time]})


def service_test(model, X, y, results_date: Optional[date] = None, ctx: Optional[native.Context] = None) -> pd.DataFrame:
    """Score a tranche with ``model`` and compute stage_4's test metrics in one device pass."""
    ctx = ctx or default_context()
    coef, b0 = _coef_intercept(model)
    t0 = time.perf_counter()
    if isinstance(X, native.DeviceArray):
        _, stats = ctx.score(X, coef, b0, y=y, want_yhat=False)
        n = X.shape[0]
    else:
        Xh = np.ascontiguousarray(np.array(X, ndmin=2), dtype=np.float32)
        yh = np.ascontiguousarray(np.asarray(y).ravel(), dtype=np.float32)
        _, stats = ctx.score(Xh, coef, b0, y=yh, want_yhat=False)
        n = Xh.shape[0]
    per_row = (time.perf_counter() - t0) / max(n, 1)
    return test_metrics_from_stats(stats, results_date or date.today(), per_row)


test_metrics_from_stats.__test__ = False  # not a pytest test despite the name
