"""GPU drop-in for the reference's ``mlops_simulation/stage_1_train_model.py``.

Same stage contract (bodywork.yaml:8-26): run with no arguments, log to stdout, exit 0 / 1;
same function names and return shapes as the reference module:

==========================  ======================================  ================================
here                        reference (stage_1_train_model.py)      what changed
==========================  ======================================  ================================
``main``                    :31-36                                  unchanged sequence
``download_latest_dataset`` :39-76                                  a local directory stands in for the
                                                                    S3 bucket (same keys, same date regex)
``model_metrics``           :79-90                                  reductions on the GPU (b2_score)
``train_model``             :93-108                                 split -> row mask; fit / predict /
                                                                    metrics on the GPU (libb2gram.so)
``persist_model``           :111-125                                same joblib file of a real sklearn
                                                                    LinearRegression; copied under models/
``persist_metrics``         :128-142                                same CSV schema; copied under
                                                                    model-metrics/
``configure_logger``        :145-158                                same format string
==========================  ======================================  ================================

The "bucket" is the directory named by ``$B2_BUCKET_DIR`` (default ``./bodywork-mlops-project``)
holding ``datasets/regression-dataset-YYYY-MM-DD.csv`` (columns ``date,y,X`` as written by
stage_3_synthetic_data_generation.py:42,49-50; several features generalise to ``X0..X{D-1}``).
"""
from __future__ import annotations

import logging
import os
import re
import shutil
import sys
from datetime import date, datetime
from typing import List, Tuple

import numpy as np
import pandas as pd
from joblib import dump

from . import _native as native
from .estimator import B200LinearRegression, default_context

BUCKET_DIR = os.environ.get("B2_BUCKET_DIR", "bodywork-mlops-project")
_DATE_RE = re.compile("20[2-9][0-9]-[0-1][0-9]-[0-3][0-9]")  # stage_1_train_model.py:47

log = logging.getLogger(__name__)


def main() -> None:
    """Main script to be executed (stage_1_train_model.py:31-36)."""
    data, data_date = download_latest_dataset(BUCKET_DIR)
    try:
        model, metrics = train_model(data)
    finally:
        if isinstance(data, TrancheRows):
            data.free()
    persist_model(model, data_date, BUCKET_DIR)
    persist_metrics(metrics, data_date, BUCKET_DIR)


def _date_from_key(key: str) -> date:
    return datetime.strptime(_DATE_RE.findall(key)[0], "%Y-%m-%d").date()


class TrancheRows:
    """The accumulated rows of binary (.b2t) tranches in pinned host memory -- what ``download_latest_dataset``
    returns instead of a DataFrame when every tranche is binary: the bytes go file -> pinned buffer -> HBM, no pandas
    object is materialised (SURVEY.md 8f rank 1).  ``train_model`` accepts it in place of the DataFrame."""

    def __init__(self, X: np.ndarray, y: np.ndarray, keep=None):
        self.X, self.y, self._keep = X, y, keep

    def __len__(self) -> int:
        return int(self.X.shape[0])

    def free(self) -> None:
        if self._keep is not None:
            for p in self._keep:
                p.free()
            self._keep = None
        self.X = self.y = None


def download_latest_dataset(bucket_dir: str):
    """All tranches under ``<bucket_dir>/datasets`` concatenated oldest -> newest, and the newest date
    (stage_1_train_model.py:39-76).  CSV tranches (the reference's format) give a DataFrame; a bucket of binary
    ``.b2t`` tranches gives ``TrancheRows`` read straight into pinned memory."""
    folder = os.path.join(bucket_dir, "datasets")
    log.info(f"loading all available training data from {folder}")
    try:
        keys = [k for k in sorted(os.listdir(folder)) if _DATE_RE.search(k) and k.endswith((".csv", ".b2t"))]
        if not keys:
            raise FileNotFoundError("no regression-dataset-* tranche found")
        dated = sorted(((k, _date_from_key(k)) for k in keys), key=lambda e: e[1])
        if all(k.endswith(".b2t") for k, _ in dated):
            from . import tranche_io
            X, y, newest, keep = tranche_io.load_all(folder, default_context())
            return TrancheRows(X, y, keep), newest
        dataset = pd.concat(_read_tranche_frame(os.path.join(folder, k)) for k, _ in dated)
    except OSError as e:
        log.error(e)
        raise RuntimeError(f"failed to load training data from {folder}")
    return dataset, dated[-1][1]


def _read_tranche_frame(path: str) -> pd.DataFrame:
    """A tranche as a DataFrame: the reference's CSV, or the binary row-major format of tranche_io."""
    if path.endswith(".csv"):
        return pd.read_csv(path)
    from . import tranche_io
    X, y, kind, day = tranche_io.read_tranche(path)
    if kind != "f32":
        X = native.from_bf16_bits(X)
    cols = {"date": str(day), "y": y}
    cols.update({("X" if X.shape[1] == 1 else f"X{j}"): X[:, j] for j in range(X.shape[1])})
    return pd.DataFrame(cols)


def feature_columns(data: pd.DataFrame) -> List[str]:
    """``['X']`` (the reference's schema) or ``['X0', 'X1', ...]``."""
    if "X" in data.columns:
        return ["X"]
    cols = [c for c in data.columns if re.fullmatch(r"X\d+", str(c))]
    if not cols:
        raise RuntimeError("dataset has no feature column 'X' or 'X0..'")
    return sorted(cols, key=lambda c: int(c[1:]))


def split_mask(n: int, test_size: float = 0.2, seed: int = 42) -> np.ndarray:
    """uint8 per row: 1 = train, 0 = test -- the membership
    ``train_test_split(X, y, test_size=0.2, random_state=42)`` (stage_1_train_model.py:98-103) draws:
    ``perm = RandomState(seed).permutation(n)``; test = the first ceil(test_size * n) entries, train = the rest.

    The permutation is MT19937 + a Fisher-Yates shuffle: sequential by construction, O(n) host work whatever the GPU
    does (the reference does it on the host too).  It stays bit-exact; ``b2_split_mask`` (csrc/split_host.cu) restates
    numpy's legacy generator and shuffle with the swap partners drawn ahead and prefetched (~10x numpy at 10^8 rows),
    the mask of an (n, test_size, seed) already drawn is re-read from ``$B2_CACHE_DIR`` when that is set, and
    ``split_mask_async`` runs it beside the host-to-device copy of the rows."""
    n_test = int(np.ceil(test_size * n))
    n_train = n - n_test            # sklearn/model_selection/_split.py: the complement when train_size is None
    if n_train < 1 or n_test < 1:
        raise ValueError(f"With n_samples={n}, test_size={test_size}, the resulting train set will be empty.")
    cache = os.environ.get("B2_CACHE_DIR")
    path = os.path.join(cache, f"split-mask-n{n}-t{test_size}-s{seed}.u8") if cache else None
    if path and os.path.exists(path) and os.path.getsize(path) == n:
        return np.fromfile(path, dtype=np.uint8)
    mask = np.empty(n, dtype=np.uint8)
    native._check(native.load().b2_split_mask(n, n_test, int(seed) & 0xFFFFFFFF, mask.ctypes.data), "b2_split_mask")
    if path:
        os.makedirs(cache, exist_ok=True)
        tmp = f"{path}.{os.getpid()}.tmp"
        mask.tofile(tmp)
        os.replace(tmp, path)
    return mask


class split_mask_async:
    """``split_mask(n)`` on a worker thread (numpy releases the GIL inside the shuffle): started before the rows go to
    the device, joined when the mask is needed."""

    def __init__(self, n: int, test_size: float = 0.2, seed: int = 42):
        import threading
        self._out, self._err = None, None

        def work():
            try:
                self._out = split_mask(n, test_size, seed)
            except Exception as exc:  # noqa: BLE001 - re-raised by result()
                self._err = exc
        self._thread = threading.Thread(target=work, daemon=True)
        self._thread.start()

    def result(self) -> np.ndarray:
        self._thread.join()
        if self._err is not None:
            raise self._err
        return self._out


def metrics_from_stats(stats: np.ndarray) -> Tuple[float, float, float]:
    """(MAPE, r_squared, max_residual) from the device reductions (include/b2gram.h, b2_score: entries 0..5)."""
    sum_ape, sse, sy, syy, mx, cnt = (float(v) for v in np.asarray(stats)[:6])
    if cnt < 1:
        raise RuntimeError("no rows were scored")
    mape = sum_ape / cnt
    ss_tot = syy - sy * sy / cnt
    if cnt < 2:
        r2 = float("nan")  # sklearn: "R^2 score is not well-defined with less than two samples"
    elif ss_tot > 0.0:
        r2 = 1.0 - sse / ss_tot
    else:
        r2 = 1.0 if sse == 0.0 else 0.0
    return mape, r2, mx


def _metrics_record(mape: float, r_squared: float, max_residual: float) -> pd.DataFrame:
    return pd.DataFrame({"date": [date.today()], "MAPE": [mape], "r_squared": [r_squared],
                         "max_residual": [max_residual]})


def model_metrics(y_actual, y_predicted) -> pd.DataFrame:
    """Regression metrics record (stage_1_train_model.py:79-90), reduced on the GPU.

    The two vectors go to ``b2_metrics`` in float64 (the reference computes on float64 arrays), so MAPE, r_squared
    and max_residual agree with scikit-learn's to rounding; float32 inputs stay float32."""
    stats = default_context().metrics(y_actual, y_predicted)
    return _metrics_record(*metrics_from_stats(stats))


def train_model(data: pd.DataFrame):
    """Train the regression model and compute hold-out metrics (stage_1_train_model.py:93-108).

    Returns ``(sklearn LinearRegression, one-row metrics DataFrame)`` like the reference.
    Numeric contract: the rows are staged as float32 (what the kernels stream; the reference keeps pandas' float64),
    sums, solve, predictions and metric reductions are float64 -- coefficients agree with the reference's to ~1e-6
    relative, metrics to ~1e-7 (asserted against fixtures produced by the unmodified reference)."""
    columns = None
    if isinstance(data, TrancheRows):
        X, y = data.X, data.y                  # pinned, fp32, straight from the tranche files
        n = X.shape[0]
    else:
        # a DataFrame holds every column as its own strided array: hand the columns to b2_upload_columns (host threads
        # gather + convert into a pinned ring beside the H2D copies) instead of DataFrame.to_numpy's transposing copy
        columns = [data[c].to_numpy() for c in feature_columns(data)]
        if len({c.dtype for c in columns}) != 1 or columns[0].dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
            X = np.ascontiguousarray(np.stack(columns, axis=1), dtype=np.float32)
            columns = None
        y = np.ascontiguousarray(data["y"].to_numpy(dtype=np.float32))
        n = y.shape[0]
    mask_job = split_mask_async(n)             # O(n) host shuffle, beside the copies below

    ctx = default_context()
    Xd = yd = md = None
    try:
        Xd = ctx.upload_columns(columns) if columns is not None else ctx.to_device(X)
        yd = ctx.to_device(y)
        md = ctx.to_device(mask_job.result())
        reg = B200LinearRegression(fit_intercept=True, ctx=ctx)
        reg.fit(Xd, yd, row_mask=md, mask_keep=1)
        _, stats = ctx.score(Xd, reg.coef_, float(reg.intercept_), y=yd, row_mask=md, mask_keep=0,
                             want_yhat=False)
    finally:
        for a in (Xd, yd, md):
            if a is not None:
                a.free()
    return reg.to_sklearn(), _metrics_record(*metrics_from_stats(stats))


def persist_model(model, data_date: date, bucket_dir: str) -> None:
    """joblib-dump the estimator as ``regressor-<date>.joblib`` (stage_1_train_model.py:113-114) and
    place it under ``<bucket_dir>/models/`` (the S3 upload of :117-121)."""
    model_filename = f"regressor-{data_date}.joblib"
    dump(model, model_filename)
    try:
        os.makedirs(os.path.join(bucket_dir, "models"), exist_ok=True)
        shutil.move(model_filename, os.path.join(bucket_dir, "models", model_filename))
        log.info(f"stored {model_filename} under {bucket_dir}/models/")
    except OSError as e:
        log.error(e)
        raise RuntimeError("could not store model - check the bucket directory")


def persist_metrics(metrics: pd.DataFrame, data_date: date, bucket_dir: str) -> None:
    """``regressor-<date>.csv`` with header ``date,MAPE,r_squared,max_residual`` (:130-131)."""
    metrics_filename = f"regressor-{data_date}.csv"
    metrics.to_csv(metrics_filename, header=True, index=False)
    try:
        os.makedirs(os.path.join(bucket_dir, "model-metrics"), exist_ok=True)
        shutil.move(metrics_filename, os.path.join(bucket_dir, "model-metrics", metrics_filename))
        log.info(f"stored {metrics_filename} under {bucket_dir}/model-metrics/")
    except OSError as e:
        log.error(e)
        raise RuntimeError("could not store model metrics - check the bucket directory")


def configure_logger() -> logging.Logger:
    """stdout logger with the reference's record format (stage_1_train_model.py:145-158)."""
    handler = logging.StreamHandler(sys.stdout)
    handler.setFormatter(logging.Formatter(
        "%(asctime)s - %(levelname)s - %(module)s.%(funcName)s - %(message)s"))
    logger = logging.getLogger(__name__)
    logger.addHandler(handler)
    logger.setLevel(logging.INFO)
    return logger


def run() -> int:
    """``__main__`` body: exit status 0 on success, 1 on any failure (stage_1_train_model.py:170-178).
    Sentry is initialised only when SENTRY_DSN is set and sentry_sdk is importable (the reference makes it
    mandatory; the drop-in must also run where no DSN secret is mounted)."""
    dsn = os.environ.get("SENTRY_DSN")
    if dsn:
        try:
            import sentry_sdk
            sentry_sdk.init(dsn, traces_sample_rate=1.0)
            sentry_sdk.set_tag("stage", "stage-1-train-model")
        except ImportError:
            pass
    global log
    log = configure_logger()
    try:
        main()
    except Exception as e:  # noqa: BLE001 - mirror of the reference's catch-all
        log.error(e)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(run())
