"""H100-native (sm_90a) retrain hot path of AlexIoannides/bodywork-mlops-demo (stage_1's least-squares fit).

Import name: ``bodywork_mlops_demo_b200`` (a shim package that points here -- the directory name
``bodywork-mlops-demo_b200`` is not a valid Python identifier).

    native      ctypes binding of libb2gram.so (include/b2gram.h)
    Context     one GPU: Gram accumulation, solve, scoring, synthetic rows, NCCL all-reduce
    B200LinearRegression   estimator-protocol mirror of sklearn's LinearRegression as stage_1 uses it
    B200RidgeCV            sklearn's RidgeCV (cv=None): the ridge alpha chosen by exact leave-one-out error
    B200ElasticNet, B200Lasso, enet_path, lasso_path
                           sklearn's ElasticNet / Lasso and their paths: coordinate descent on the fp64 Gram
    B200ElasticNetCV, B200LassoCV, fold_ids
                           sklearn's ElasticNetCV / LassoCV: fold statistics in one pass, every path in one launch
    B200BayesianRidge, B200ARDRegression
                           sklearn's BayesianRidge / ARDRegression: evidence maximisation on the fp64 Gram, anchored by
                           one fp64 residual pass; predict(return_std=True) in one fp64 tensor-core pass
    B200PoissonRegressor, B200GammaRegressor, B200TweedieRegressor
                           sklearn's GLM regressors (solver="newton-cholesky"): each Newton iteration is one pass for the
                           loss, gradient and fp64 tensor-core Hessian and one pass for every line-search step
    B200LogisticRegression sklearn's binary LogisticRegression (solver="newton-cholesky"): the same Newton passes on the
                           half-binomial loss, labels as stored, probabilities and labels in one predict pass
    B200RidgeClassifier    sklearn's RidgeClassifier, 2 to 32 classes: the fp64 Gram, one class-sum pass and one solve
                           with every class as a right-hand side; decisions and labels in one fp64 tensor-core pass
    B200RidgeClassifierCV  sklearn's RidgeClassifierCV (cv=None): the alpha chosen by the exact leave-one-out error of
                           every class target, all alphas in one fp64 pass over the rows
    B200MultinomialLogisticRegression
                           sklearn's LogisticRegression (solver="newton-cholesky") for 2 to 32 classes: multinomial
                           Newton fits with every class-pair Hessian block on the fp64 tensor core (two classes: the
                           binary fit)
    B200LinearSVC          sklearn's LinearSVC (liblinear's primal solver, squared hinge) for 2 to 32 classes: trust-region
                           Newton fits whose Hessian is updated on the fp64 tensor core from the rows that cross the margin
    B200LinearSVR          sklearn's LinearSVR (loss="squared_epsilon_insensitive", primal): the same solver
    B200LinearDiscriminantAnalysis
                           sklearn's LinearDiscriminantAnalysis (svd, lsqr, eigen) for 2 to 32 classes: the class means
                           and one fp64 tensor-core pass for the within-class scatter, the solvers on the host;
                           probabilities and projections in one fp64 decision pass
    B200QuadraticDiscriminantAnalysis
                           sklearn's QuadraticDiscriminantAnalysis (svd, eigen) for 2 to 32 classes: the class means and
                           every class's scatter from one fp64 tensor-core pass over the rows in class order, the
                           solvers on the host; K quadratic forms per row in one fp64 decision pass
    stage_1_train_model    drop-in for mlops_simulation/stage_1_train_model.py
"""
from . import _native as native
from ._native import (BF16, F32, KERNEL_AUTO, KERNEL_NARROW, KERNEL_SIMT, KERNEL_TCGEN05, PRECISION_BF16, PRECISION_SPLIT, Context,
                      DeviceArray, PinnedArray)
from .estimator import (B200ARDRegression, B200BayesianRidge, B200ElasticNet, B200ElasticNetCV, B200GammaRegressor,
                        B200Lasso, B200LassoCV, B200LinearRegression, B200LinearSVC, B200LinearSVR, B200LogisticRegression,
                        B200LinearDiscriminantAnalysis,
                        B200QuadraticDiscriminantAnalysis,
                        B200MultinomialLogisticRegression,
                        B200PoissonRegressor,
                        B200RidgeClassifier, B200RidgeClassifierCV, B200RidgeCV, B200TweedieRegressor, default_context,
                        enet_path, fold_ids, lasso_path)
from . import sharding, tranche_io  # noqa: F401

__all__ = ["native", "Context", "DeviceArray", "PinnedArray", "B200LinearRegression", "B200RidgeCV", "B200ElasticNet",
           "B200Lasso", "B200ElasticNetCV", "B200LassoCV", "B200BayesianRidge", "B200ARDRegression",
           "B200PoissonRegressor", "B200GammaRegressor", "B200TweedieRegressor", "B200LogisticRegression",
           "B200RidgeClassifier", "B200RidgeClassifierCV", "B200MultinomialLogisticRegression", "B200LinearSVC", "B200LinearSVR",
           "B200LinearDiscriminantAnalysis", "B200QuadraticDiscriminantAnalysis", "fold_ids", "enet_path", "lasso_path", "default_context",
           "F32", "BF16", "KERNEL_AUTO", "KERNEL_SIMT", "KERNEL_TCGEN05", "KERNEL_NARROW", "PRECISION_SPLIT", "PRECISION_BF16"]
__version__ = "0.1.0"
