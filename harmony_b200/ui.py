"""``RunHarmony`` — host-side mirror of /root/reference/R/ui.R:91-309 (``RunHarmony.default``).

Only argument preparation lives here (the reference does it in R too); all arithmetic on the
cell matrices happens behind the C ABI (include/harmony_b200.h) in hand-written CUDA.
"""
import math
import os
import sys

import numpy as np

from ._arrays import as_columns, factorise, label_device, resolve_device
from .harmony_option import HarmonyOptions, check_legacy_args, harmony_options
from .utils import harmonize, is_cuda_tensor


def _cells_and_columns(data_mat, meta_data, vars_use, verbose):
    """data_mat, meta_data and vars_use of RunHarmony / MapQuery -> (on_device, data_mat, cols, vars_use, N, Z) with Z
    the [N, d] view of data_mat (R/ui.R:157-189)."""
    on_device = is_cuda_tensor(data_mat)   # stays where it is: setup reads it on its device
    if not on_device:
        data_mat = np.asarray(data_mat)
    if data_mat.ndim != 2:
        raise ValueError("data_mat must be a matrix")
    cols, forced = as_columns(meta_data, data_mat.shape)
    if forced is not None:
        vars_use = forced
    if vars_use is None:
        raise ValueError("must provide variables names (e.g. vars_use='stim')")
    if isinstance(vars_use, str):
        vars_use = [vars_use]
    vars_use = list(vars_use)
    if any(v not in cols for v in vars_use):
        raise ValueError("must provide variables names (e.g. vars_use='stim')")
    N = len(next(iter(cols.values())))
    # R/ui.R:178-189: cells must end up as columns; here the row-major [N, d] view is the same bytes
    if data_mat.shape[0] == N:
        Z = data_mat
    elif data_mat.shape[1] == N:
        if verbose:
            print("Transposing data matrix", file=sys.stderr)
        Z = data_mat.T
    else:
        raise ValueError("number of labels do not correspond to number of samples in data matrix")
    return on_device, data_mat, cols, vars_use, N, Z


def _factorise(cols, vars_use, data_mat, on_device):
    """The used label columns -> (phi_i [N, C], B_vec, level_names, N_b): as.factor levels = sorted unique values
    (R/ui.R:210-221), global level ids in phi_i.  Device label columns are factorised on their device, and phi_i is
    then an int32 CUDA tensor (host columns are copied over)."""
    phi_cols, B_vec, level_names = [], [], []
    offset = 0
    device = label_device(cols, vars_use, data_mat, on_device)
    for v in vars_use:
        # device columns hold integer / bool labels: torch's sorted unique levels are np.unique's (and as.factor's)
        levels, codes = factorise(cols[v], device)
        if is_cuda_tensor(levels):
            levels = levels.cpu().numpy()
        phi_cols.append(codes + offset)
        B_vec.append(len(levels))
        level_names.append(levels)
        offset += len(levels)
    B = offset
    if device is None:
        phi_i = np.ascontiguousarray(np.stack(phi_cols, axis=1))      # [N, C]
        N_b = np.bincount(phi_i.reshape(-1), minlength=B).astype(np.float64)
    else:
        import torch
        phi_i = torch.stack(phi_cols, dim=1).contiguous()             # [N, C] int32 on the embedding's device
        N_b = torch.bincount(phi_i.reshape(-1), minlength=B).cpu().numpy().astype(np.float64)
    return phi_i, B_vec, level_names, N_b


def prepare_inputs(data_mat, meta_data, vars_use=None, theta=None, sigma=0.1, lambda_=None, nclust=None,
                   early_stop=True, options=None, verbose=False):
    """Everything RunHarmony.default computes before ``new(harmony)`` (R/ui.R:133-258).

    Returns a dict with the exact argument list of ``harmony::setup`` (src/harmony.h:25-30), with
    the sparse ``phi`` expressed as its row-index slot: ``phi_i[n, c]`` = row of the c-th non-zero of
    column n (each cell has exactly one level per covariate, so columns hold C non-zeros).

    With a CUDA ``data_mat``, a used metadata column (or the bare vector) may be an integer or bool CUDA tensor on the
    same device: it is factorised there, and ``phi_i`` is then an [N, C] int32 CUDA tensor (host columns are
    factorised as usual and copied over).  ``level_names`` are always host arrays.
    """
    options = harmony_options() if options is None else options
    if not isinstance(options, HarmonyOptions):
        raise TypeError("Error: .options must be created from harmony_options()!")
    epsilon_harmony = options.epsilon_harmony if early_stop else -math.inf
    on_device, data_mat, cols, vars_use, N, Z = _cells_and_columns(data_mat, meta_data, vars_use, verbose)
    if nclust is None:
        nclust = min(int(round(N / 30.0)), 100)
    if theta is None:
        theta = [2.0] * len(vars_use)
    else:
        theta = list(np.atleast_1d(np.asarray(theta, dtype=np.float64)))
        if len(theta) != len(vars_use):
            raise ValueError("Please specify theta for each variable")
    sigma = np.atleast_1d(np.asarray(sigma, dtype=np.float64))
    if len(sigma) == 1 and nclust > 1:
        sigma = np.repeat(sigma, nclust)
    phi_i, B_vec, level_names, N_b = _factorise(cols, vars_use, data_mat, on_device)
    B = sum(B_vec)
    if lambda_ is None:                                               # R/ui.R:224-229
        lambda_vec = None
    else:
        lam = np.atleast_1d(np.asarray(lambda_, dtype=np.float64))
        if not np.all(lam > 0):
            raise ValueError("Provided lambdas must be positive")
        if len(lam) == 1:
            lambda_vec = np.concatenate([[0.0], np.repeat(lam, B)])
        else:
            if len(lam) != len(vars_use):
                raise ValueError(
                    f"You specified a lambda value for each covariate but the number of lambdas specified "
                    f"({len(lam)}) and the number of covariates ({len(vars_use)}) mismatch.")
            lambda_vec = np.concatenate([[0.0], np.repeat(lam, B_vec)])
    theta_vec = np.repeat(np.asarray(theta, dtype=np.float64), B_vec)
    tau = options.tau
    with np.errstate(divide="ignore", invalid="ignore"):              # tau = 0 -> N_b/0 = Inf -> factor 1
        theta_vec = theta_vec * (1 - np.exp(-(N_b / (nclust * tau)) ** 2)) if tau != 0 else theta_vec * 1.0
    if not on_device:
        Z = np.ascontiguousarray(Z, dtype=np.float64)
    return dict(Z=Z, phi_i=phi_i, B_vec=np.asarray(B_vec, dtype=np.int32),
                sigma=sigma, theta=theta_vec, lambda_=lambda_vec, alpha=float(options.alpha),
                max_iter_kmeans=int(options.max_iter_cluster), epsilon_kmeans=float(options.epsilon_cluster),
                epsilon_harmony=float(epsilon_harmony), K=int(nclust), block_size=float(options.block_size),
                batch_proportion_cutoff=float(options.batch_prop_cutoff), level_names=level_names,
                vars_use=vars_use)


def RunHarmony(data_mat, meta_data, vars_use=None, theta=None, sigma=0.1, lambda_=None, nclust=None, max_iter=10,
               early_stop=True, ncores=1, plot_convergence=False, return_object=False, verbose=True,
               options=None, seed=None, device=None, **kwargs):
    """RunHarmony.default (R/ui.R:91-309) on the GPU.

    ``ncores`` (CPU BLAS threads, R/ui.R:101,123-128) is accepted and ignored; ``seed`` replaces R's
    ``set.seed`` for the k-means initialisation and the per-round update orders.  Returns the
    corrected embedding [N, d] (same orientation rule as the reference: the transpose of what
    ``getZcorr()`` holds) or the ``harmony`` object when ``return_object`` is true.

    ``data_mat`` may be a float32 / float64 CUDA tensor (either orientation): the object is created on its device
    and the result is a [N, d] tensor of the same dtype on that device; the embedding never visits the host.
    """
    from .harmony import harmony  # needs the CUDA extension; fails loudly when it is missing

    check_legacy_args(**kwargs)
    a = prepare_inputs(data_mat, meta_data, vars_use, theta, sigma, lambda_, nclust, early_stop, options, verbose)
    if verbose and a["lambda_"] is None:
        print("Using automatic lambda estimation", file=sys.stderr)
    obj = harmony(device=resolve_device(device, data_mat, "data_mat"))
    obj.setup(a["Z"], a["phi_i"], a["sigma"], a["theta"], a["lambda_"], a["alpha"], a["max_iter_kmeans"],
              a["epsilon_kmeans"], a["epsilon_harmony"], a["K"], a["block_size"], a["B_vec"],
              a["batch_proportion_cutoff"], verbose)
    if seed is None:   # R without set.seed(): the session's random stream differs from run to run
        seed = int.from_bytes(os.urandom(8), "little")
    obj.set_seed(seed)
    if verbose:
        print("Initializing state using k-means centroids initialization", file=sys.stderr)
    obj.init_cluster_cpp()
    harmonize(obj, max_iter, verbose)
    if plot_convergence:
        from .utils import HarmonyConvergencePlot
        HarmonyConvergencePlot(obj)
    if return_object:
        return obj
    if is_cuda_tensor(data_mat):
        return obj.get_tensor("Z_corr", dtype=data_mat.dtype)
    return np.ascontiguousarray(obj.getZcorr().T)   # t(harmonyObj$getZcorr()), R/ui.R:292-295: cells x PCs


def MapQuery(data_mat, meta_data, vars_use, reference, lambda_=1.0, return_object=False, verbose=True, device=None):
    """Maps query cells onto a finished integration in one pass, without rerunning Harmony (DESIGN.md §8).

    ``data_mat``: the query's embedding in the reference's PC space (projecting genes onto the PCs is the caller's
    job), [Nq, d] or [d, Nq], a host array or a float32 / float64 CUDA tensor, with ``meta_data`` / ``vars_use`` naming
    the query's own covariates exactly as in RunHarmony (device labels included).  ``reference``: a HarmonyReference
    (``harmony.reference()``, or ``HarmonyReference.load``).  ``lambda_``: ridge penalty of the query's levels, a scalar
    or one value per covariate, each > 0.

    Every query cell is softly assigned to the reference's clusters; then one ridge correction per cluster, whose
    intercept the reference's statistics anchor, removes the query's batch terms.  The reference's cells do not move.
    Returns the mapped embedding [Nq, d] (numpy, or a CUDA tensor of data_mat's dtype on its device) or, with
    ``return_object``, the harmony object (getR() is the query's assignment)."""
    from .mapping import HarmonyReference
    if not isinstance(reference, HarmonyReference):
        raise TypeError("reference must be a HarmonyReference (harmony.reference() or HarmonyReference.load)")
    on_device, data_mat, cols, vars_use, N, Z = _cells_and_columns(data_mat, meta_data, vars_use, verbose)
    if Z.shape[1] != reference.d:
        raise ValueError(f"the query has {Z.shape[1]} dimensions, the reference {reference.d}")
    lam = np.atleast_1d(np.asarray(lambda_, dtype=np.float64))
    if not np.all(np.isfinite(lam) & (lam > 0)):
        raise ValueError("Provided lambdas must be positive")
    if len(lam) not in (1, len(vars_use)):
        raise ValueError(f"lambda_ must be one value or one per covariate ({len(vars_use)}), not {len(lam)}")
    device = resolve_device(device, data_mat, "data_mat")
    phi_i, B_vec, _, _ = _factorise(cols, vars_use, data_mat, on_device)
    lambda_vec = np.repeat(lam, B_vec) if len(lam) > 1 else np.repeat(lam, sum(B_vec))
    from .harmony import harmony  # needs the CUDA extension; fails loudly when it is missing
    obj = harmony(device=device)
    if verbose:
        print(f"Mapping {N} cells onto a {reference.K}-cluster reference", file=sys.stderr)
    obj.map_setup(Z, phi_i, np.asarray(B_vec, dtype=np.int32), lambda_vec, reference)
    obj.map()
    if return_object:
        return obj
    if on_device:
        return obj.get_tensor("Z_corr", dtype=data_mat.dtype)
    return np.ascontiguousarray(obj.getZcorr().T)
