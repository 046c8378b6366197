"""Generate tests/golden/ref_3dmfv_grid_gmm.npz from the REFERENCE's own get_3d_grid_gmm (3DmFV-Net/utils/utils.py:69-92), in the
build container.  The module cannot be imported (it imports sklearn, matplotlib and the rest at the top), so the function is lifted
out of the source file with `ast` and executed with numpy only, under a stand-in for sklearn's GaussianMixture that keeps the
attributes the function assigns (weights_, means_, covariances_) and ignores the precision Cholesky import.  No reference source is
copied into this repo.

    python tests/golden/make_golden_3dmfv.py            # needs /root/reference

Keys: w{r}, mu{r}, cov{r} (float64, as the function leaves them) for subdivisions r in {3, 5, 8}, variance 0.04."""
import ast
import os
import sys
import types

import numpy as np

REF = os.environ.get("PSA_REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _GaussianMixture:
    def __init__(self, n_components=1, covariance_type="full"):
        self.n_components = n_components
        self.covariance_type = covariance_type


def lift(path, name):
    tree = ast.parse(open(path).read())
    ns = {"np": np, "GaussianMixture": _GaussianMixture}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == name:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    assert name in ns, name
    return ns[name]


def main():
    # `from sklearn.mixture.gaussian_mixture import _compute_precision_cholesky` inside the function: a stub module
    gm = types.ModuleType("sklearn.mixture.gaussian_mixture")
    gm._compute_precision_cholesky = lambda cov, kind: None
    for name, mod in (("sklearn", types.ModuleType("sklearn")), ("sklearn.mixture", types.ModuleType("sklearn.mixture")),
                      ("sklearn.mixture.gaussian_mixture", gm)):
        sys.modules.setdefault(name, mod)
    fn = lift(os.path.join(REF, "3DmFV-Net", "utils", "utils.py"), "get_3d_grid_gmm")
    out = {}
    for r in (3, 5, 8):
        gmm = fn(subdivisions=[r, r, r], variance=0.04)
        out[f"w{r}"] = np.asarray(gmm.weights_)
        out[f"mu{r}"] = np.asarray(gmm.means_)
        out[f"cov{r}"] = np.asarray(gmm.covariances_)
    dst = os.path.join(ROOT, "tests", "golden", "ref_3dmfv_grid_gmm.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
