"""The set-up the test modules share: seeded models, the synthetic datasets, device uploads, bit-exact comparisons and
the harness of the brute-force case modules (parametrize ids, declared claims, launch constants read from csrc/)."""
import functools
import os
import re

import numpy as np
import scipy.sparse as ssp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "igmc_b200", "csrc")


# ---- models and datasets ----------------------------------------------------------------------------------------------
def model(R, *, h=1, rgcn="pyg-1.4", dgcnn=False, nb=4, seed=0, adj_dropout=None, cuda=True, in0=None, layers=4,
          pyg2_bias=False):
    """the suite's IGMC (``layers`` x 32) or DGCNN_RS ([32, 32, 32, 1], k = 30) regression model on R relations with
    ``nb`` bases and in0 = 2h + 2 input features, its parameters drawn after torch.manual_seed(seed) (seed None: from
    the current torch RNG state).  adj_dropout None keeps the constructor's default.  With ``pyg2_bias`` a pyg-2
    model's conv biases are redrawn from U(-0.3, 0.3), so the bias path is not all zeros."""
    from igmc_b200.models import DGCNN_RS, IGMC
    if seed is not None:
        torch.manual_seed(seed)
    in0 = 2 * h + 2 if in0 is None else in0
    kw = dict(num_relations=R, num_bases=nb, regression=True, rgcn=rgcn)
    if adj_dropout is not None:
        kw["adj_dropout"] = adj_dropout
    if dgcnn:
        m = DGCNN_RS(in0, latent_dim=[32, 32, 32, 1], k=30, **kw)
    else:
        m = IGMC(in0, latent_dim=[32] * layers, **kw)
    if pyg2_bias and rgcn == "pyg-2":
        with torch.no_grad():
            for c in m.convs:
                c.bias.uniform_(-0.3, 0.3)
    return m.cuda() if cuda else m


def checkpoints(m, K, d):
    """K checkpoint files under d: m's parameters plus seeded noise (seeds 100 + k); m itself is left unchanged"""
    paths = []
    own = {k: v.clone() for k, v in m.state_dict().items()}
    for k in range(K):
        torch.manual_seed(100 + k)
        with torch.no_grad():
            m.flat_params.add_(torch.randn_like(m.flat_params) * 0.05)
        paths.append(os.path.join(d, "ck%d.pt" % k))
        torch.save(m.state_dict(), paths[-1])
    m.load_state_dict(own)
    return paths


@functools.lru_cache(maxsize=None)
def dataset(name):
    """make_synthetic_dataset(name, seed=0); "r13" is a 400 x 300 matrix of 13 rating levels, more relations than
    the relation-space plans take (plan 0)"""
    from igmc_b200.data import build_adj, make_synthetic_dataset, synth_ratings
    if name == "r13":
        nu, ni = 400, 300
        u, v, lab = synth_ratings(nu, ni, 9000, 13, seed=4)
        return dict(adj_train=build_adj(u, v, lab, nu, ni), num_relations=13, num_users=nu, num_items=ni)
    return make_synthetic_dataset(name, seed=0)


def adj(name):
    """the training rating matrix of dataset(name)"""
    return dataset(name)["adj_train"]


def random_csr(nu, ni, density, seed, full_rows=(), empty_rows=(), empty_cols=(), single_cols=()):
    """a random nu x ni rating matrix (values 1..5, sorted indices) with each cell rated at ``density``: the rows in
    ``full_rows`` rate every item, ``empty_rows`` and ``empty_cols`` nothing, and each item of ``single_cols`` has
    exactly one rater"""
    rng = np.random.default_rng(seed)
    dense = rng.random((nu, ni)) < density
    dense[list(full_rows)] = True
    dense[list(empty_rows)] = False
    dense[:, list(empty_cols)] = False
    for v in single_cols:
        dense[:, v] = False
        dense[int(rng.integers(nu)), v] = True
    A = ssp.csr_matrix(np.where(dense, rng.integers(1, 6, (nu, ni)), 0).astype(np.float32))
    A.sort_indices()
    return A


def rows_csr(rows):
    """int32 (row_ptr, col) of a list of item rows, each kept in its given order"""
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.concatenate([np.asarray(r, np.int64) for r in rows] + [np.zeros(0, np.int64)]).astype(np.int32)
    return rp, ci


# ---- device arrays and comparisons ------------------------------------------------------------------------------------
def dev(a, dtype=torch.int32):
    """a host array as a CUDA tensor of torch ``dtype``, cast by torch"""
    return torch.as_tensor(np.asarray(a)).to(dtype).cuda()


def dev_np(a, dtype=None):
    """a host array, cast by numpy to numpy ``dtype`` if one is given, as a contiguous CUDA tensor"""
    a = np.asarray(a)
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).cuda()


def nonempty(a):
    """a host array, or one zero of its dtype when it is empty: a kernel argument that must be a valid pointer"""
    a = np.asarray(a)
    return a if a.size else np.zeros(1, a.dtype)


def filled(n, value, dtype=torch.int32, guard=16):
    """a CUDA buffer of n entries and ``guard`` more, all ``value``: a sentinel the kernel must not write past n"""
    return torch.full((max(int(n), 0) + guard,), value, dtype=dtype, device="cuda")


def csr_struct(row_ptr, col, rating, nu, ni):
    """igmc_csr_t of host row arrays (no columns), an empty graph's arrays as one zero; (struct, the device tensors it
    points into)"""
    from igmc_b200 import _lib
    t = (dev_np(nonempty(row_ptr), np.int32), dev_np(nonempty(col), np.int32), dev_np(nonempty(rating), np.uint8))
    return _lib.CSR(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), None, None, nu, ni), t


def same(a, b):
    """fp32 arrays equal bit for bit, NaN matching any NaN (the device and numpy write different NaN payloads)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    n = np.isnan(a)
    return a.shape == b.shape and np.array_equal(n, np.isnan(b)) and np.array_equal(a[~n].view(np.uint32),
                                                                                   b[~n].view(np.uint32))


# ---- the brute-force case harness -------------------------------------------------------------------------------------
def pid(c):
    """a case's parametrize id among every kernel's cases"""
    return "%s: %s" % (c["kernel"], c["name"])


def name_id(c):
    """a case's parametrize id among one kernel's cases"""
    return c["name"]


def assert_claims(regimes, case, extra=None):
    """the case still reaches the regimes it claims: re-derived by its kernel's entry of ``regimes``, or ``extra``"""
    got = regimes[case["kernel"]](case) if extra is None else extra
    assert case["claims"] <= got, ("the case no longer reaches", case["claims"] - got)


def claims_are_declared(module, cases=None):
    """every case of a case module states its claims as a non-empty set of data: no builder computes them with the
    regime function they are checked against"""
    with open(module.__file__) as f:
        assert not re.search(r"claims\W*\]?\s*=\s*\w*regimes", f.read())
    cases = module.all_cases() if cases is None else cases
    assert all(isinstance(c["claims"], set) and c["claims"] for c in cases)


def launch_constants_match(constants):
    """{(csrc file, name): value}: each name is one constexpr int of its file, written as a number or as an IGMC_*
    #define of include/igmc_b200.h, and equals the value the cases were built for"""
    with open(os.path.join(ROOT, "include", "igmc_b200.h")) as f:
        defines = dict(re.findall(r"#define\s+(IGMC_\w+)\s+(\d+)", f.read()))
    for (src, name), value in constants.items():
        with open(os.path.join(CSRC, src)) as f:
            m = re.findall(r"constexpr\s+int\s+%s\s*=\s*(\w+)\s*;" % name, f.read())
        assert [defines.get(x, x) for x in m] == [str(value)], (src, name, m, value)
