"""The MMD misspecification test without a GPU: the host's shuffle tables against the UNMODIFIED reference (through
oracle.ref_shim) for the same seed, its error and warning texts, the device envelope check, and the refusal to run
without a CUDA device."""
import warnings

import pytest
import torch
import torch.nn as nn

from oracle import ref_shim
from sbi_b200 import _lib
from sbi_b200 import misspecification as M
from sbi_b200.diagnostics import calc_misspecification_mmd

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    from sbi.diagnostics import misspecification as R
    return R


def _errors_equal(ours, theirs):
    with pytest.raises(Exception) as a:
        ours()
    with pytest.raises(Exception) as b:
        theirs()
    assert type(a.value) is type(b.value) and str(a.value) == str(b.value), (a.value, b.value)


class _Net(nn.Module):
    def __init__(self, emb):
        super().__init__()
        self.embedding_net = emb


class _Trainer:
    def __init__(self, net):
        self._neural_net = net


@needs_ref
@pytest.mark.parametrize("n,n_shuffle,max_samples", [(50, 7, 20), (30, 3, 1000), (10_000, 4, 1000)])
def test_shuffle_table_is_the_references_draws(ref, monkeypatch, n, n_shuffle, max_samples):
    drawn = []
    real = torch.randperm

    def spy(*a, **k):
        out = real(*a, **k)
        drawn.append(out[:max_samples].clone())
        return out
    torch.manual_seed(5)
    monkeypatch.setattr(ref.torch, "randperm", spy)
    monkeypatch.setattr(ref, "compute_rbf_mmd_median_heuristic", lambda x, y, mode="biased": torch.tensor(0.))
    ref.calculate_baseline_mmd(3, torch.randn(n, 2), n_shuffle=n_shuffle, max_samples=max_samples)
    monkeypatch.undo()
    after_ref = torch.randn(3)
    torch.manual_seed(5)
    torch.randn(n, 2)
    table = M.shuffle_table(n, n_shuffle, max_samples)
    assert torch.equal(table, torch.stack(drawn))
    assert torch.equal(torch.randn(3), after_ref)   # the generator is left where the reference leaves it


@needs_ref
def test_errors_match_reference(ref):
    x_obs, x = torch.randn(5, 2), torch.randn(4, 2)
    _errors_equal(lambda: calc_misspecification_mmd(x_obs, x), lambda: ref.calc_misspecification_mmd(x_obs, x))
    _errors_equal(lambda: M.calculate_baseline_mmd(5, x), lambda: ref.calculate_baseline_mmd(5, x))
    x = torch.randn(40, 2)
    for kw in (dict(mode="latent"), dict(mode="embedding"), dict(mode="embedding", inference=_Trainer(None)),
               dict(mode="embedding", inference=object()),
               dict(mode="embedding", inference=_Trainer(_Net(None)))):
        _errors_equal(lambda: calc_misspecification_mmd(x_obs, x, **kw),
                      lambda: ref.calc_misspecification_mmd(x_obs, x, **kw))
    for n_shuffle in (0, 3):
        torch.manual_seed(1)
        _errors_equal(lambda: calc_misspecification_mmd(x_obs, x, n_shuffle=n_shuffle, mmd_mode="median"),
                      lambda: ref.calc_misspecification_mmd(x_obs, x, n_shuffle=n_shuffle, mmd_mode="median"))
    _errors_equal(lambda: M.compute_rbf_mmd(x_obs, x, mode="x"), lambda: ref.compute_rbf_mmd(x_obs, x, mode="x"))
    _errors_equal(lambda: M.calculate_baseline_mmd(3, x, n_shuffle=-1),
                  lambda: ref.calculate_baseline_mmd(3, x, n_shuffle=-1))


@needs_ref
def test_bad_mode_draws_what_the_reference_draws(ref):
    x_obs, x = torch.randn(5, 2), torch.randn(40, 2)
    for impl in (M, ref):
        torch.manual_seed(3)
        with pytest.raises(ValueError):
            impl.calculate_p_misspecification(x_obs, x, n_shuffle=4, mode="x")
        if impl is M:
            ours = torch.randn(4)
        else:
            assert torch.equal(torch.randn(4), ours)


@needs_ref
def test_identity_warning_matches_reference(ref):
    """The warning comes before any device work; the run itself then needs the device (no CPU fallback)."""
    x_obs, x = torch.randn(5, 2), torch.randn(40, 2)
    tr = _Trainer(_Net(nn.Identity()))
    seen = []
    for impl in (M, ref):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            try:
                impl.calc_misspecification_mmd(x_obs, x, inference=tr, mode="embedding", n_shuffle=2)
            except RuntimeError:
                assert impl is M and not torch.cuda.is_available()
        seen.append([(c.category, str(c.message)) for c in w if "embedding net" in str(c.message)])
    assert seen[0] == seen[1] and len(seen[0]) == 1


@pytest.mark.parametrize("n_shuffle,max_samples,n", [(_lib.SBI_MMD_MAX_SETS, 10, 20), (2, 70_000, 70_000)])
def test_oversize_request_raises_before_launch(n_shuffle, max_samples, n):
    x = torch.randn(n, 1)
    if not torch.cuda.is_available():
        pytest.skip("the envelope check runs after the inputs reach the device")
    with pytest.raises(_lib.SbiB200Error, match=r"MMD: \d+ index sets of \d+ rows"):
        M.calculate_p_misspecification(x[:1], x, n_shuffle=n_shuffle, max_samples=max_samples)


def test_envelope_check_names_the_sizes():
    z = torch.zeros(4, 3)
    with pytest.raises(_lib.SbiB200Error, match=r"MMD: 2 index sets of 70000 rows over a \(4, 3\) matrix"):
        M._mmd_sets(z, torch.zeros(2, 70_000, dtype=torch.int32), torch.tensor([[1, 3], [1, 3]]))
    with pytest.raises(_lib.SbiB200Error, match=r"MMD: 65537 index sets"):
        M._mmd_sets(z, torch.zeros(65_537, 4, dtype=torch.int32), torch.tensor([[1, 3]]))
    with pytest.raises(_lib.SbiB200Error, match=r"over a \(4, 0\) matrix"):
        M._mmd_sets(torch.zeros(4, 0), torch.zeros(1, 4, dtype=torch.int32), torch.tensor([[1, 3]]))


def test_module_imports_without_sklearn():
    import subprocess
    import sys
    code = ("import sys\n"
            "class Block:\n"
            "    def find_spec(self, name, path, target=None):\n"
            "        if name.split('.')[0] == 'sklearn': raise ImportError('blocked')\n"
            "sys.meta_path.insert(0, Block())\n"
            "from sbi_b200.diagnostics import calc_misspecification_mmd\n"
            "from sbi_b200 import misspecification\n"
            "print('ok')\n")
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


@no_gpu
def test_no_cpu_fallback():
    x_obs, x = torch.randn(3, 2), torch.randn(50, 2)
    for call in (lambda: calc_misspecification_mmd(x_obs, x, n_shuffle=4),
                 lambda: M.calculate_baseline_mmd(3, x, n_shuffle=4),
                 lambda: M.compute_rbf_mmd(x_obs, x), lambda: M.compute_rbf_mmd_median_heuristic(x_obs, x),
                 lambda: M.median_heuristic(x_obs, x), lambda: M.rbf_kernel(x_obs, x, 1.0)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()
