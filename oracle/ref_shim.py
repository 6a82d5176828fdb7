"""Make the UNMODIFIED reference sbi (staged under oracle/_ref by build()) importable.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The reference's third-party arithmetic
library ``nflows==0.14`` is absent and not installable offline, so this module

* aliases ``oracle.nflows_port`` (our restatement) under the module name ``nflows``;
* registers inert stub modules for packages sbi imports at module top but that the
  hot path never calls (zuko, pyro, matplotlib, skorch, pymc, arviz, ...): attribute
  access on a stub returns another stub / a dummy class, so ``from x import Y`` works;
* puts the reference root on ``sys.path``.

Used by ``tests/golden/make_golden.py`` (fixture generation), by tests that are skipped when
no copy of the reference exists, and by ``bench.py --impl reference``.
"""
import importlib
import importlib.abc
import importlib.machinery
import os
import sys
import types

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _find_reference():
    """$SBI_REFERENCE_ROOT if set, else the unmodified reference package that build() staged under
    oracle/_ref (oracle/ref_build.py; git-ignored)."""
    for c in (os.environ.get("SBI_REFERENCE_ROOT"), os.path.join(_REPO, "oracle", "_ref")):
        if c and os.path.isdir(os.path.join(c, "sbi")):
            return c
    return os.path.join(_REPO, "oracle", "_ref")


REFERENCE_ROOT = _find_reference()

_STUB_ROOTS = ("zuko", "pyro", "matplotlib", "skorch", "pymc", "arviz", "tabpfn",
               "pytest_harvest", "torchtestcase")


class _StubMeta(type):
    def __getattr__(cls, name):  # class-level attribute access, e.g. Figure.something
        if name.startswith("__"):
            raise AttributeError(name)
        return _make_stub_class(f"{cls.__name__}.{name}")

    def __call__(cls, *a, **k):
        if cls.__dict__.get("_stub_instantiable", True):
            return type.__call__(cls)
        raise RuntimeError(f"stub {cls.__name__} cannot be instantiated")

    def __or__(cls, other):
        return cls

    def __ror__(cls, other):
        return cls

    def __getitem__(cls, item):
        return cls


def _make_stub_class(name):
    return _StubMeta(name.split(".")[-1], (), {"__module__": "oracle_stub",
                                               "__init__": lambda self, *a, **k: None})


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        full = f"{self.__name__}.{name}"
        if full in sys.modules:
            return sys.modules[full]
        if name[:1].isupper() or name in ("pyplot",):
            if name == "pyplot":
                return importlib.import_module(full)
            obj = _make_stub_class(full)
        else:
            # lower-case names may be submodules (zuko.flows) or functions; return a
            # stub module, which is also callable.
            obj = importlib.import_module(full)
        setattr(self, name, obj)
        return obj

    def __call__(self, *a, **k):
        raise RuntimeError(f"stub {self.__name__} called: not available offline")


class _StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path, target=None):
        if fullname.split(".")[0] in _STUB_ROOTS:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def _alias_nflows():
    from oracle import nflows_port

    prefix = nflows_port.__name__
    # make sure every submodule is imported
    for sub in ("utils.torchutils", "utils.typechecks", "distributions.base",
                "distributions.normal", "distributions.mixture", "flows.base",
                "nn.nets.resnet", "nn.nde.made", "transforms.base", "transforms.standard",
                "transforms.linear", "transforms.lu", "transforms.permutations",
                "transforms.coupling", "transforms.autoregressive", "transforms.made",
                "transforms.splines.rational_quadratic"):
        importlib.import_module(f"{prefix}.{sub}")
    for name, mod in list(sys.modules.items()):
        if name == prefix or name.startswith(prefix + "."):
            sys.modules["nflows" + name[len(prefix):]] = mod


_installed = False


def install():
    """Idempotently install the shim; returns True if /root/reference is available."""
    global _installed
    if not os.path.isdir(os.path.join(REFERENCE_ROOT, "sbi")):
        return False
    if _installed:
        return True
    _alias_nflows()
    sys.meta_path.append(_StubFinder())
    if REFERENCE_ROOT not in sys.path:
        sys.path.append(REFERENCE_ROOT)   # at the END: the reference tree has its own `tests` package
    _installed = True
    return True


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "sbi"))
