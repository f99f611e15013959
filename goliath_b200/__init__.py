"""goliath_b200 — H100-native (sm_90a) implementation of the goliath avatar render hot path.

Public surface (mirrors the reference's extension modules, SURVEY.md §8b):
  goliath_b200.sgutilslib / sgutils        — SG specular shade       (extensions/sgutils)
  goliath_b200.gsplat                      — project_gaussians / rasterize_gaussians (gsplat 0.1.11 API)
  goliath_b200.utilslib / utils            — compute_raydirs          (extensions/utils)
  goliath_b200.mvpraymarchlib / mvpraymarch— MVP raymarcher           (extensions/mvpraymarch)
  goliath_b200.install_dropins()           — register the modules under the reference's import names
"""
__version__ = "0.1.0"


def install_dropins():
    """Make `import sgutilslib`, `import gsplat`, ... resolve to this package, so that the reference's
    ca_code/models/*.py and extensions/*/*.py wrappers run unchanged (SURVEY.md §0.3)."""
    import importlib
    import sys

    for name in ("sgutilslib", "gsplat", "utilslib", "mvpraymarchlib"):
        try:
            sys.modules.setdefault(name, importlib.import_module("goliath_b200." + name))
        except ImportError:
            pass
