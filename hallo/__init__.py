"""`hallo` overlay package: makes the H100 engine a drop-in under the reference's own import paths.

scripts/inference.py:38-47 imports `hallo.animate.face_animate`, `hallo.models.{audio_proj, unet_3d, unet_2d_condition,
face_locator, image_proj}`, `hallo.datasets.*`, `hallo.utils.*`.  This package sits FIRST on sys.path
(`PYTHONPATH=/path/to/hallo_b200_repo:/path/to/hallo`) and provides only the hot-path modules

    hallo.models.unet_3d                 -> hallo_b200.models.unet_3d
    hallo.models.audio_proj              -> hallo_b200.models.audio_proj
    hallo.models.mutual_self_attention   -> hallo_b200.models.mutual_self_attention
    hallo.animate.face_animate           -> hallo_b200.animate.face_animate

Every other `hallo.*` module (datasets, utils, face_locator, image_proj, unet_2d_condition, wav2vec ...) resolves to
the reference checkout found later on sys.path (or named by $HALLO_REFERENCE_ROOT): the package `__path__`s are
extended with the reference's directories, ours searched first.  So the script runs unchanged; see INTEGRATION.md.
"""
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))


def _reference_dirs(sub: str = ""):
    """Directories named hallo/<sub> that belong to OTHER sys.path entries (the maintainer's reference checkout)."""
    roots = []
    env = os.environ.get("HALLO_REFERENCE_ROOT")
    if env:
        roots.append(env)
    roots += [p for p in sys.path if p]
    out = []
    for r in roots:
        d = os.path.join(os.path.abspath(r), "hallo", sub) if sub else os.path.join(os.path.abspath(r), "hallo")
        if os.path.isdir(d) and os.path.abspath(d) != os.path.abspath(os.path.join(_HERE, sub)) and d not in out:
            out.append(d)
    return out


__path__ = [_HERE] + _reference_dirs()
