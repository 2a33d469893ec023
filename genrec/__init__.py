"""Import-path shim: ``genrec.models.{hstu,sasrec,rqvae}`` and ``genrec.data.{amazon_hstu,amazon_sasrec}`` resolve to the
H100-native modules in ``genrec_b200`` so that the reference's gin files (``import genrec.data.amazon_hstu`` /
``import genrec.models.hstu``, config/hstu/amazon.gin:5-6) and trainers find the hot path under the names they already use.

This package does NOT shadow the rest of the reference: every level extends its ``__path__`` over all ``genrec`` directories on
``sys.path`` (``pkgutil.extend_path``), so with a reference checkout on the path AFTER this repository
(``PYTHONPATH=/path/to/genrec_b200_repo:/path/to/phonism_genrec``) ``genrec.trainers.hstu_trainer``, ``genrec.modules.*``,
``genrec.models.tiger`` ... still import from the reference, while the five modules named above come from here.
Without a reference checkout the five modules work on their own (tests/test_modules_cpu.py)."""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
