"""python-paillier_b200: an H100-native batched Paillier engine behind the ``phe`` API.

The directory name carries a hyphen (it mirrors the reference repo's name), so import it with
``importlib.import_module("python-paillier_b200")`` or through the root-level alias module
``paillier_b200`` (``import paillier_b200 as phe``).
"""
from .engine import (Engine, EngineError, EngineUnavailable, ModContext, PrivateContext, PublicContext,  # noqa: F401
                     get_engine, ints_to_limbs, limbs_to_ints)

from .encoding import EncodedNumber  # noqa: F401,E402
from .paillier import (DEFAULT_KEYSIZE, EncryptedNumber, PaillierPrivateKey, PaillierPrivateKeyring,  # noqa: F401,E402
                       PaillierPublicKey, generate_paillier_keypair, generate_paillier_keypairs)
from . import util  # noqa: F401,E402
from .vector import EncryptedVector, PackedEncryptedVector  # noqa: F401,E402

__version__ = "0.1.0"
