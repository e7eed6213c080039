"""Drop-in ``phe.paillier`` API on top of the H100 engine.

Same classes, method names, argument meaning and exceptions as the reference
(phe/paillier.py of data61/python-paillier 1.5.0); the big-integer work -- ``r^n mod n^2`` (:137, :622), the CRT pair
(:346-353), ``a*b mod n^2`` (:719), ``c^k mod n^2`` (:749-751) -- runs in the CUDA kernels, batch of
one for the scalar methods and full batches for the ``*_batch`` methods / ``EncryptedVector``
(vector.py).  Nothing here falls back to CPU bigint arithmetic for those operations.
"""
import random

try:
    from collections.abc import Mapping
except ImportError:          # pragma: no cover
    Mapping = dict

from . import engine as _engine
from .encoding import EncodedNumber
from .util import getprimeover, invert, isqrt, mulmod, powmod

DEFAULT_KEYSIZE = 3072


def generate_paillier_keypair(private_keyring=None, n_length=DEFAULT_KEYSIZE):
    """New (PaillierPublicKey, PaillierPrivateKey) with an n of exactly n_length bits
    (phe/paillier.py:37-68).  Key generation is host-side and not part of the accelerated path."""
    while True:
        p = getprimeover(n_length // 2)
        q = getprimeover(n_length // 2)
        if p != q and (p * q).bit_length() == n_length:
            break
    public_key = PaillierPublicKey(p * q)
    private_key = PaillierPrivateKey(public_key, p, q)
    if private_keyring is not None:
        private_keyring.add(private_key)
    return public_key, private_key


def generate_paillier_keypairs(count, n_length=DEFAULT_KEYSIZE):
    """`count` key pairs at once (the reference's test-suite makes 100 of them one by one, phe/tests/paillier_test.py:62-71):
    all prime candidates of a round are tested in one batched Miller-Rabin launch (util.getprimeover_batch)."""
    from .util import getprimeover_batch
    keys = []
    pool = []
    while len(keys) < count:
        need = 2 * (count - len(keys)) + 2
        pool += getprimeover_batch(n_length // 2, need)
        while len(pool) >= 2 and len(keys) < count:
            p, q = pool.pop(), pool.pop()
            if p != q and (p * q).bit_length() == n_length:
                pk = PaillierPublicKey(p * q)
                keys.append((pk, PaillierPrivateKey(pk, p, q)))
    return keys


class PaillierPublicKey(object):
    """Public key n (g = n + 1) with the encryption methods (phe/paillier.py:71-194)."""

    def __init__(self, n):
        self.g = n + 1
        self.n = n
        self.nsquare = n * n
        self.max_int = n // 3 - 1
        self._ctx = None

    def __repr__(self):
        return "<PaillierPublicKey {}>".format(hex(hash(self))[2:][:10])

    def __eq__(self, other):
        return self.n == other.n

    def __hash__(self):
        return hash(self.n)

    # the engine context is created on first use and is not part of the key's value
    def engine_context(self):
        if self._ctx is None:
            self._ctx = _engine.PublicContext(self.n)
        return self._ctx

    def __getstate__(self):
        return {"n": self.n}

    def __setstate__(self, state):
        self.__init__(state["n"])

    def get_random_lt_n(self):
        return random.SystemRandom().randrange(1, self.n)

    def raw_encrypt(self, plaintext, r_value=None):
        """(1 + n*plaintext) * r^n mod n^2 as a Python int (phe/paillier.py:102-139)."""
        if not isinstance(plaintext, int):
            raise TypeError('Expected int type plaintext but got: %s' % type(plaintext))
        r = r_value or self.get_random_lt_n()
        if r == 1:
            # powmod(1, n, n^2) is the reference's own shortcut (phe/util.py:45-46): nothing to exponentiate
            return (self.n * plaintext + 1) % self.nsquare
        if not 0 < r < self.nsquare:
            r %= self.nsquare
        if r >= 1 << (32 * self.engine_context().n_limbs):
            # an obfuscator wider than n: r^n through the generic seam, then one mulmod
            return mulmod((self.n * plaintext + 1) % self.nsquare, powmod(r, self.n, self.nsquare), self.nsquare)
        return self.engine_context().raw_encrypt([plaintext], [r])[0]

    def raw_encrypt_batch(self, plaintexts, r_values=None):
        """Batched raw_encrypt: list of ints -> list of ints (one kernel launch)."""
        return self._raw_encrypt_batch(plaintexts, r_values, self.engine_context())

    def _raw_encrypt_batch(self, plaintexts, r_values, ctx):
        """raw_encrypt_batch on the engine context `ctx`: this key's PublicContext or its private key's PrivateContext,
        which give the same bits."""
        plaintexts = list(plaintexts)
        for m in plaintexts:
            if not isinstance(m, int):
                raise TypeError('Expected int type plaintext but got: %s' % type(m))
        rnd = random.SystemRandom()
        if r_values is None:
            r_values = [rnd.randrange(1, self.n) for _ in plaintexts]
        else:
            r_values = list(r_values)
            if len(r_values) != len(plaintexts):
                raise ValueError("plaintexts and r_values differ in length")
        # per element exactly what raw_encrypt does with r (phe/paillier.py:136-137): a falsy r draws a fresh one,
        # anything outside (0, n^2) is reduced as powmod would; the rare element whose r does not fit the engine's
        # rows (n <= 2^(32 Ln) <= r < n^2, legal for the reference) takes the scalar path
        lim = 1 << (32 * self.engine_context().n_limbs)
        r_values = [(r or rnd.randrange(1, self.n)) for r in r_values]
        r_values = [r if 0 < r < self.nsquare else r % self.nsquare for r in r_values]
        wide = {i: self.raw_encrypt(plaintexts[i], r) for i, r in enumerate(r_values) if r >= lim}
        if not wide:
            return ctx.raw_encrypt(plaintexts, r_values)
        keep = [i for i in range(len(plaintexts)) if i not in wide]
        bulk = iter(ctx.raw_encrypt([plaintexts[i] for i in keep], [r_values[i] for i in keep]))
        return [wide[i] if i in wide else next(bulk) for i in range(len(plaintexts))]

    def encrypt(self, value, precision=None, r_value=None):
        encoding = value if isinstance(value, EncodedNumber) else EncodedNumber.encode(self, value, precision)
        return self.encrypt_encoded(encoding, r_value)

    def encrypt_encoded(self, encoding, r_value):
        """phe/paillier.py:177-194: with r_value None the ciphertext is obfuscated with a fresh random r
        (here in the same kernel launch as the encryption)."""
        if r_value is None:
            ciphertext = self.raw_encrypt(encoding.encoding, self.get_random_lt_n())
            number = EncryptedNumber(self, ciphertext, encoding.exponent)
            number._mark_obfuscated()
            return number
        return EncryptedNumber(self, self.raw_encrypt(encoding.encoding, r_value=r_value or 1), encoding.exponent)

    def encrypt_batch(self, values, precision=None, r_values=None):
        """Encode and encrypt a sequence in one launch; returns an EncryptedVector (device resident)."""
        from .vector import EncryptedVector
        return EncryptedVector.encrypt(self, values, precision=precision, r_values=r_values)

    def encrypt_packed(self, values, bound, frac_bits=24, headroom=1024, r_values=None):
        """Fixed-point values packed many to a ciphertext (PackedEncryptedVector, DESIGN.md section 3.10): |x| <= bound,
        frac_bits fractional bits, slots wide enough for `headroom` such vectors to be added.  r_values: one per
        ciphertext, or None for fresh ones."""
        from .vector import PackedEncryptedVector
        return PackedEncryptedVector.encrypt(self, values, bound, frac_bits, headroom, r_values)


class PaillierPrivateKey(object):
    """Private key (p, q) with CRT decryption (phe/paillier.py:197-380)."""

    def __init__(self, public_key, p, q):
        if not p * q == public_key.n:
            raise ValueError('given public key does not match the given p and q.')
        if p == q:
            raise ValueError('p and q have to be different')
        self.public_key = public_key
        self.p, self.q = (p, q) if p < q else (q, p)
        self.psquare = self.p * self.p
        self.qsquare = self.q * self.q
        self._ctx = None
        # derived on the device by the engine (p^-1 mod q, h(p), h(q); phe/paillier.py:233-235)
        ctx = self.engine_context()
        self.p_inverse = ctx.p_inverse
        self.hp = ctx.hp
        self.hq = ctx.hq

    def engine_context(self):
        if self._ctx is None:
            self._ctx = _engine.PrivateContext(self.p, self.q)
        return self._ctx

    def __getstate__(self):
        return {"n": self.public_key.n, "p": self.p, "q": self.q}

    def __setstate__(self, state):
        self.__init__(PaillierPublicKey(state["n"]), state["p"], state["q"])

    @staticmethod
    def from_totient(public_key, totient):
        """Recover (p, q) from the totient (p-1)(q-1) (phe/paillier.py:237-262)."""
        p_plus_q = public_key.n - totient + 1
        p_minus_q = isqrt(p_plus_q * p_plus_q - public_key.n * 4)
        q = (p_plus_q - p_minus_q) // 2
        p = p_plus_q - q
        if not p * q == public_key.n:
            raise ValueError('given public key and totient do not match.')
        return PaillierPrivateKey(public_key, p, q)

    def __repr__(self):
        return "<PaillierPrivateKey for {}>".format(repr(self.public_key))

    def decrypt(self, encrypted_number):
        return self.decrypt_encoded(encrypted_number).decode()

    def decrypt_encoded(self, encrypted_number, Encoding=None):
        if not isinstance(encrypted_number, EncryptedNumber):
            raise TypeError('Expected encrypted_number to be an EncryptedNumber'
                            ' not: %s' % type(encrypted_number))
        if self.public_key != encrypted_number.public_key:
            raise ValueError('encrypted_number was encrypted against a '
                             'different key!')
        if Encoding is None:
            Encoding = EncodedNumber
        encoded = self.raw_decrypt(encrypted_number.ciphertext(be_secure=False))
        return Encoding(self.public_key, encoded, encrypted_number.exponent)

    def raw_decrypt(self, ciphertext):
        """CRT decryption of one raw ciphertext (phe/paillier.py:328-354), in the K2 kernel."""
        if not isinstance(ciphertext, int):
            raise TypeError('Expected ciphertext to be an int, not: %s' % type(ciphertext))
        return self.engine_context().raw_decrypt([ciphertext])[0]

    def raw_encrypt_batch(self, plaintexts, r_values=None):
        """public_key.raw_encrypt_batch element by element, computed with p and q (pai_priv_encrypt)."""
        return self.public_key._raw_encrypt_batch(plaintexts, r_values, self.engine_context())

    def encrypt_batch(self, values, precision=None, r_values=None):
        """public_key.encrypt_batch (same ciphertexts and exponents for the same r_values), computed with p and q."""
        from .vector import EncryptedVector
        return EncryptedVector.encrypt(self.public_key, values, precision=precision, r_values=r_values, private_key=self)

    def encrypt_packed(self, values, bound, frac_bits=24, headroom=1024, r_values=None):
        """public_key.encrypt_packed (the same ciphertexts for the same r_values), computed with p and q."""
        from .vector import PackedEncryptedVector
        return PackedEncryptedVector.encrypt(self.public_key, values, bound, frac_bits, headroom, r_values, private_key=self)

    def raw_decrypt_batch(self, ciphertexts):
        for c in ciphertexts:
            if not isinstance(c, int):
                raise TypeError('Expected ciphertext to be an int, not: %s' % type(c))
        return self.engine_context().raw_decrypt(list(ciphertexts))

    def decrypt_batch(self, vector):
        """Decrypt and decode an EncryptedVector -> list of Python numbers (a PackedEncryptedVector -> float64 tensor)."""
        return vector.decrypt(self)

    # the reference exposes these helpers as methods (phe/paillier.py:356-374); kept for API parity
    def h_function(self, x, xsquare):
        return invert(self.l_function(powmod(self.public_key.g, x - 1, xsquare), x), x)

    def l_function(self, x, p):
        return (x - 1) // p

    def crt(self, mp, mq):
        u = mulmod(mq - mp, self.p_inverse, self.q)
        return mp + (u * self.p)

    def __eq__(self, other):
        return self.p == other.p and self.q == other.q

    def __hash__(self):
        return hash((self.p, self.q))


class PaillierPrivateKeyring(Mapping):
    """dict-like holder of private keys indexed by public key (phe/paillier.py:383-439)."""

    def __init__(self, private_keys=None):
        self.__keyring = {k.public_key: k for k in (private_keys or [])}

    def __getitem__(self, key):
        return self.__keyring[key]

    def __len__(self):
        return len(self.__keyring)

    def __iter__(self):
        return iter(self.__keyring)

    def __delitem__(self, public_key):
        del self.__keyring[public_key]

    def add(self, private_key):
        if not isinstance(private_key, PaillierPrivateKey):
            raise TypeError("private_key should be of type PaillierPrivateKey, "
                            "not %s" % type(private_key))
        self.__keyring[private_key.public_key] = private_key

    def decrypt(self, encrypted_number):
        return self.__keyring[encrypted_number.public_key].decrypt(encrypted_number)


class EncryptedNumber(object):
    """One Paillier ciphertext with its fixed-point exponent (phe/paillier.py:442-751).

    ``+`` multiplies ciphertexts mod n^2, ``*`` by a plaintext scalar exponentiates; results are not
    obfuscated until ``ciphertext(be_secure=True)`` / ``obfuscate()`` is called, as in the reference.
    """

    def __init__(self, public_key, ciphertext, exponent=0):
        self.public_key = public_key
        self.__ciphertext = ciphertext
        self.exponent = exponent
        self.__is_obfuscated = False
        if isinstance(self.ciphertext, EncryptedNumber):        # same (ineffective) check as phe/paillier.py:485
            raise TypeError('ciphertext should be an integer')
        if not isinstance(self.public_key, PaillierPublicKey):
            raise TypeError('public_key should be a PaillierPublicKey')

    def _mark_obfuscated(self):
        self.__is_obfuscated = True

    # ---- operators
    def __add__(self, other):
        if isinstance(other, EncryptedNumber):
            return self._add_encrypted(other)
        if isinstance(other, EncodedNumber):
            return self._add_encoded(other)
        return self._add_scalar(other)

    def __radd__(self, other):
        return self.__add__(other)

    def __mul__(self, other):
        if isinstance(other, EncryptedNumber):
            raise NotImplementedError('Good luck with that...')
        encoding = other if isinstance(other, EncodedNumber) else EncodedNumber.encode(self.public_key, other)
        product = self._raw_mul(encoding.encoding)
        return EncryptedNumber(self.public_key, product, self.exponent + encoding.exponent)

    def __rmul__(self, other):
        return self.__mul__(other)

    def __sub__(self, other):
        return self + (other * -1)

    def __rsub__(self, other):
        return other + (self * -1)

    def __truediv__(self, scalar):
        return self.__mul__(1 / scalar)

    # ---- ciphertext access / obfuscation
    def ciphertext(self, be_secure=True):
        if be_secure and not self.__is_obfuscated:
            self.obfuscate()
        return self.__ciphertext

    def obfuscate(self):
        """c <- c * r^n mod n^2 with a fresh random r (phe/paillier.py:603-624)."""
        pk = self.public_key
        r = pk.get_random_lt_n()
        r_pow_n = pk.raw_encrypt(0, r)                 # (1 + n*0) * r^n = r^n mod n^2, in the K1 kernel
        self.__ciphertext = self._raw_add(self.__ciphertext, r_pow_n)
        self.__is_obfuscated = True

    def decrease_exponent_to(self, new_exp):
        if new_exp > self.exponent:
            raise ValueError('New exponent %i should be more negative than '
                             'old exponent %i' % (new_exp, self.exponent))
        multiplied = self * pow(EncodedNumber.BASE, self.exponent - new_exp)
        multiplied.exponent = new_exp
        return multiplied

    # ---- additions
    def _add_scalar(self, scalar):
        encoded = EncodedNumber.encode(self.public_key, scalar, max_exponent=self.exponent)
        return self._add_encoded(encoded)

    def _align(self, other):
        """Bring self and other (EncryptedNumber or EncodedNumber) to the lower of the two exponents."""
        a, b = self, other
        if a.exponent > b.exponent:
            a = self.decrease_exponent_to(b.exponent)
        elif a.exponent < b.exponent:
            b = b.decrease_exponent_to(a.exponent)
        return a, b

    def _add_encoded(self, encoded):
        if self.public_key != encoded.public_key:
            raise ValueError("Attempted to add numbers encoded against "
                             "different public keys!")
        a, b = self._align(encoded)
        encrypted_scalar = a.public_key.raw_encrypt(b.encoding, 1)       # nude ciphertext, no exponentiation
        return EncryptedNumber(a.public_key, a._raw_add(a.ciphertext(False), encrypted_scalar), a.exponent)

    def _add_encrypted(self, other):
        if self.public_key != other.public_key:
            raise ValueError("Attempted to add numbers encrypted against "
                             "different public keys!")
        a, b = self._align(other)
        return EncryptedNumber(a.public_key, a._raw_add(a.ciphertext(False), b.ciphertext(False)), a.exponent)

    # ---- raw operations (engine, batch of one)
    def _raw_add(self, e_a, e_b):
        """E(a) * E(b) mod n^2 (phe/paillier.py:705-719)."""
        pk = self.public_key
        lim = 1 << (32 * pk.engine_context().c_limbs)
        if not (0 <= e_a < lim and 0 <= e_b < lim):
            e_a, e_b = e_a % pk.nsquare, e_b % pk.nsquare
        return pk.engine_context().raw_add([e_a], [e_b])[0]

    def _raw_mul(self, plaintext):
        """E(a) ^ plaintext mod n^2 with the reference's negative-scalar branch (phe/paillier.py:721-751)."""
        if not isinstance(plaintext, int):
            raise TypeError('Expected ciphertext to be int, not %s' % type(plaintext))
        pk = self.public_key
        if plaintext < 0 or plaintext >= pk.n:
            raise ValueError('Scalar out of bounds: %i' % plaintext)
        c = self.ciphertext(False)
        if not 0 <= c < (1 << (32 * pk.engine_context().c_limbs)):
            c %= pk.nsquare
        out, status = pk.engine_context().raw_mul([c], [plaintext])
        if status[0]:
            raise ZeroDivisionError('invert() no inverse exists')
        return out[0]
