"""Host-side mirror of the reference's prover surface over the C ABI (include/zkb200.h).

Names follow upstream bellman 0.1.0 as the reference uses them:
  Parameters.read(buf, checked)      core/proofs/src/confidential.rs:99
  create_proof / create_random_proof core/proofs/src/confidential.rs:149, anonymous.rs:165
  multiexp(bases, exponents)         bellman::multiexp::multiexp  (SURVEY.md §3.2)
  EvaluationDomain.{fft,ifft,coset_fft,icoset_fft}   bellman::domain (SURVEY.md §8 a7)
  Proof (192-byte wire form)         core/bellman-verifier/src/lib.rs:40-110
Errors mirror bellman::SynthesisError (zface/src/error.rs:17,45-48).

All numeric arrays are numpy uint64 little-endian limbs: Fr canonical (n,4) at this boundary,
points in "limb form" (Montgomery x|y).  Everything computes on the GPU through libzkb200.so;
importing works without a GPU, any compute call without one raises ZkError(ZK_ERR_CUDA).
"""
from __future__ import annotations

import collections
import ctypes as C
import re
import secrets

import numpy as np

from . import _lib
from ._lib import ZkError, check

R_MODULUS = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


class SynthesisError(Exception):
    """bellman::SynthesisError variants reachable from the prover path."""
    NAMES = {-3: "AssignmentMissing", -4: "PolynomialDegreeTooLarge", -5: "UnexpectedIdentity", -6: "IoError",
             -7: "IoError(GroupDecodingError)", -8: "IoError(NotInField)", -9: "MalformedVerifyingKey"}

    def __init__(self, code, msg):
        super().__init__("%s: %s" % (self.NAMES.get(code, "Error(%d)" % code), msg))
        self.code = code


def _ck(code):
    if code == 0:
        return
    msg = _lib.lib().zk_last_error().decode()
    if code in SynthesisError.NAMES:
        raise SynthesisError(code, msg)
    raise ZkError(code, msg)


def _u64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.reshape(shape) if shape is not None else a


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Context:
    """One CUDA device + stream (the analogue of bellman's multicore::Worker)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self._h = C.c_void_p()
        _ck(_lib.lib().zk_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(self._h)))
        self.device = device

    @property
    def stream(self) -> int:
        return _lib.lib().zk_ctx_stream(self._h) or 0

    def sync(self):
        _ck(_lib.lib().zk_ctx_sync(self._h))

    OPT_AFFINE_MIN_ENTRIES, OPT_AFFINE_LEVELS, OPT_VERIFY_LANES = 1, 2, 3

    def set_opt(self, opt: int, value: int):
        """zk_ctx_set_opt: tuning only (batched-affine threshold / rounds); results never depend on it."""
        _ck(_lib.lib().zk_ctx_set_opt(self._h, opt, value))

    def profile(self, enable: bool):
        _ck(_lib.lib().zk_ctx_profile(self._h, int(enable)))

    def profile_read(self):
        """(total ms, launches) of the dominant kernel since profile(True), CUDA events on this stream."""
        ms, n = C.c_double(), C.c_uint64()
        _ck(_lib.lib().zk_ctx_profile_read(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def profile_counts(self):
        """(G1 bucket additions, G2 bucket additions, G1 left to the XYZZ pass, G2 left to the XYZZ pass) executed by this
        context's MSMs (lanes included) since profile()."""
        v = [C.c_uint64() for _ in range(4)]
        _ck(_lib.lib().zk_ctx_profile_counts(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def close(self):
        if self._h:
            _lib.lib().zk_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Bases:
    """Device-resident base points (+ window tables) for multiexp; group 1 = G1, 2 = G2."""

    def __init__(self, ctx: Context, group: int, limbs, window_bits: int = 0, precompute: bool = True):
        w = 12 if group == 1 else 24
        limbs = _u64(limbs, (-1, w))
        self.ctx, self.group, self.n = ctx, group, limbs.shape[0]
        self._h = C.c_void_p()
        _ck(_lib.lib().zk_bases_upload(ctx._h, group, _p(limbs), self.n, window_bits, int(precompute), C.byref(self._h)))
        self.window_bits = _lib.lib().zk_bases_window_bits(self._h)

    def free(self):
        if self._h:
            _lib.lib().zk_bases_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def multiexp(bases: Bases, exponents) -> bytes:
    """sum_i exponents[i] * bases[i]; exponents canonical (n,4) uint64 in HOST memory.
    Returns the uncompressed encoding (96 B G1 / 192 B G2)."""
    e = _u64(exponents, (-1, 4))
    out = np.zeros(96 if bases.group == 1 else 192, np.uint8)
    _ck(_lib.lib().zk_msm(bases.ctx._h, bases._h, _p(e), e.shape[0], _p(out)))
    return out.tobytes()


def multiexp_begin(ctx: Context, bases: Bases, exponents):
    """multiexp as a future (bellman's multiexp returns one): enqueue on `ctx`, collect with multiexp_end(ctx, bases).  `bases`
    may have been created through another context of the same device; alternate two contexts to pipeline successive MSMs."""
    e = _u64(exponents, (-1, 4))
    _ck(_lib.lib().zk_msm_begin(ctx._h, bases._h, _p(e), e.shape[0]))
    ctx._keep = e                         # the upload is asynchronous: keep the buffer alive until multiexp_end


def multiexp_device_begin(ctx: Context, bases: Bases, d_scalars_ptr: int, n: int):
    _ck(_lib.lib().zk_msm_device_begin(ctx._h, bases._h, C.c_void_p(d_scalars_ptr), n))


def multiexp_partial_device_begin(ctx: Context, bases: Bases, d_scalars_ptr: int, n: int, d_out_ptr: int):
    _ck(_lib.lib().zk_msm_partial_device_begin(ctx._h, bases._h, C.c_void_p(d_scalars_ptr), n, C.c_void_p(d_out_ptr)))


def points_fold_begin(ctx: Context, group: int, d_partials_ptr: int, count: int):
    _ck(_lib.lib().zk_points_fold_begin(ctx._h, group, C.c_void_p(d_partials_ptr), count))


def tail_stream(ctx: Context) -> int:
    """CUDA stream (high priority) on which a context finishes its futures; enqueue the all-gather of partials here."""
    return int(_lib.lib().zk_ctx_tail_stream(ctx._h))


def multiexp_end(ctx: Context, bases: Bases) -> bytes:
    out = np.zeros(96 if bases.group == 1 else 192, np.uint8)
    _ck(_lib.lib().zk_msm_end(ctx._h, _p(out)))
    ctx._keep = None
    return out.tobytes()


def multiexp_partial_device(bases: Bases, d_scalars_ptr: int, n: int, d_out_ptr: int):
    """Partial MSM result (XYZZ point, zk_partial_size bytes) left in device memory for the NCCL all-gather."""
    _ck(_lib.lib().zk_msm_partial_device(bases.ctx._h, bases._h, C.c_void_p(d_scalars_ptr), n, C.c_void_p(d_out_ptr)))


def points_fold(ctx: Context, group: int, d_partials_ptr: int, count: int) -> bytes:
    out = np.zeros(96 if group == 1 else 192, np.uint8)
    _ck(_lib.lib().zk_points_fold(ctx._h, group, C.c_void_p(d_partials_ptr), count, _p(out)))
    return out.tobytes()


def partial_size(group: int) -> int:
    return _lib.lib().zk_partial_size(group)


def multiexp_device(bases: Bases, d_scalars_ptr: int, n: int, batch: int = 1) -> bytes:
    out = np.zeros((96 if bases.group == 1 else 192) * batch, np.uint8)
    _ck(_lib.lib().zk_msm_batch_device(bases.ctx._h, bases._h, C.c_void_p(d_scalars_ptr), n, batch, _p(out)))
    return out.tobytes()


class EvaluationDomain:
    """Radix-2 domain over Fr; data are MONTGOMERY-form (n,4) uint64 arrays, natural order."""
    FFT, IFFT, COSET_FFT, ICOSET_FFT = 0, 1, 2, 3

    def __init__(self, ctx: Context, coeffs_mont):
        a = _u64(coeffs_mont, (-1, 4))
        m, exp = 1, 0
        while m < a.shape[0]:
            m *= 2
            exp += 1
            if exp >= 32:
                raise SynthesisError(-4, "PolynomialDegreeTooLarge")
        self.ctx, self.exp = ctx, exp
        self.coeffs = np.zeros((m, 4), np.uint64)
        self.coeffs[: a.shape[0]] = a

    def _run(self, mode):
        _ck(_lib.lib().zk_ntt_fr(self.ctx._h, _p(self.coeffs), self.exp, mode))
        return self

    def fft(self): return self._run(self.FFT)
    def ifft(self): return self._run(self.IFFT)
    def coset_fft(self): return self._run(self.COSET_FFT)
    def icoset_fft(self): return self._run(self.ICOSET_FFT)


class Parameters:
    """groth16::Parameters<Bls12> held on the device."""

    def __init__(self, ctx: Context, handle, counts):
        self.ctx, self._h = ctx, handle
        self.n_ic, self.n_h, self.n_l, self.n_a, self.n_b_g1, self.n_b_g2 = counts

    @staticmethod
    def read(ctx: Context, buf: bytes, checked: bool = True) -> "Parameters":
        b = np.frombuffer(buf, np.uint8)
        h = C.c_void_p()
        _ck(_lib.lib().zk_params_load(ctx._h, _p(b), len(buf), int(checked), C.byref(h)))
        cnt = np.zeros(6, np.uint64)
        _ck(_lib.lib().zk_params_counts(h, _p(cnt)))
        return Parameters(ctx, h, [int(x) for x in cnt])

    @staticmethod
    def read_cached(ctx: Context, buf: bytes, cache_path: str) -> "Parameters":
        """Parameters::read(buf, true) through the decoded-CRS cache on disk (zk_params_load_cached); `.cache_hit` tells which
        path ran.  The reference re-reads and re-checks the whole proving key on every start (crypto_components.rs:320-328)."""
        b = np.frombuffer(buf, np.uint8)
        h, hit = C.c_void_p(), C.c_int(0)
        _ck(_lib.lib().zk_params_load_cached(ctx._h, _p(b), len(buf), cache_path.encode(), C.byref(hit), C.byref(h)))
        cnt = np.zeros(6, np.uint64)
        _ck(_lib.lib().zk_params_counts(h, _p(cnt)))
        prm = Parameters(ctx, h, [int(x) for x in cnt])
        prm.cache_hit = bool(hit.value)
        return prm

    def write(self) -> bytes:
        """Parameters::write (core/proofs/src/confidential.rs:83): the resident CRS as the exact byte stream `read` consumes."""
        out = np.zeros(int(_lib.lib().zk_params_size(self._h)), np.uint8)
        _ck(_lib.lib().zk_params_write(self.ctx._h, self._h, _p(out)))
        return out.tobytes()

    def vk_bytes(self) -> bytes:
        """VerifyingKey::write of `params.vk` (core/proofs/src/setup.rs:31): the head of the Parameters stream."""
        out = np.zeros(int(_lib.lib().zk_params_vk_size(self._h)), np.uint8)
        _ck(_lib.lib().zk_params_write_vk(self.ctx._h, self._h, _p(out)))
        return out.tobytes()

    def free(self):
        if self._h:
            _lib.lib().zk_params_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PreparedVerifyingKey:
    """bellman_verifier::PreparedVerifyingKey<Bls12> on the device (core/bellman-verifier/src/lib.rs:110-245)."""

    def __init__(self, ctx: Context, handle):
        self.ctx, self._h = ctx, handle
        self.num_inputs = int(_lib.lib().zk_pvk_num_inputs(handle))

    @staticmethod
    def read(ctx: Context, buf: bytes) -> "PreparedVerifyingKey":
        """PreparedVerifyingKey::read — the bytes of zface/params/conf_vk.dat."""
        b = np.frombuffer(buf, np.uint8)
        h = C.c_void_p()
        _ck(_lib.lib().zk_pvk_load(ctx._h, _p(b), len(buf), C.byref(h)))
        return PreparedVerifyingKey(ctx, h)

    @staticmethod
    def prepare(ctx: Context, vk_bytes: bytes) -> "PreparedVerifyingKey":
        """prepare_verifying_key(&vk) (verifier.rs:15-30); vk_bytes = VerifyingKey encoding / head of Parameters::write."""
        b = np.frombuffer(vk_bytes, np.uint8)
        h = C.c_void_p()
        _ck(_lib.lib().zk_pvk_prepare(ctx._h, _p(b), len(vk_bytes), C.byref(h)))
        return PreparedVerifyingKey(ctx, h)

    def write(self) -> bytes:
        out = np.zeros(int(_lib.lib().zk_pvk_size(self._h)), np.uint8)
        _ck(_lib.lib().zk_pvk_write(self._h, _p(out)))
        return out.tobytes()

    def free(self):
        if self._h:
            _lib.lib().zk_pvk_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


VERDICT_OK, VERDICT_FALSE, VERDICT_INVALID_DATA, VERDICT_POINT_INFINITY = 1, 0, 2, 3


def verify_proofs(pvk: PreparedVerifyingKey, proofs: bytes, public_inputs) -> list:
    """Proof::read + verify_proof (verifier.rs:32-63) for len(proofs)/192 proofs; public_inputs: one list of ints per
    proof (without the leading ONE).  Returns the verdict codes of include/zkb200.h; raises
    SynthesisError(MalformedVerifyingKey) when the input count does not match the key."""
    n = len(proofs) // 192
    assert len(proofs) == 192 * n and len(public_inputs) == n
    n_in = len(public_inputs[0]) if n else pvk.num_inputs
    assert all(len(x) == n_in for x in public_inputs)
    inp = _u64([_fr_limbs(v) for row in public_inputs for v in row]) if n * n_in else np.zeros(1, np.uint64)
    pb = np.frombuffer(proofs, np.uint8) if n else np.zeros(1, np.uint8)
    out = np.zeros(max(n, 1), np.uint8)
    _ck(_lib.lib().zk_groth16_verify_batch(pvk.ctx._h, pvk._h, n, _p(pb), _p(inp), n_in, _p(out)))
    return [int(v) for v in out[:n]]


def verify_proof(pvk: PreparedVerifyingKey, proof: bytes, public_inputs) -> bool:
    """verify_proof(pvk, proof, inputs) -> Ok(bool); a proof that Proof::read rejects raises ZkError (io::Error there)."""
    v = verify_proofs(pvk, proof, [list(public_inputs)])[0]
    if v >= 2:
        raise ZkError(-7, "Proof::read: %s" % ("PointInfinity" if v == 3 else "InvalidData"))
    return v == 1


def verify_proofs_device(pvk: PreparedVerifyingKey, n: int, d_proofs_ptr: int, d_inputs_ptr: int, n_inputs: int, d_verdicts_ptr: int):
    _ck(_lib.lib().zk_groth16_verify_batch_device(pvk.ctx._h, pvk._h, n, C.c_void_p(d_proofs_ptr), C.c_void_p(d_inputs_ptr), n_inputs,
                                                  C.c_void_p(d_verdicts_ptr)))


# ---- Jubjub public inputs (modules/zk-system/src/lib.rs:56-165) ---------------------------------------------------------
# zk_jubjub_into_xy status codes: Point::read -> NotInField / NotOnCurve, as_prime_order -> None
JUBJUB_OK, JUBJUB_NOT_IN_FIELD, JUBJUB_NOT_ON_CURVE, JUBJUB_NOT_PRIME_ORDER = 0, 1, 2, 3
VERDICT_INPUT_REJECTED = 4          # a public-input point was rejected (checked before Proof::read, so it wins over 2 / 3)
ANONIMITY_SIZE = 12                 # core/proofs/src/constants.rs:1
CONFIDENTIAL_POINTS, ANONYMOUS_POINTS = 11, 4 * ANONIMITY_SIZE + 4


def jubjub_into_xy(ctx: Context, encodings: bytes):
    """Point::read + as_prime_order + into_xy (core/jubjub/src/curve/edwards.rs:92-164, 319-352) for len/32 encodings.
    Returns (xy uint64 (n, 2, 4): canonical x then y, zero when rejected; status uint8 (n,): JUBJUB_*)."""
    n = len(encodings) // 32
    assert len(encodings) == 32 * n
    xy = np.zeros((max(n, 1), 2, 4), np.uint64)
    st = np.zeros(max(n, 1), np.uint8)
    enc = np.frombuffer(encodings, np.uint8) if n else np.zeros(1, np.uint8)
    _ck(_lib.lib().zk_jubjub_into_xy(ctx._h, n, _p(enc), _p(xy), _p(st)))
    return xy[:n], st[:n]


def verify_proofs_with_points(pvk: PreparedVerifyingKey, proofs: bytes, points: bytes, n_points: int) -> list:
    """verify_confidential_proof / verify_anonymous_proof (lib.rs:56-165) for len(proofs)/192 transactions: each one's public
    inputs are the (x, y) of its n_points 32-byte Jubjub encodings, in PublicInputBuilder push order (confidential_points /
    anonymous_points).  Verdicts as verify_proofs, plus VERDICT_INPUT_REJECTED; raises SynthesisError(MalformedVerifyingKey)
    when 2 * n_points + 1 != ic.len()."""
    n = len(proofs) // 192
    assert len(proofs) == 192 * n and len(points) == 32 * n_points * n
    pb = np.frombuffer(proofs, np.uint8) if n else np.zeros(1, np.uint8)
    pt = np.frombuffer(points, np.uint8) if n * n_points else np.zeros(1, np.uint8)
    out = np.zeros(max(n, 1), np.uint8)
    _ck(_lib.lib().zk_groth16_verify_points_batch(pvk.ctx._h, pvk._h, n, _p(pb), _p(pt), n_points, _p(out)))
    return [int(v) for v in out[:n]]


def verify_proofs_with_points_device(pvk: PreparedVerifyingKey, n: int, d_proofs_ptr: int, d_points_ptr: int, n_points: int,
                                     d_verdicts_ptr: int):
    """The same on device pointers, asynchronous on the context's stream."""
    _ck(_lib.lib().zk_groth16_verify_points_batch_device(pvk.ctx._h, pvk._h, n, C.c_void_p(d_proofs_ptr), C.c_void_p(d_points_ptr),
                                                         n_points, C.c_void_p(d_verdicts_ptr)))


def _pt32(b) -> bytes:
    b = bytes(b)
    assert len(b) == 32, len(b)
    return b


def _ct64(b) -> bytes:
    b = bytes(b)
    assert len(b) == 64, len(b)       # Ciphertext: left point then right point
    return b


def confidential_points(address_sender, address_recipient, amount_sender, amount_recipient, randomness, fee_sender,
                        balance_sender, rvk, g_epoch, nonce) -> bytes:
    """The 11 points verify_confidential_proof pushes (lib.rs:69-100), in its order: randomness goes before fee_sender, and
    the 64-byte balance_sender ciphertext contributes its left, then its right point.  352 bytes."""
    return b"".join([_pt32(address_sender), _pt32(address_recipient), _pt32(amount_sender), _pt32(amount_recipient),
                     _pt32(randomness), _pt32(fee_sender), _ct64(balance_sender), _pt32(rvk), _pt32(g_epoch), _pt32(nonce)])


def anonymous_points(enc_keys, left_ciphertexts, enc_balances, right_ciphertext, rvk, g_epoch, nonce) -> bytes:
    """The 52 points verify_anonymous_proof pushes (lib.rs:128-153): 12 encryption keys, 12 left ciphertexts, the left points
    of the 12 balance ciphertexts, then their right points, then right_ciphertext, rvk, g_epoch, nonce.  1664 bytes."""
    assert len(enc_keys) == len(left_ciphertexts) == len(enc_balances) == ANONIMITY_SIZE
    bal = [_ct64(c) for c in enc_balances]
    return b"".join([_pt32(k) for k in enc_keys] + [_pt32(c) for c in left_ciphertexts] + [c[:32] for c in bal] +
                    [c[32:] for c in bal] + [_pt32(right_ciphertext), _pt32(rvk), _pt32(g_epoch), _pt32(nonce)])


# ---- RedJubjub transaction signatures (core/primitives/src/signature.rs:65-82) ------------------------------------------
# zk_redjubjub_verify_batch verdicts; every value but REDJUBJUB_OK is the reference's `false`
REDJUBJUB_BAD_EQUATION, REDJUBJUB_OK, REDJUBJUB_BAD_VK, REDJUBJUB_BAD_R, REDJUBJUB_BAD_S = 0, 1, 2, 3, 4


def _cat(items, size: int) -> bytes:
    b = bytes(items) if isinstance(items, (bytes, bytearray, memoryview)) else b"".join(bytes(x) for x in items)
    assert len(b) % size == 0, len(b)
    return b


def message_offsets(msgs) -> np.ndarray:
    """The n + 1 offsets of the concatenated messages (uint64)."""
    off = np.zeros(len(msgs) + 1, np.uint64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    return off


def redjubjub_verify(ctx: Context, vks, sigs, msgs) -> list:
    """PublicKey::verify(msg, sig, FixedGenerators::Diversifier) (core/jubjub/src/redjubjub.rs:127-155) for each signature.
    vks: 32-byte keys, sigs: 64-byte signatures (rbar | sbar), each a list or one concatenation; msgs: a list of byte strings.
    Returns the REDJUBJUB_* verdict of each."""
    vk, sg = _cat(vks, 32), _cat(sigs, 64)
    n = len(msgs)
    assert len(vk) == 32 * n and len(sg) == 64 * n
    mb = b"".join(bytes(m) for m in msgs)
    out = np.zeros(max(n, 1), np.uint8)
    off = message_offsets(msgs)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    _ck(_lib.lib().zk_redjubjub_verify_batch(ctx._h, n, _p(buf(vk)), _p(buf(sg)), _p(buf(mb)), _p(off), _p(out)))
    return [int(v) for v in out[:n]]


def redjubjub_verify_device(ctx: Context, n: int, d_vks_ptr: int, d_sigs_ptr: int, d_msgs_ptr: int, d_msg_off_ptr: int,
                            d_verdicts_ptr: int):
    """The same on device pointers (d_msg_off: n + 1 uint64 offsets), asynchronous on the context's stream."""
    _ck(_lib.lib().zk_redjubjub_verify_batch_device(ctx._h, n, C.c_void_p(d_vks_ptr), C.c_void_p(d_sigs_ptr), C.c_void_p(d_msgs_ptr),
                                                    C.c_void_p(d_msg_off_ptr), C.c_void_p(d_verdicts_ptr)))


# zk_redjubjub_batch_verify_device only: some z_i >= r_J (the host form raises ZK_ERR_NOT_CANONICAL instead)
REDJUBJUB_BAD_Z = 5


def jubjub_msm(ctx: Context, points, scalars) -> bytes:
    """sum_i scalars[i] P_i over Jubjub (edwards::Point<Unknown>): points are 32-byte Point::write encodings, read without a
    subgroup test; scalars are 32-byte little-endian Fs values < r_J (or ints).  Returns the 32-byte encoding of the sum."""
    pt = _cat(points, 32)
    if not isinstance(scalars, (bytes, bytearray, memoryview)):
        scalars = [s.to_bytes(32, "little") if isinstance(s, int) else s for s in scalars]
    sc = _cat(scalars, 32)
    n = len(pt) // 32
    assert len(sc) == 32 * n
    out = np.zeros(32, np.uint8)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    _ck(_lib.lib().zk_jubjub_msm(ctx._h, n, _p(buf(pt)), _p(buf(sc)), _p(out)))
    return out.tobytes()


def random_batch_scalars(n: int) -> bytes:
    """n uniform Fs values from the operating system's CSPRNG (E::Fs::rand), 32 bytes each: the z_i of a batch check."""
    r_j = 0x0e7db4ea6533afa906673b0101343b00a6682093ccc81082d0970e5ed6f72cb7
    return b"".join((int.from_bytes(secrets.token_bytes(64), "little") % r_j).to_bytes(32, "little") for _ in range(n))


def redjubjub_batch_verify(ctx: Context, vks, sigs, msgs, zs=None):
    """redjubjub::batch_verify(rng, batch, FixedGenerators::Diversifier) (core/jubjub/src/redjubjub.rs:166-204) with the
    randomizers zs (32-byte canonical Fs each, or one concatenation; None draws them with random_batch_scalars).
    Returns (verdict, first_bad): verdict 1 when the batch passes, 0 when the combined equation fails, or the
    REDJUBJUB_BAD_VK / _R / _S code of the lowest rejected entry, whose index is first_bad (None otherwise)."""
    vk, sg = _cat(vks, 32), _cat(sigs, 64)
    n = len(msgs)
    assert len(vk) == 32 * n and len(sg) == 64 * n
    z = random_batch_scalars(n) if zs is None else _cat(zs, 32)
    assert len(z) == 32 * n
    mb = b"".join(bytes(m) for m in msgs)
    off = message_offsets(msgs)
    verdict = np.zeros(1, np.uint8)
    first = np.zeros(1, np.uint64)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    _ck(_lib.lib().zk_redjubjub_batch_verify(ctx._h, n, _p(buf(vk)), _p(buf(sg)), _p(buf(mb)), _p(off), _p(buf(z)), _p(verdict), _p(first)))
    v = int(verdict[0])
    return v, (int(first[0]) if v not in (REDJUBJUB_OK, REDJUBJUB_BAD_EQUATION) else None)


def redjubjub_batch_verify_device(ctx: Context, n: int, d_vks_ptr: int, d_sigs_ptr: int, d_msgs_ptr: int, d_msg_off_ptr: int,
                                  d_zs_ptr: int, d_verdict_ptr: int, d_first_bad_ptr: int = 0):
    """The same on device pointers (d_msg_off: n + 1 uint64 offsets; d_zs: n * 32 bytes; d_verdict: one byte; d_first_bad:
    one uint64 or 0), asynchronous on the context's stream."""
    _ck(_lib.lib().zk_redjubjub_batch_verify_device(ctx._h, n, C.c_void_p(d_vks_ptr), C.c_void_p(d_sigs_ptr), C.c_void_p(d_msgs_ptr),
                                                    C.c_void_p(d_msg_off_ptr), C.c_void_p(d_zs_ptr), C.c_void_p(d_verdict_ptr),
                                                    C.c_void_p(d_first_bad_ptr) if d_first_bad_ptr else None))


def redjubjub_verify_batched(ctx: Context, vks, sigs, msgs, zs=None) -> list:
    """Per-signature verdicts, as redjubjub_verify returns them, through one batch check first: when the batch passes every
    verdict is REDJUBJUB_OK, otherwise redjubjub_verify decides each signature.  The one difference from redjubjub_verify
    is the reference's own soundness error: a batch with a bad signature passes with probability ~1 / r_J over the draw of
    zs, so zs must be unpredictable to the signers (None draws them with random_batch_scalars)."""
    n = len(msgs)
    verdict, _ = redjubjub_batch_verify(ctx, vks, sigs, msgs, zs)
    if verdict == REDJUBJUB_OK:
        return [REDJUBJUB_OK] * n
    return redjubjub_verify(ctx, vks, sigs, msgs)


# ---- lifted-ElGamal balance decryption (core/crypto/src/elgamal.rs:87-136, zface/src/utils/getter.rs:135-175) ------------
# zk_elgamal_decrypt_batch statuses: Some(value), None, DecryptionKey::read fails, Ciphertext::read of the balance / of the
# pending transfer fails
ELGAMAL_OK, ELGAMAL_NOT_FOUND, ELGAMAL_BAD_KEY, ELGAMAL_BAD_BALANCE, ELGAMAL_BAD_PENDING = 0, 1, 2, 3, 4
ELGAMAL_BOUND = 1_000_000                          # the reference's search range, elgamal.rs:102
ELGAMAL_ZERO = (b"\x01" + bytes(31)) * 2           # Ciphertext::zero(): two identities, what zface uses for an empty slot


def elgamal_decrypt(ctx: Context, dks, cts, pending=None):
    """Ciphertext::decrypt(dk, FixedGenerators::Diversifier) of each ciphertext, after adding its pending transfer if
    `pending` is given.  dks: 32-byte keys, cts / pending: 64-byte ciphertexts, each a list or one concatenation.
    Returns (statuses, values): the ELGAMAL_* status of each, and its amount (0 unless the status is ELGAMAL_OK)."""
    dk, ct = _cat(dks, 32), _cat(cts, 64)
    n = len(dk) // 32
    assert len(ct) == 64 * n
    pd = None if pending is None else _cat(pending, 64)
    assert pd is None or len(pd) == 64 * n
    values = np.zeros(max(n, 1), np.uint32)
    st = np.zeros(max(n, 1), np.uint8)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    _ck(_lib.lib().zk_elgamal_decrypt_batch(ctx._h, n, _p(buf(dk)), _p(buf(ct)), None if pd is None else _p(buf(pd)), _p(values), _p(st)))
    return [int(s) for s in st[:n]], [int(v) for v in values[:n]]


def elgamal_decrypt_device(ctx: Context, n: int, d_dks_ptr: int, d_cts_ptr: int, d_pending_ptr: int, d_values_ptr: int,
                           d_status_ptr: int):
    """The same on device pointers (d_pending = 0: no pending transfers; d_values: n uint32), asynchronous on the context's
    stream."""
    _ck(_lib.lib().zk_elgamal_decrypt_batch_device(ctx._h, n, C.c_void_p(d_dks_ptr), C.c_void_p(d_cts_ptr),
                                                   C.c_void_p(d_pending_ptr) if d_pending_ptr else None, C.c_void_p(d_values_ptr),
                                                   C.c_void_p(d_status_ptr)))


# ---- building confidential transfers (zface's gen_proof / gen_xt around the proof) ----------------------------------------
# zk_confidential_fields_batch: the 9 points of a row in ConfidentialTx's constructor order
CONFIDENTIAL_FIELDS = ("address_sender", "address_recipient", "amount_sender", "amount_recipient", "fee_sender", "randomness", "rvk",
                       "g_epoch", "nonce")


def _buf(b: bytes):
    return np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)


def _scalars(v, n: int) -> bytes:
    """n 32-byte little-endian scalars from ints or byte strings (or one concatenation)"""
    if not isinstance(v, (bytes, bytearray, memoryview)):
        v = [s.to_bytes(32, "little") if isinstance(s, int) else s for s in v]
    b = _cat(v, 32)
    assert len(b) == 32 * n, (len(b), n)
    return b


def _rows(out: np.ndarray, size: int, n: int) -> list:
    return [out[size * i:size * (i + 1)].tobytes() for i in range(n)]


def keys_from_seed(ctx: Context, seeds):
    """SpendingKey::from_seed -> DecryptionKey -> EncryptionKey (core/keys/src/lib.rs) of each seed (byte strings of any
    length).  Returns (sks, dks, eks): lists of 32-byte values."""
    n = len(seeds)
    sk, dk, ek = (np.zeros(max(32 * n, 1), np.uint8) for _ in range(3))
    _ck(_lib.lib().zk_keys_from_seed_batch(ctx._h, n, _p(_buf(b"".join(bytes(s) for s in seeds))), _p(message_offsets(seeds)), _p(sk), _p(dk),
                                           _p(ek)))
    return _rows(sk, 32, n), _rows(dk, 32, n), _rows(ek, 32, n)


def keys_from_seed_device(ctx: Context, n: int, d_seeds_ptr: int, d_seed_off_ptr: int, d_sks_ptr: int, d_dks_ptr: int, d_eks_ptr: int):
    """The same on device pointers (d_seed_off: n + 1 uint64 offsets), asynchronous on the context's stream."""
    _ck(_lib.lib().zk_keys_from_seed_batch_device(ctx._h, n, C.c_void_p(d_seeds_ptr), C.c_void_p(d_seed_off_ptr), C.c_void_p(d_sks_ptr),
                                                  C.c_void_p(d_dks_ptr), C.c_void_p(d_eks_ptr)))


def g_epoch(ctx: Context, epochs) -> list:
    """GEpoch::group_hash(epoch) (core/primitives/src/g_epoch.rs:102-145) of each epoch: a list of 32-byte encodings."""
    n = len(epochs)
    ep = np.ascontiguousarray(epochs, np.uint32) if n else np.zeros(1, np.uint32)
    out = np.zeros(max(32 * n, 1), np.uint8)
    _ck(_lib.lib().zk_g_epoch_batch(ctx._h, n, _p(ep), _p(out)))
    return _rows(out, 32, n)


def g_epoch_device(ctx: Context, n: int, d_epochs_ptr: int, d_g_epochs_ptr: int):
    """The same on device pointers (d_epochs: n uint32), asynchronous on the context's stream."""
    _ck(_lib.lib().zk_g_epoch_batch_device(ctx._h, n, C.c_void_p(d_epochs_ptr), C.c_void_p(d_g_epochs_ptr)))


def confidential_fields(ctx: Context, sks, eks_recipient, amounts, fees, rs, alphas, g_epoch_enc):
    """The ciphertexts, rvk and nonce of n confidential transfers (MultiCiphertexts::<Confidential>::encrypt and ProofContext):
    sks / rs / alphas are scalars < r_J (ints or 32 bytes), eks_recipient 32-byte keys, amounts / fees uint32, g_epoch_enc
    the call's 32-byte g_epoch.  Returns (fields, rsks, dks, status): fields[i] is a dict of the CONFIDENTIAL_FIELDS
    (ConfidentialTx(sender, recipient, **fields[i]) builds the extrinsic), rsks / dks 32-byte values, status the
    zk_jubjub_into_xy code of each recipient key (0: ok; otherwise the row is zero)."""
    n = len(amounts)
    sk, r, al = _scalars(sks, n), _scalars(rs, n), _scalars(alphas, n)
    ek = _cat(eks_recipient, 32)
    assert len(ek) == 32 * n and len(fees) == n
    am = np.ascontiguousarray(amounts, np.uint32) if n else np.zeros(1, np.uint32)
    fe = np.ascontiguousarray(fees, np.uint32) if n else np.zeros(1, np.uint32)
    f = np.zeros(max(288 * n, 1), np.uint8)
    rsk, dk, st = np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    _ck(_lib.lib().zk_confidential_fields_batch(ctx._h, n, _p(_buf(sk)), _p(_buf(ek)), _p(am), _p(fe), _p(_buf(r)), _p(_buf(al)),
                                                _p(_buf(_pt32(g_epoch_enc))), _p(f), _p(rsk), _p(dk), _p(st)))
    fields = [dict(zip(CONFIDENTIAL_FIELDS, _rows(f[288 * i:288 * (i + 1)], 32, 9))) for i in range(n)]
    return fields, _rows(rsk, 32, n), _rows(dk, 32, n), [int(s) for s in st[:n]]


def confidential_fields_device(ctx: Context, n: int, d_sks_ptr: int, d_eks_recipient_ptr: int, d_amounts_ptr: int, d_fees_ptr: int,
                               d_rs_ptr: int, d_alphas_ptr: int, d_g_epoch_ptr: int, d_fields_ptr: int, d_rsks_ptr: int, d_dks_ptr: int,
                               d_status_ptr: int):
    """The same on device pointers (d_amounts / d_fees: n uint32; d_fields: n * 288 bytes), asynchronous on the context's
    stream; ctx.sync() raises ZK_ERR_NOT_CANONICAL or ZK_ERR_DECODE (g_epoch)."""
    _ck(_lib.lib().zk_confidential_fields_batch_device(ctx._h, n, *(C.c_void_p(p) for p in (
        d_sks_ptr, d_eks_recipient_ptr, d_amounts_ptr, d_fees_ptr, d_rs_ptr, d_alphas_ptr, d_g_epoch_ptr, d_fields_ptr, d_rsks_ptr,
        d_dks_ptr, d_status_ptr))))


# zk_anonymous_fields_batch: the 27 points of a row, enc_keys and left_ciphertexts 12 each, in AnonymousTx's argument order
ANONYMOUS_FIELDS = ("enc_keys", "left_ciphertexts", "right_ciphertext", "rvk", "nonce")
ANON_BAD_INDEX, ANON_BAD_POSITIONS = 4, 5     # zk_anonymous_fields_batch statuses besides the zk_jubjub_into_xy codes


def anonymous_fields(ctx: Context, keys, sks, rings, positions, amounts, rs, alphas, g_epoch_enc):
    """The ciphertexts, rvk and nonce of n anonymous transfers (MultiCiphertexts::<Anonymous>::encrypt in gen_proof's ring
    order, and ProofContext): keys the table of 32-byte encryption keys the rings index; sks / rs / alphas scalars < r_J
    (ints or 32 bytes); rings n rows of 11 indices (recipient, then the ten decoys); positions n pairs (s_index, t_index);
    amounts uint32; g_epoch_enc the call's 32-byte g_epoch.  Returns (fields, rsks, dks, status): fields[i] is a dict of
    the ANONYMOUS_FIELDS, enc_keys and left_ciphertexts lists of 12 (AnonymousTx(members, fields[i]["left_ciphertexts"],
    ...) builds the extrinsic, members being the accounts of enc_keys); rsks / dks 32-byte values; status 0, a
    zk_jubjub_into_xy code, ANON_BAD_INDEX or ANON_BAD_POSITIONS (non-zero: the row is zero)."""
    n = len(amounts)
    ky = _cat(keys, 32)
    sk, r, al = _scalars(sks, n), _scalars(rs, n), _scalars(alphas, n)
    rg = np.ascontiguousarray(np.asarray(rings, np.int64).reshape(-1).astype(np.uint32)) if n else np.zeros(1, np.uint32)
    pos = np.ascontiguousarray(np.asarray(positions, np.int64).reshape(-1).astype(np.uint8)) if n else np.zeros(1, np.uint8)
    assert (len(rg) == 11 * n and len(pos) == 2 * n) or not n
    am = np.ascontiguousarray(amounts, np.uint32) if n else np.zeros(1, np.uint32)
    f = np.zeros(max(864 * n, 1), np.uint8)
    rsk, dk, st = np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(32 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    _ck(_lib.lib().zk_anonymous_fields_batch(ctx._h, len(ky) // 32, _p(_buf(ky)), n, _p(_buf(sk)), _p(rg), _p(pos), _p(am), _p(_buf(r)),
                                             _p(_buf(al)), _p(_buf(_pt32(g_epoch_enc))), _p(f), _p(rsk), _p(dk), _p(st)))
    fields = []
    for i in range(n):
        pts = _rows(f[864 * i:864 * (i + 1)], 32, 27)
        fields.append(dict(zip(ANONYMOUS_FIELDS, [pts[:12], pts[12:24], pts[24], pts[25], pts[26]])))
    return fields, _rows(rsk, 32, n), _rows(dk, 32, n), [int(s) for s in st[:n]]


def anonymous_fields_device(ctx: Context, n_keys: int, d_keys_ptr: int, n: int, d_sks_ptr: int, d_rings_ptr: int, d_positions_ptr: int,
                            d_amounts_ptr: int, d_rs_ptr: int, d_alphas_ptr: int, d_g_epoch_ptr: int, d_fields_ptr: int, d_rsks_ptr: int,
                            d_dks_ptr: int, d_status_ptr: int):
    """The same on device pointers (d_keys: n_keys * 32 bytes, 0 when n_keys = 0; d_rings: n * 11 uint32; d_positions:
    n * 2 bytes; d_amounts: n uint32; d_fields: n * 864 bytes), asynchronous on the context's stream; ctx.sync() raises
    ZK_ERR_NOT_CANONICAL or ZK_ERR_DECODE (g_epoch)."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_anonymous_fields_batch_device(ctx._h, n_keys, v(d_keys_ptr), n, *(v(p) for p in (
        d_sks_ptr, d_rings_ptr, d_positions_ptr, d_amounts_ptr, d_rs_ptr, d_alphas_ptr, d_g_epoch_ptr, d_fields_ptr, d_rsks_ptr, d_dks_ptr,
        d_status_ptr))))


def redjubjub_sign(ctx: Context, sks, msgs, ts) -> list:
    """PrivateKey::sign(msg, rng, FixedGenerators::Diversifier) (core/jubjub/src/redjubjub.rs:73-103) of each message, with
    the 80 bytes ts[i] in place of the RNG's output (draw them with secrets.token_bytes(80)).  sks: scalars < r_J (ints or
    32 bytes).  Returns the 64-byte signatures (rbar | sbar)."""
    n = len(msgs)
    sk, t = _scalars(sks, n), _cat(ts, 80)
    assert len(t) == 80 * n
    out = np.zeros(max(64 * n, 1), np.uint8)
    _ck(_lib.lib().zk_redjubjub_sign_batch(ctx._h, n, _p(_buf(sk)), _p(_buf(t)), _p(_buf(b"".join(bytes(m) for m in msgs))),
                                           _p(message_offsets(msgs)), _p(out)))
    return _rows(out, 64, n)


def redjubjub_sign_device(ctx: Context, n: int, d_sks_ptr: int, d_ts_ptr: int, d_msgs_ptr: int, d_msg_off_ptr: int, d_sigs_ptr: int):
    """The same on device pointers (d_ts: n * 80 bytes; d_msg_off: n + 1 uint64 offsets), asynchronous on the context's
    stream."""
    _ck(_lib.lib().zk_redjubjub_sign_batch_device(ctx._h, n, C.c_void_p(d_sks_ptr), C.c_void_p(d_ts_ptr), C.c_void_p(d_msgs_ptr),
                                                  C.c_void_p(d_msg_off_ptr), C.c_void_p(d_sigs_ptr)))


# ---- wallet keys: zface's hierarchical key derivation (zface/src/derive/mod.rs) ----------------------------------------
# An extended key is 73 opaque bytes (ExtendedSpendingKey / ExtendedProofGenerationKey::write); child indices are raw u32,
# HD_HARDENED and above hardened.  Row statuses of the derive calls besides the zk_jubjub_into_xy codes:
XK_BYTES = 73
HD_HARDENED = 1 << 31
HD_BAD_INDEX, HD_HARDENED_INDEX, HD_DEPTH = 4, 5, 6


def _idx32(v, n: int, what: str):
    """n raw u32 indices; a value outside 0 .. 2^32 - 1 is refused, not wrapped (-1 would become a hardened index)"""
    if not n:
        return np.zeros(1, np.uint32)
    a = [int(x) for x in np.asarray(v, dtype=object).reshape(-1)]
    if len(a) != n:
        raise ValueError("%s: %d values for %d rows" % (what, len(a), n))
    bad = next((i for i, x in enumerate(a) if not 0 <= x < 1 << 32), None)
    if bad is not None:
        raise ValueError("%s[%d] = %d is not a u32" % (what, bad, a[bad]))
    return np.ascontiguousarray(np.array(a, np.uint64).astype(np.uint32))


def _opt(want: bool, size: int, n: int):
    return np.zeros(max(size * n, 1), np.uint8) if want else None


def _opt_rows(out, size: int, n: int):
    return _rows(out, size, n) if out is not None else None


def _dptr(p: int):
    return C.c_void_p(p) if p else None


def xsk_master(ctx: Context, seeds, xpgk: bool = True, dk: bool = True, ek: bool = True):
    """ExtendedSpendingKey::master(seed) of each seed (byte strings of any length, e.g. a bip39 seed) — what zface's
    `wallet init` / `recover` build.  Returns (xsks, xpgks, dks, eks): xsks 73-byte extended spending keys; xpgks their
    ExtendedProofGenerationKeys (73 bytes), dks / eks the master account's decryption and encryption keys (32 bytes), each
    list None when not asked for."""
    n = len(seeds)
    xsk, xp, d, e = np.zeros(max(XK_BYTES * n, 1), np.uint8), _opt(xpgk, XK_BYTES, n), _opt(dk, 32, n), _opt(ek, 32, n)
    _ck(_lib.lib().zk_xsk_master_batch(ctx._h, n, _p(_buf(b"".join(bytes(s) for s in seeds))), _p(message_offsets(seeds)), _p(xsk),
                                       *(_p(a) if a is not None else None for a in (xp, d, e))))
    return _rows(xsk, XK_BYTES, n), _opt_rows(xp, XK_BYTES, n), _opt_rows(d, 32, n), _opt_rows(e, 32, n)


def xsk_master_device(ctx: Context, n: int, d_seeds_ptr: int, d_seed_off_ptr: int, d_xsks_ptr: int, d_xpgks_ptr: int = 0,
                      d_dks_ptr: int = 0, d_eks_ptr: int = 0):
    """The same on device pointers (d_seed_off: n + 1 uint64 offsets; 0 for an output not wanted), asynchronous on the
    context's stream."""
    _ck(_lib.lib().zk_xsk_master_batch_device(ctx._h, n, *(_dptr(p) for p in (d_seeds_ptr, d_seed_off_ptr, d_xsks_ptr, d_xpgks_ptr, d_dks_ptr,
                                                                                d_eks_ptr))))


def xsk_derive(ctx: Context, parents, parent_idx, child_idx, xpgk: bool = True, dk: bool = True, ek: bool = True):
    """ExtendedSpendingKey::derive_child: row i derives child child_idx[i] (a raw u32, >= HD_HARDENED hardened) of
    parents[parent_idx[i]], parents being 73-byte xsks (a list, or their concatenation).  Account k of a wallet is
    xsk_derive(ctx, [master], [0], [k]).  Returns (xsks, xpgks, dks, eks, status): as xsk_master, and status 0,
    HD_BAD_INDEX or HD_DEPTH per row (non-zero: the row is zero).  Raises ZK_ERR_NOT_CANONICAL naming the parent when a
    named parent's sk >= r_J."""
    pb = _cat(parents, XK_BYTES)
    n = len(parent_idx)
    pi, ci = _idx32(parent_idx, n, "parent_idx"), _idx32(child_idx, n, "child_idx")
    xsk, st = np.zeros(max(XK_BYTES * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    xp, d, e = _opt(xpgk, XK_BYTES, n), _opt(dk, 32, n), _opt(ek, 32, n)
    _ck(_lib.lib().zk_xsk_derive_batch(ctx._h, len(pb) // XK_BYTES, _p(_buf(pb)), n, _p(pi), _p(ci), _p(xsk),
                                       *(_p(a) if a is not None else None for a in (xp, d, e)), _p(st)))
    return _rows(xsk, XK_BYTES, n), _opt_rows(xp, XK_BYTES, n), _opt_rows(d, 32, n), _opt_rows(e, 32, n), [int(s) for s in st[:n]]


def xsk_derive_device(ctx: Context, n_parents: int, d_parents_ptr: int, n: int, d_parent_idx_ptr: int, d_child_idx_ptr: int,
                      d_xsks_ptr: int, d_xpgks_ptr: int, d_dks_ptr: int, d_eks_ptr: int, d_status_ptr: int):
    """The same on device pointers (d_parents: n_parents * 73 bytes; d_parent_idx / d_child_idx: n uint32; 0 for an output
    not wanted), asynchronous on the context's stream; ctx.sync() raises ZK_ERR_NOT_CANONICAL for a named parent whose
    sk >= r_J, whose rows are left unwritten.  A path chains calls, each level's d_xsks the next level's d_parents; no
    output may overlap d_parents."""
    _ck(_lib.lib().zk_xsk_derive_batch_device(ctx._h, n_parents, _dptr(d_parents_ptr), n, *(_dptr(p) for p in (
        d_parent_idx_ptr, d_child_idx_ptr, d_xsks_ptr, d_xpgks_ptr, d_dks_ptr, d_eks_ptr, d_status_ptr))))


def xpgk_derive(ctx: Context, parents, parent_idx, child_idx, dk: bool = True, ek: bool = True):
    """ExtendedProofGenerationKey::derive_child, the watch-only derivation: as xsk_derive over 73-byte xpgk parents, with
    no spending key.  Returns (xpgks, dks, eks, status): status 0; HD_BAD_INDEX; the zk_jubjub_into_xy code (1 / 2 / 3)
    of a parent whose pgk fails ProofGenerationKey::read; HD_HARDENED_INDEX; or HD_DEPTH (non-zero: the row is zero).
    The dks decrypt the derived accounts' balances with elgamal_decrypt."""
    pb = _cat(parents, XK_BYTES)
    n = len(parent_idx)
    pi, ci = _idx32(parent_idx, n, "parent_idx"), _idx32(child_idx, n, "child_idx")
    xp, st = np.zeros(max(XK_BYTES * n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
    d, e = _opt(dk, 32, n), _opt(ek, 32, n)
    _ck(_lib.lib().zk_xpgk_derive_batch(ctx._h, len(pb) // XK_BYTES, _p(_buf(pb)), n, _p(pi), _p(ci), _p(xp),
                                        *(_p(a) if a is not None else None for a in (d, e)), _p(st)))
    return _rows(xp, XK_BYTES, n), _opt_rows(d, 32, n), _opt_rows(e, 32, n), [int(s) for s in st[:n]]


def xpgk_derive_device(ctx: Context, n_parents: int, d_parents_ptr: int, n: int, d_parent_idx_ptr: int, d_child_idx_ptr: int,
                       d_xpgks_ptr: int, d_dks_ptr: int, d_eks_ptr: int, d_status_ptr: int):
    """The same on device pointers, as xsk_derive_device; asynchronous on the context's stream."""
    _ck(_lib.lib().zk_xpgk_derive_batch_device(ctx._h, n_parents, _dptr(d_parents_ptr), n, *(_dptr(p) for p in (
        d_parent_idx_ptr, d_child_idx_ptr, d_xpgks_ptr, d_dks_ptr, d_eks_ptr, d_status_ptr))))


# ---- confidential-transfer balance updates of one block (modules/encrypted-balances/src/lib.rs:25-96, 133-222) ----------
# account flags and zk_balances_confidential_block statuses
ACCOUNT_BALANCE, ACCOUNT_PENDING, ACCOUNT_DUE = 1, 2, 4
BLOCK_APPLIED, BLOCK_NOT_APPLIED, BLOCK_BAD_POINT, BLOCK_BAD_INDEX = 0, 1, 2, 3


def confidential_block(ctx: Context, balances, pendings, flags, sender, recipient, tx_points, applied):
    """rollover + sub_enc_balance + add_pending_transfer over a block, in order (zk_balances_confidential_block).
    balances / pendings: 64 bytes per account; flags: one ACCOUNT_* byte per account; sender / recipient: account indices;
    tx_points: 128 bytes per transaction (amount_sender | amount_recipient | fee_sender | randomness); applied: one byte per
    transaction.  Returns (balance_sender, balance_after, status, new_balances, new_pendings, new_flags) as bytes;
    balance_after is zero for transactions that are not applied.  Raises SynthesisError(ZK_ERR_DECODE) naming the account
    when a touched account's stored ciphertext does not read."""
    n_acct, n_tx = len(flags), len(sender)
    bal, pend, fl, tp, ap = (_cat(balances, 64), _cat(pendings, 64), bytes(flags), _cat(tx_points, 128), bytes(applied))
    assert len(bal) == len(pend) == 64 * n_acct and len(recipient) == n_tx and len(tp) == 128 * n_tx and len(ap) == n_tx
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    idx = lambda v: np.ascontiguousarray(v, np.uint32) if n_tx else np.zeros(1, np.uint32)
    bs, ba = np.zeros(max(64 * n_tx, 1), np.uint8), np.zeros(max(64 * n_tx, 1), np.uint8)
    st = np.zeros(max(n_tx, 1), np.uint8)
    nb, npd = np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(64 * n_acct, 1), np.uint8)
    nf = np.zeros(max(n_acct, 1), np.uint8)
    _ck(_lib.lib().zk_balances_confidential_block(ctx._h, n_acct, _p(buf(bal)), _p(buf(pend)), _p(buf(fl)), n_tx, _p(idx(sender)),
                                                  _p(idx(recipient)), _p(buf(tp)), _p(buf(ap)), _p(bs), _p(ba), _p(st), _p(nb), _p(npd), _p(nf)))
    return (bs[:64 * n_tx].tobytes(), ba[:64 * n_tx].tobytes(), st[:n_tx].tobytes(), nb[:64 * n_acct].tobytes(),
            npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())


def confidential_block_device(ctx: Context, n_accounts: int, d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int, n_tx: int,
                              d_sender_ptr: int, d_recipient_ptr: int, d_tx_points_ptr: int, d_applied_ptr: int,
                              d_balance_sender_ptr: int, d_balance_after_ptr: int, d_status_ptr: int, d_new_balances_ptr: int,
                              d_new_pendings_ptr: int, d_new_flags_ptr: int):
    """The same on device pointers (d_sender / d_recipient: uint32), asynchronous on the context's stream; ctx.sync()
    raises SynthesisError(ZK_ERR_DECODE) naming a touched account whose stored ciphertext did not read.  Only the applied
    transactions' entries of d_balance_after are written."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_balances_confidential_block_device(ctx._h, n_accounts, v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr), n_tx,
                                                         v(d_sender_ptr), v(d_recipient_ptr), v(d_tx_points_ptr), v(d_applied_ptr),
                                                         v(d_balance_sender_ptr), v(d_balance_after_ptr), v(d_status_ptr),
                                                         v(d_new_balances_ptr), v(d_new_pendings_ptr), v(d_new_flags_ptr)))


class ConfidentialTx:
    """One confidential_transfer extrinsic (lib.rs:25-35) with its accounts as indices into the block's account table."""

    def __init__(self, sender: int, recipient: int, address_sender, address_recipient, amount_sender, amount_recipient, fee_sender,
                 randomness, rvk, g_epoch, nonce):
        self.sender, self.recipient = sender, recipient
        self.address_sender, self.address_recipient = _pt32(address_sender), _pt32(address_recipient)
        self.amount_sender, self.amount_recipient = _pt32(amount_sender), _pt32(amount_recipient)
        self.fee_sender, self.randomness = _pt32(fee_sender), _pt32(randomness)
        self.rvk, self.g_epoch, self.nonce = _pt32(rvk), _pt32(g_epoch), _pt32(nonce)

    def points(self) -> bytes:
        return self.amount_sender + self.amount_recipient + self.fee_sender + self.randomness


def import_confidential_block(ctx: Context, pvk: PreparedVerifyingKey, accounts, txs, proofs):
    """Verify and apply a block of confidential transfers the way the runtime does, one extrinsic after another, with the
    state and the proofs of the whole block on the device.  accounts = (balances, pendings, flags) as confidential_block
    takes them; txs: ConfidentialTx list; proofs: 192 bytes each.

    A proof is checked against the sender's balance as it stands at its transaction, which depends on which of the
    sender's earlier transactions passed.  So every transaction starts as applied, and each round computes the balances
    (confidential_block), verifies the undecided transactions (verify_proofs_with_points), and decides, in each sender's
    chain, the transactions up to and including the first whose verdict is not 1: their balances were exact.  The rest
    waits for the next round.  A block takes 1 + (the most failures in one sender's chain) rounds at most; a block with
    no failures takes one.

    Returns (verdicts, (new_balances, new_pendings, new_flags), balance_after, rounds): the reference's verdict per
    transaction (1 passes; the other values as verify_proofs_with_points).  Raises ValueError for an account index out of
    range, SynthesisError(ZK_ERR_DECODE) for a touched account whose stored ciphertext does not read."""
    balances, pendings, flags = accounts
    n = len(txs)
    if any(not (0 <= t.sender < len(flags) and 0 <= t.recipient < len(flags)) for t in txs):
        raise ValueError("import_confidential_block: account index out of range")
    proofs = _cat(proofs, 192)
    assert len(proofs) == 192 * n
    sender = np.array([t.sender for t in txs], np.uint32)
    recipient = np.array([t.recipient for t in txs], np.uint32)
    # every transaction's public-input points in confidential_points order; columns 6-7 (balance_sender) are filled per round
    inputs = np.frombuffer(b"".join(t.address_sender + t.address_recipient + t.amount_sender + t.amount_recipient + t.randomness +
                                    t.fee_sender + bytes(64) + t.rvk + t.g_epoch + t.nonce for t in txs), np.uint8)
    inputs = inputs.reshape(n, CONFIDENTIAL_POINTS, 32).copy()
    tx_points = inputs[:, [2, 3, 5, 4], :].tobytes()          # amount_sender | amount_recipient | fee_sender | randomness
    proof_rows = np.frombuffer(proofs, np.uint8).reshape(n, 192)
    verdicts = np.full(n, -1, np.int16)                      # -1: undecided
    chains = None
    rounds = 0
    while True:
        out = confidential_block(ctx, balances, pendings, flags, sender, recipient, tx_points,
                                 ((verdicts == -1) | (verdicts == 1)).astype(np.uint8).tobytes())
        undecided = np.flatnonzero(verdicts == -1)
        if not len(undecided):
            break
        rounds += 1
        inputs[:, 6:8, :] = np.frombuffer(out[0], np.uint8).reshape(n, 2, 32)
        sel = slice(None) if len(undecided) == n else undecided
        got = np.array(verify_proofs_with_points(pvk, proof_rows[sel].tobytes(), inputs[sel].tobytes(), CONFIDENTIAL_POINTS), np.int16)
        if (got == 1).all():
            verdicts[undecided] = 1
            break                   # every balance of this round was exact: out is the final state
        if chains is None:
            chains = {}
            for k, s in enumerate(sender.tolist()):
                chains.setdefault(s, []).append(k)
        got_of = dict(zip(undecided.tolist(), got.tolist()))
        for chain in chains.values():
            for k in chain:
                if verdicts[k] != -1:
                    continue
                verdicts[k] = got_of[k]
                if got_of[k] != 1:
                    break
    verdicts = [int(v) for v in verdicts]
    return verdicts, out[3:], out[1], rounds


# ---- anonymous-transfer state updates of one block (modules/anonymous-balances/src/lib.rs:23-82, 169-232) ---------------
# statuses as BLOCK_*; account flags as ACCOUNT_*


def anonymous_block(ctx: Context, keys, balances, pendings, flags, members, tx_points, tx_extra, g_epoch, applied):
    """rollover of the 12 ring members, the balances verify_anonymous_proof reads, and add_pending_transfer for every member
    of the applied transactions (zk_balances_anonymous_block).  keys: 32 bytes per account (its EncKey); balances /
    pendings / flags: as confidential_block; members: ANONIMITY_SIZE account indices per transaction (flat or one row per
    transaction); tx_points: 416 bytes per transaction (left_ciphertexts | right_ciphertext); tx_extra: 64 bytes per
    transaction (rvk | nonce); g_epoch: 32 bytes; applied: one byte per transaction, applied when 1 (a verdict of
    verify_proofs_with_points passes unchanged).  Returns (enc_balances, verify_points, status, new_balances, new_pendings,
    new_flags) as bytes: 768 and 1664 bytes per transaction for the first two.  Raises SynthesisError(ZK_ERR_DECODE) naming
    the account when a touched account's stored ciphertext does not read."""
    n_acct = len(flags)
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1).astype(np.uint32))
    assert len(mem) % ANONIMITY_SIZE == 0
    n_tx = len(mem) // ANONIMITY_SIZE
    ky, bal, pend, fl = _cat(keys, 32), _cat(balances, 64), _cat(pendings, 64), bytes(flags)
    tp, tx, ge, ap = _cat(tx_points, 32 * (ANONIMITY_SIZE + 1)), _cat(tx_extra, 64), _pt32(g_epoch), bytes(applied)
    assert len(ky) == 32 * n_acct and len(bal) == len(pend) == 64 * n_acct
    assert len(tp) == 32 * (ANONIMITY_SIZE + 1) * n_tx and len(tx) == 64 * n_tx and len(ap) == n_tx
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    eb = np.zeros(max(64 * ANONIMITY_SIZE * n_tx, 1), np.uint8)
    vp = np.zeros(max(32 * ANONYMOUS_POINTS * n_tx, 1), np.uint8)
    st = np.zeros(max(n_tx, 1), np.uint8)
    nb, npd = np.zeros(max(64 * n_acct, 1), np.uint8), np.zeros(max(64 * n_acct, 1), np.uint8)
    nf = np.zeros(max(n_acct, 1), np.uint8)
    _ck(_lib.lib().zk_balances_anonymous_block(ctx._h, n_acct, _p(buf(ky)), _p(buf(bal)), _p(buf(pend)), _p(buf(fl)), n_tx,
                                               _p(mem if n_tx else np.zeros(1, np.uint32)), _p(buf(tp)), _p(buf(tx)), _p(buf(ge)),
                                               _p(buf(ap)), _p(eb), _p(vp), _p(st), _p(nb), _p(npd), _p(nf)))
    return (eb[:64 * ANONIMITY_SIZE * n_tx].tobytes(), vp[:32 * ANONYMOUS_POINTS * n_tx].tobytes(), st[:n_tx].tobytes(),
            nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())


def anonymous_block_device(ctx: Context, n_accounts: int, d_keys_ptr: int, d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int,
                           n_tx: int, d_members_ptr: int, d_tx_points_ptr: int, d_tx_extra_ptr: int, d_g_epoch_ptr: int, d_applied_ptr: int,
                           d_enc_balances_ptr: int, d_verify_points_ptr: int, d_status_ptr: int, d_new_balances_ptr: int,
                           d_new_pendings_ptr: int, d_new_flags_ptr: int):
    """The same on device pointers (d_members: uint32), asynchronous on the context's stream; ctx.sync() raises
    SynthesisError(ZK_ERR_DECODE) naming a touched account whose stored ciphertext did not read."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_balances_anonymous_block_device(ctx._h, n_accounts, v(d_keys_ptr), v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr),
                                                      n_tx, v(d_members_ptr), v(d_tx_points_ptr), v(d_tx_extra_ptr), v(d_g_epoch_ptr),
                                                      v(d_applied_ptr), v(d_enc_balances_ptr), v(d_verify_points_ptr), v(d_status_ptr),
                                                      v(d_new_balances_ptr), v(d_new_pendings_ptr), v(d_new_flags_ptr)))


ANON_TRANSFER, ANON_ISSUE = 0, 1    # zk_anonymous_calls_block kinds


class AnonymousTx:
    """One anonymous_transfer extrinsic (lib.rs:23-30) with its ring as indices into the block's account table: the 12
    members (enc_keys), their left ciphertexts, right_ciphertext, the signer's rvk and the nonce."""
    kind = ANON_TRANSFER

    def __init__(self, members, left_ciphertexts, right_ciphertext, rvk, nonce):
        self.members = [int(m) for m in members]
        self.left_ciphertexts = [_pt32(c) for c in left_ciphertexts]
        if len(self.members) != ANONIMITY_SIZE or len(self.left_ciphertexts) != ANONIMITY_SIZE:
            raise ValueError("AnonymousTx: a ring of %d members and %d left ciphertexts; the anonymous key takes %d"
                             % (len(self.members), len(self.left_ciphertexts), ANONIMITY_SIZE))
        self.right_ciphertext, self.rvk, self.nonce = _pt32(right_ciphertext), _pt32(rvk), _pt32(nonce)

    def points(self) -> bytes:
        return b"".join(self.left_ciphertexts) + self.right_ciphertext


def anonymous_calls_block(ctx: Context, keys, balances, pendings, flags, kind, members, tx_points, tx_extra, g_epoch, applied):
    """anonymous_transfer and issue in block order (zk_anonymous_calls_block): the arguments of anonymous_block plus kind,
    one ANON_* byte per transaction.  An issue's issuer is its members[0] (the other 11 are ignored), its total slot 0 and
    its randomness slot 12 of its tx_points row; its tx_extra row is ignored.  Returns (enc_balances, verify_points,
    issued, status, new_balances, new_pendings, new_flags) as bytes: issued holds 64 bytes per transaction, the Issued
    ciphertext of each applied issue and zero bytes elsewhere; an issue's enc_balances and verify_points rows are zero.
    Raises SynthesisError(ZK_ERR_DECODE) as anonymous_block."""
    n_acct = len(flags)
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1).astype(np.uint32))
    assert len(mem) % ANONIMITY_SIZE == 0
    n_tx = len(mem) // ANONIMITY_SIZE
    ky, bal, pend, fl, kd = _cat(keys, 32), _cat(balances, 64), _cat(pendings, 64), bytes(flags), bytes(kind)
    tp, tx, ge, ap = _cat(tx_points, 32 * (ANONIMITY_SIZE + 1)), _cat(tx_extra, 64), _pt32(g_epoch), bytes(applied)
    assert len(ky) == 32 * n_acct and len(bal) == len(pend) == 64 * n_acct and len(kd) == n_tx
    assert len(tp) == 32 * (ANONIMITY_SIZE + 1) * n_tx and len(tx) == 64 * n_tx and len(ap) == n_tx
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    z = lambda n: np.zeros(max(n, 1), np.uint8)
    eb, vp, iss, st = z(64 * ANONIMITY_SIZE * n_tx), z(32 * ANONYMOUS_POINTS * n_tx), z(64 * n_tx), z(n_tx)
    nb, npd, nf = z(64 * n_acct), z(64 * n_acct), z(n_acct)
    _ck(_lib.lib().zk_anonymous_calls_block(ctx._h, n_acct, _p(buf(ky)), _p(buf(bal)), _p(buf(pend)), _p(buf(fl)), n_tx, _p(buf(kd)),
                                            _p(mem if n_tx else np.zeros(1, np.uint32)), _p(buf(tp)), _p(buf(tx)), _p(buf(ge)), _p(buf(ap)),
                                            _p(eb), _p(vp), _p(iss), _p(st), _p(nb), _p(npd), _p(nf)))
    return (eb[:64 * ANONIMITY_SIZE * n_tx].tobytes(), vp[:32 * ANONYMOUS_POINTS * n_tx].tobytes(), iss[:64 * n_tx].tobytes(),
            st[:n_tx].tobytes(), nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes())


def anonymous_calls_block_device(ctx: Context, n_accounts: int, d_keys_ptr: int, d_balances_ptr: int, d_pendings_ptr: int,
                                 d_flags_ptr: int, n_tx: int, d_kind_ptr: int, d_members_ptr: int, d_tx_points_ptr: int, d_tx_extra_ptr: int,
                                 d_g_epoch_ptr: int, d_applied_ptr: int, d_enc_balances_ptr: int, d_verify_points_ptr: int,
                                 d_issued_ptr: int, d_status_ptr: int, d_new_balances_ptr: int, d_new_pendings_ptr: int,
                                 d_new_flags_ptr: int):
    """The same on device pointers (d_members: uint32), asynchronous on the context's stream; only the applied issues'
    entries of d_issued are written.  ctx.sync() raises SynthesisError(ZK_ERR_DECODE) as anonymous_block_device."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_anonymous_calls_block_device(ctx._h, n_accounts, v(d_keys_ptr), v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr),
                                                   n_tx, v(d_kind_ptr), v(d_members_ptr), v(d_tx_points_ptr), v(d_tx_extra_ptr),
                                                   v(d_g_epoch_ptr), v(d_applied_ptr), v(d_enc_balances_ptr), v(d_verify_points_ptr),
                                                   v(d_issued_ptr), v(d_status_ptr), v(d_new_balances_ptr), v(d_new_pendings_ptr),
                                                   v(d_new_flags_ptr)))


class AnonIssueTx:
    """One issue extrinsic of anonymous-balances (lib.rs:87-99): issuer is an index into the block's account table; rvk is
    the signer."""
    kind = ANON_ISSUE

    def __init__(self, issuer: int, total, fee, balance, randomness, rvk, nonce):
        self.issuer = int(issuer)
        self.total, self.fee, self.balance, self.randomness = _pt32(total), _pt32(fee), _ct64(balance), _pt32(randomness)
        self.rvk, self.nonce = _pt32(rvk), _pt32(nonce)

    @property
    def members(self):
        return [self.issuer] * ANONIMITY_SIZE

    def points(self) -> bytes:
        return self.total + bytes(32 * (ANONIMITY_SIZE - 1)) + self.randomness

    def verify_points(self, keys, g_epoch) -> bytes:
        """what lib.rs:111-122 passes to verify_confidential_proof: (issuer, issuer, total, total, balance, rvk, fee,
        randomness, nonce); keys: the account table's EncKeys"""
        ky = _cat(keys, 32)
        issuer = ky[32 * self.issuer:32 * self.issuer + 32]
        return confidential_points(issuer, issuer, self.total, self.total, self.randomness, self.fee, self.balance, self.rvk,
                                   _pt32(g_epoch), self.nonce)


def import_anonymous_calls_block(ctx: Context, anon_pvk: PreparedVerifyingKey, conf_pvk: PreparedVerifyingKey, accounts, txs, g_epoch,
                                 proofs):
    """Verify and apply a block of anonymous-balances extrinsics (AnonymousTx and AnonIssueTx, in block order) the way the
    runtime does, with the state, the verifier's inputs and the verdicts on the device.  accounts = (keys, balances,
    pendings, flags) as anonymous_block takes them; g_epoch: the block's 32-byte LastGEpoch; proofs: 192 bytes each,
    checked with conf_pvk for issues and anon_pvk for transfers.

    An issue's proof reads only its own fields, and a transfer changes pending balances only, so nothing a proof is checked
    against depends on a transfer's verdict.  One upload, then: the issues' proofs on their 11 points; the state pass with
    the issue verdicts as the mask (no transfer applied), which gives every transfer's 52 public-input points; the
    transfers' proofs on them; the state pass again with all the verdicts; one download.  A block without issues takes
    zk_balances_anonymous_block's passes.

    Returns (verdicts, (new_balances, new_pendings, new_flags), enc_balances, issued): the reference's verdict per
    transaction (1 passes; the other values as verify_proofs_with_points), the 12 balances (768 bytes, zero for an issue)
    each transfer's proof was checked against, and the Issued ciphertext (64 bytes) of each applied issue, None
    elsewhere.  Raises ValueError for an account index out of range, SynthesisError(ZK_ERR_DECODE) for a touched account
    whose stored ciphertext does not read."""
    import torch
    keys, balances, pendings, flags = accounts
    n_acct, n = len(flags), len(txs)
    if any(not all(0 <= m < n_acct for m in t.members) for t in txs):
        raise ValueError("import_anonymous_block: account index out of range")
    proofs = _cat(proofs, 192)
    assert len(proofs) == 192 * n
    ky, bal, pend, fl, ge = _cat(keys, 32), _cat(balances, 64), _cat(pendings, 64), bytes(flags), _pt32(g_epoch)
    assert len(ky) == 32 * n_acct and len(bal) == len(pend) == 64 * n_acct
    if not n:
        return [], (bal, pend, fl), b"", []
    kind = np.array([t.kind for t in txs], np.uint8)
    iss_idx, tr_idx = np.flatnonzero(kind == ANON_ISSUE), np.flatnonzero(kind == ANON_TRANSFER)
    n_iss, n_tr = len(iss_idx), len(tr_idx)
    members = np.array([t.members for t in txs], np.uint32).reshape(-1)
    proof_rows = np.frombuffer(proofs, np.uint8).reshape(n, 192)
    iss_points = b"".join(txs[k].verify_points(ky, ge) for k in iss_idx.tolist())
    idx = np.concatenate([iss_idx, tr_idx]).astype(np.int64)
    # one host buffer of the inputs (members and the index lists first, 4- and 8-byte aligned), one of the outputs
    parts = [idx.tobytes(), members.tobytes(), ky, bal, pend, fl, b"".join(t.points() for t in txs),
             b"".join(t.rvk + t.nonce for t in txs),
             ge, kind.tobytes(), proof_rows[iss_idx].tobytes(), proof_rows[tr_idx].tobytes(), iss_points]
    offs = np.cumsum([0] + [len(p) for p in parts]).tolist()
    dev = torch.device("cuda", ctx.device)
    d_in = torch.frombuffer(bytearray(b"".join(parts)), dtype=torch.uint8).to(dev)
    sizes = [64 * ANONIMITY_SIZE * n, 32 * ANONYMOUS_POINTS * n, 64 * n, n, 64 * n_acct, 64 * n_acct, n_acct, n, n]
    oo = np.cumsum([0] + sizes).tolist()
    d_out = torch.zeros(oo[-1], dtype=torch.uint8, device=dev)     # the last 2n bytes: the mask, then the compact verdicts
    torch.cuda.current_stream(dev).synchronize()                    # the context's stream is not torch's
    pi = lambda i: d_in.data_ptr() + offs[i]
    po = lambda i: d_out.data_ptr() + oo[i]
    d_idx = d_in[offs[0]:offs[1]].view(torch.int64)
    mask, compact = d_out[oo[7]:oo[8]], d_out[oo[8]:oo[9]]
    rows = d_out[oo[1]:oo[2]].view(n, 32 * ANONYMOUS_POINTS)
    ctx_stream = torch.cuda.ExternalStream(ctx.stream, device=dev) if ctx.stream else torch.cuda.default_stream(dev)

    def sync_pvk(pvk):
        if pvk.ctx is not ctx:
            ctx.sync()
        return pvk

    def done_pvk(pvk):
        if pvk.ctx is not ctx:
            pvk.ctx.sync()

    def state():
        if n_iss:
            anonymous_calls_block_device(ctx, n_acct, pi(2), pi(3), pi(4), pi(5), n, pi(9), pi(1), pi(6), pi(7), pi(8), po(7), po(0), po(1),
                                         po(2), po(3), po(4), po(5), po(6))
        else:
            anonymous_block_device(ctx, n_acct, pi(2), pi(3), pi(4), pi(5), n, pi(1), pi(6), pi(7), pi(8), po(7), po(0), po(1), po(3),
                                   po(4), po(5), po(6))
    if n_iss:
        verify_proofs_with_points_device(sync_pvk(conf_pvk), n_iss, pi(10), pi(12), CONFIDENTIAL_POINTS, po(8))
        done_pvk(conf_pvk)
        with torch.cuda.stream(ctx_stream):
            mask.index_copy_(0, d_idx[:n_iss], compact[:n_iss])
    state()
    if n_tr:
        with torch.cuda.stream(ctx_stream):
            tr_rows = rows.index_select(0, d_idx[n_iss:]) if n_iss else rows
        # without issues the verdicts land in the mask directly
        verify_proofs_with_points_device(sync_pvk(anon_pvk), n_tr, pi(11), tr_rows.data_ptr(), ANONYMOUS_POINTS,
                                         po(8) + n_iss if n_iss else po(7))
        done_pvk(anon_pvk)
        if n_iss:
            with torch.cuda.stream(ctx_stream):
                mask.index_copy_(0, d_idx[n_iss:], compact[n_iss:])
        state()
    ctx.sync()
    host = d_out[:oo[8]].cpu().numpy().tobytes()
    verdicts = [int(v) for v in host[oo[7]:oo[8]]]
    st = host[oo[3]:oo[4]]
    issued = [host[oo[2] + 64 * k:oo[2] + 64 * k + 64] if kind[k] == ANON_ISSUE and st[k] == BLOCK_APPLIED else None for k in range(n)]
    return verdicts, (host[oo[4]:oo[5]], host[oo[5]:oo[6]], host[oo[6]:oo[7]]), host[oo[0]:oo[1]], issued


def import_anonymous_block(ctx: Context, pvk: PreparedVerifyingKey, accounts, txs, g_epoch, proofs):
    """Verify and apply a block of anonymous transfers the way the runtime does, with the state, the verifier's inputs and
    the verdicts on the device: import_anonymous_calls_block for a block without issues.  accounts = (keys, balances,
    pendings, flags) as anonymous_block takes them; txs: AnonymousTx list; g_epoch: the block's 32-byte LastGEpoch;
    proofs: 192 bytes each.

    Returns (verdicts, (new_balances, new_pendings, new_flags), enc_balances): the reference's verdict per transaction (1
    passes; the other values as verify_proofs_with_points) and the 12 balances (768 bytes) each transaction's proof was
    checked against.  Raises ValueError for an account index out of range, SynthesisError(ZK_ERR_DECODE) for a touched
    account whose stored ciphertext does not read."""
    verdicts, state, enc_balances, _ = import_anonymous_calls_block(ctx, pvk, None, accounts, txs, g_epoch, proofs)
    return verdicts, state, enc_balances


# ---- encrypted-asset calls of one block (modules/encrypted-assets/src/lib.rs:32-215, 266-358) -----------------------------
# zk_assets_block kinds; statuses as BLOCK_*, slot flags as ACCOUNT_*
ASSET_TRANSFER, ASSET_ISSUE, ASSET_DESTROY = 0, 1, 2
ASSET_ID_MAX = 2**32 - 1            # AssetId = u32 (runtime/src/lib.rs)


def assets_block(ctx: Context, balances, pendings, flags, kind, slot_a, slot_b, tx_points, applied):
    """confidential_transfer, issue and destroy over a block of (AssetId, EncKey) slots, in order (zk_assets_block).
    balances / pendings: 64 bytes per slot; flags: one ACCOUNT_* byte per slot; kind: one ASSET_* byte per transaction;
    slot_a: the sender's / issuer's (new id, issuer) / owner's slot; slot_b: the recipient's slot (transfers only);
    tx_points: 128 bytes per transaction (transfer: amount_sender | amount_recipient | fee_sender | randomness; issue: total
    | - | - | randomness); applied: one byte per transaction, applied when 1.  Returns (balance_sender, balance_after,
    event_ct, event_flags, status, new_balances, new_pendings, new_flags) as bytes; balance_after, event_ct and event_flags
    are zero where the call writes nothing.  Raises SynthesisError(ZK_ERR_DECODE) naming the slot when a named slot's
    stored ciphertext does not read."""
    n_slots, n_tx = len(flags), len(kind)
    bal, pend, fl, kd, tp, ap = (_cat(balances, 64), _cat(pendings, 64), bytes(flags), bytes(kind), _cat(tx_points, 128), bytes(applied))
    assert len(bal) == len(pend) == 64 * n_slots and len(slot_a) == len(slot_b) == n_tx and len(tp) == 128 * n_tx and len(ap) == n_tx
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    idx = lambda v: np.ascontiguousarray(np.asarray(v, np.int64).astype(np.uint32)) if n_tx else np.zeros(1, np.uint32)
    z = lambda n: np.zeros(max(n, 1), np.uint8)
    bs, ba, ev, ef, st = z(64 * n_tx), z(64 * n_tx), z(128 * n_tx), z(n_tx), z(n_tx)
    nb, npd, nf = z(64 * n_slots), z(64 * n_slots), z(n_slots)
    _ck(_lib.lib().zk_assets_block(ctx._h, n_slots, _p(buf(bal)), _p(buf(pend)), _p(buf(fl)), n_tx, _p(buf(kd)), _p(idx(slot_a)),
                                   _p(idx(slot_b)), _p(buf(tp)), _p(buf(ap)), _p(bs), _p(ba), _p(ev), _p(ef), _p(st), _p(nb), _p(npd), _p(nf)))
    return (bs[:64 * n_tx].tobytes(), ba[:64 * n_tx].tobytes(), ev[:128 * n_tx].tobytes(), ef[:n_tx].tobytes(), st[:n_tx].tobytes(),
            nb[:64 * n_slots].tobytes(), npd[:64 * n_slots].tobytes(), nf[:n_slots].tobytes())


def assets_block_device(ctx: Context, n_slots: int, d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int, n_tx: int, d_kind_ptr: int,
                        d_slot_a_ptr: int, d_slot_b_ptr: int, d_tx_points_ptr: int, d_applied_ptr: int, d_balance_sender_ptr: int,
                        d_balance_after_ptr: int, d_event_ct_ptr: int, d_event_flags_ptr: int, d_status_ptr: int, d_new_balances_ptr: int,
                        d_new_pendings_ptr: int, d_new_flags_ptr: int):
    """The same on device pointers (d_slot_a / d_slot_b: uint32), asynchronous on the context's stream; ctx.sync() raises
    SynthesisError(ZK_ERR_DECODE) naming a named slot whose stored ciphertext did not read.  Only the applied transactions'
    entries of d_balance_after (transfers) and d_event_ct / d_event_flags (issues and destroys) are written."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_assets_block_device(ctx._h, n_slots, v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr), n_tx, v(d_kind_ptr),
                                          v(d_slot_a_ptr), v(d_slot_b_ptr), v(d_tx_points_ptr), v(d_applied_ptr), v(d_balance_sender_ptr),
                                          v(d_balance_after_ptr), v(d_event_ct_ptr), v(d_event_flags_ptr), v(d_status_ptr),
                                          v(d_new_balances_ptr), v(d_new_pendings_ptr), v(d_new_flags_ptr)))


class AssetTransferTx:
    """One confidential_transfer extrinsic of encrypted-assets (lib.rs:86-99): its accounts are the slots (asset_id,
    address_sender) and (asset_id, address_recipient); rvk is the signer, g_epoch the block's LastGEpoch."""
    kind = ASSET_TRANSFER

    def __init__(self, asset_id: int, address_sender, address_recipient, amount_sender, amount_recipient, fee_sender, randomness,
                 rvk, g_epoch, nonce):
        self.asset_id = int(asset_id)
        self.address_sender, self.address_recipient = _pt32(address_sender), _pt32(address_recipient)
        self.amount_sender, self.amount_recipient = _pt32(amount_sender), _pt32(amount_recipient)
        self.fee_sender, self.randomness = _pt32(fee_sender), _pt32(randomness)
        self.rvk, self.g_epoch, self.nonce = _pt32(rvk), _pt32(g_epoch), _pt32(nonce)

    def points(self) -> bytes:
        return self.amount_sender + self.amount_recipient + self.fee_sender + self.randomness

    def verify_points(self, balance_sender: bytes) -> bytes:
        return confidential_points(self.address_sender, self.address_recipient, self.amount_sender, self.amount_recipient,
                                   self.randomness, self.fee_sender, balance_sender, self.rvk, self.g_epoch, self.nonce)


class IssueTx:
    """One issue extrinsic (lib.rs:32-41): the new asset's slot is (NextAssetId, issuer)."""
    kind = ASSET_ISSUE

    def __init__(self, issuer, total, fee, balance, randomness, rvk, g_epoch, nonce):
        self.issuer, self.total, self.fee = _pt32(issuer), _pt32(total), _pt32(fee)
        self.balance, self.randomness = _ct64(balance), _pt32(randomness)
        self.rvk, self.g_epoch, self.nonce = _pt32(rvk), _pt32(g_epoch), _pt32(nonce)

    def points(self) -> bytes:
        return self.total + bytes(64) + self.randomness

    def verify_points(self) -> bytes:
        """what lib.rs:53-64 passes: (issuer, issuer, total, total, balance, rvk, fee, randomness, nonce)"""
        return confidential_points(self.issuer, self.issuer, self.total, self.total, self.randomness, self.fee, self.balance, self.rvk,
                                   self.g_epoch, self.nonce)


class DestroyTx:
    """One destroy extrinsic (lib.rs:167-177) of the slot (asset_id, owner)."""
    kind = ASSET_DESTROY

    def __init__(self, owner, asset_id: int, dummy_amount, dummy_fee, dummy_balance, randomness, rvk, g_epoch, nonce):
        self.owner, self.asset_id = _pt32(owner), int(asset_id)
        self.dummy_amount, self.dummy_fee, self.dummy_balance = _pt32(dummy_amount), _pt32(dummy_fee), _ct64(dummy_balance)
        self.randomness, self.rvk, self.g_epoch, self.nonce = _pt32(randomness), _pt32(rvk), _pt32(g_epoch), _pt32(nonce)

    def points(self) -> bytes:
        return bytes(128)

    def verify_points(self) -> bytes:
        """what lib.rs:188-199 passes: (owner, owner, dummy_amount, dummy_amount, dummy_balance, rvk, dummy_fee, randomness,
        nonce)"""
        return confidential_points(self.owner, self.owner, self.dummy_amount, self.dummy_amount, self.randomness, self.dummy_fee,
                                   self.dummy_balance, self.rvk, self.g_epoch, self.nonce)


def _asset_slots(name: str, slots: list, balances, pendings, flags, txs, verdicts, next_asset_id: int, new_slot_flags: int):
    """Asset ids, then slots, once the issue and destroy verdicts are known: the passing issues are numbered from
    next_asset_id, and every (asset_id, key) a transaction names is resolved to a row of the slot table; new ones are
    appended to `slots` (in place) and to the table, absent, with new_slot_flags.  A failing issue or destroy names no slot.
    Returns ((balances, pendings, flags) of the grown table, asset_ids, slot_a, slot_b)."""
    n = len(txs)
    index = {s: i for i, s in enumerate(slots)}
    bal, pend, fl = bytearray(_cat(balances, 64)), bytearray(_cat(pendings, 64)), bytearray(flags)

    def slot(asset_id, key):
        s = (asset_id, key)
        if s not in index:
            index[s] = len(slots)
            slots.append(s)
            bal.extend(bytes(64)); pend.extend(bytes(64)); fl.append(new_slot_flags & 0xFF & ~(ACCOUNT_BALANCE | ACCOUNT_PENDING))
        return index[s]
    asset_ids = [None] * n
    next_id = int(next_asset_id)
    none = 0xFFFFFFFF                                         # past every slot: a failed issue or destroy touches nothing
    slot_a, slot_b = np.full(n, none, np.uint32), np.full(n, none, np.uint32)
    for k, t in enumerate(txs):
        if t.kind == ASSET_ISSUE:
            if verdicts[k] != 1:
                continue
            if next_id > ASSET_ID_MAX:
                raise ValueError("%s: asset id %d would pass 2^32 - 1" % (name, next_id))
            asset_ids[k] = next_id
            slot_a[k] = slot(next_id, t.issuer)
            next_id += 1
        elif t.kind == ASSET_DESTROY:
            if verdicts[k] == 1:
                slot_a[k] = slot(t.asset_id, t.owner)
        else:
            slot_a[k] = slot(t.asset_id, t.address_sender)
            slot_b[k] = slot(t.asset_id, t.address_recipient)
    return (bytes(bal), bytes(pend), bytes(fl)), asset_ids, slot_a, slot_b


def _asset_events(kinds, ba: bytes, ev: bytes, ef: bytes, st: bytes) -> list:
    """The event ciphertexts of each applied transaction, from zk_assets_block's outputs (see import_assets_block)."""
    events = [None] * len(kinds)
    for k in range(len(kinds)):
        if st[k] != BLOCK_APPLIED:
            continue
        if kinds[k] == ASSET_TRANSFER:
            events[k] = ba[64 * k:64 * k + 64]
        elif kinds[k] == ASSET_ISSUE:
            events[k] = ev[128 * k:128 * k + 64]
        else:
            events[k] = tuple(ev[128 * k + 64 * w:128 * k + 64 * w + 64] if ef[k] >> w & 1 else b"" for w in range(2))
    return events


def import_assets_block(ctx: Context, pvk: PreparedVerifyingKey, state, txs, proofs, next_asset_id: int, new_slot_flags: int):
    """Verify and apply a block of encrypted-asset extrinsics the way the runtime does, one after another.  state =
    (slots, balances, pendings, flags): slots lists the (asset_id, enc_key) of each row of the slot table, the rest as
    assets_block takes them; txs: AssetTransferTx / IssueTx / DestroyTx list; proofs: 192 bytes each; next_asset_id: the
    NextAssetId before the block; new_slot_flags: the flags of a slot the block creates (ACCOUNT_DUE when current_epoch >
    0, since its LastRollOver is absent).

    Issue and destroy proofs read only extrinsic fields, so they are verified first, in one batch.  The passing issues are
    numbered from next_asset_id, which names their slots.  Every (asset_id, key) is then resolved to a slot; new ones are
    appended, absent.  A transfer's proof reads its sender's balance, which depends on the sender slot's earlier transfers
    that passed (issues and destroys are decided by then), so the transfers take the rounds of import_confidential_block,
    with chains keyed by sender slot: at most 1 + (the most failures in one chain), one when nothing fails.

    Returns (verdicts, asset_ids, events, (slots, new_balances, new_pendings, new_flags), rounds): the reference's verdict
    per transaction (1 passes; the other values as verify_proofs_with_points); the id each passing issue created (None
    elsewhere); the event ciphertexts of each applied transaction (a transfer: the sender's balance after; an issue: the
    total, also its TotalSupply; a destroy: (taken balance, taken pending), b"" for an absent one, as Ciphertext::default())
    and None for the others.  Raises ValueError when an asset id would pass 2^32 - 1, SynthesisError(ZK_ERR_DECODE) for a
    named slot whose stored ciphertext does not read."""
    slots, balances, pendings, flags = state
    slots = [(int(a), _pt32(k)) for a, k in slots]
    n = len(txs)
    proofs = _cat(proofs, 192)
    assert len(proofs) == 192 * n and len(flags) == len(slots)
    proof_rows = np.frombuffer(proofs, np.uint8).reshape(n, 192) if n else np.zeros((0, 192), np.uint8)
    kinds = np.array([t.kind for t in txs], np.uint8)
    verdicts = np.full(n, -1, np.int16)                      # -1: undecided
    fixed = np.flatnonzero(kinds != ASSET_TRANSFER)
    if len(fixed):
        pts = b"".join(txs[k].verify_points() for k in fixed.tolist())
        verdicts[fixed] = verify_proofs_with_points(pvk, proof_rows[fixed].tobytes(), pts, CONFIDENTIAL_POINTS)
    table, asset_ids, slot_a, slot_b = _asset_slots("import_assets_block", slots, balances, pendings, flags, txs, verdicts, next_asset_id,
                                                    new_slot_flags)
    tx_points = b"".join(t.points() for t in txs)
    is_transfer = kinds == ASSET_TRANSFER
    chains = None
    rounds = 0
    while True:
        mask = np.where(is_transfer, (verdicts == -1) | (verdicts == 1), verdicts == 1).astype(np.uint8)
        out = assets_block(ctx, *table, kinds.tobytes(), slot_a, slot_b, tx_points, mask.tobytes())
        undecided = np.flatnonzero(verdicts == -1)
        if not len(undecided):
            break
        rounds += 1
        bs = out[0]
        pts = b"".join(txs[k].verify_points(bs[64 * k:64 * k + 64]) for k in undecided.tolist())
        got = np.array(verify_proofs_with_points(pvk, proof_rows[undecided].tobytes(), pts, CONFIDENTIAL_POINTS), np.int16)
        if (got == 1).all():
            verdicts[undecided] = 1
            break                   # every balance of this round was exact: out is the final state
        if chains is None:
            chains = {}
            for k in np.flatnonzero(is_transfer).tolist():
                chains.setdefault(int(slot_a[k]), []).append(k)
        got_of = dict(zip(undecided.tolist(), got.tolist()))
        for chain in chains.values():
            for k in chain:
                if verdicts[k] != -1:
                    continue
                verdicts[k] = got_of[k]
                if got_of[k] != 1:
                    break
    events = _asset_events(kinds, *out[1:5])
    return [int(v) for v in verdicts], asset_ids, events, (slots,) + out[5:], rounds


# ---- block import in one call: the rounds of import_confidential_block / import_assets_block on the device --------------
def _import_error(name: str, e: ZkError):
    """zk_import_*'s ZK_ERR_INVALID for an index out of range becomes the drivers' ValueError"""
    if e.code == -2 and "out of range" in str(e):
        return ValueError("%s: %s" % (name, e))
    return e


def _confidential_rows(txs) -> bytes:
    """each transfer's 11 verifier points in confidential_points order, balance_sender (slots 6-7) zero"""
    return b"".join(t.address_sender + t.address_recipient + t.amount_sender + t.amount_recipient + t.randomness + t.fee_sender +
                    bytes(64) + t.rvk + t.g_epoch + t.nonce for t in txs)


def _conf_section(name: str, accounts, txs, proofs):
    """confidential_import's C arguments after ctx and the key, and the function that reads its result from them"""
    balances, pendings, flags = accounts
    n_acct, n = len(flags), len(txs)
    if any(not (0 <= t.sender < 2**32 and 0 <= t.recipient < 2**32) for t in txs):
        raise ValueError("%s: account index out of range" % name)
    proofs = _cat(proofs, 192)
    bal, pend, fl = _cat(balances, 64), _cat(pendings, 64), bytes(flags)
    assert len(proofs) == 192 * n and len(bal) == len(pend) == 64 * n_acct
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    idx = lambda v: np.array(v or [0], np.uint32)
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    v, ba, st, nb, npd, nf = z(n), z(64 * n), z(n), z(64 * n_acct), z(64 * n_acct), z(n_acct)
    rounds = C.c_uint(0)
    keep = [buf(bal), buf(pend), buf(fl), idx([t.sender for t in txs]), idx([t.recipient for t in txs]), buf(_confidential_rows(txs)),
            buf(proofs)]
    args = [n_acct] + [_p(a) for a in keep[:3]] + [n] + [_p(a) for a in keep[3:]] + [_p(x) for x in (v, ba, st, nb, npd, nf)] + [C.byref(rounds)]

    def result():
        return ([int(x) for x in v[:n]], (nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes()),
                ba[:64 * n].tobytes(), rounds.value)
    return args, result, keep


def confidential_import(ctx: Context, pvk: PreparedVerifyingKey, accounts, txs, proofs):
    """import_confidential_block in one call (zk_import_confidential_block): the rounds run on the device, between one
    upload and one download, and the proofs are checked on ctx.  Same arguments, result and errors, except that a key of
    another shape raises SynthesisError(MalformedVerifyingKey) even for a block without transfers."""
    args, result, _keep = _conf_section("confidential_import", accounts, txs, proofs)
    if pvk.ctx is not ctx:
        pvk.ctx.sync()
    try:
        _ck(_lib.lib().zk_import_confidential_block(ctx._h, pvk._h, *args))
    except ZkError as e:
        raise _import_error("confidential_import", e) from None
    return result()


def confidential_import_device(ctx: Context, pvk: PreparedVerifyingKey, n_accounts: int, d_balances_ptr: int, d_pendings_ptr: int,
                               d_flags_ptr: int, n_tx: int, d_sender_ptr: int, d_recipient_ptr: int, d_rows_ptr: int, d_proofs_ptr: int,
                               d_verdicts_ptr: int, d_balance_after_ptr: int, d_status_ptr: int, d_new_balances_ptr: int,
                               d_new_pendings_ptr: int, d_new_flags_ptr: int) -> int:
    """zk_import_confidential_block_device on device pointers (d_sender / d_recipient: uint32; d_rows: n_tx * 352 bytes in
    confidential_points order, slots 6-7 ignored).  Blocks on the context's stream once before the first round and once
    after each; returns the number of rounds, with the outputs complete."""
    v = lambda x: C.c_void_p(x) if x else None
    rounds = C.c_uint(0)
    _ck(_lib.lib().zk_import_confidential_block_device(ctx._h, pvk._h, n_accounts, v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr),
                                                       n_tx, v(d_sender_ptr), v(d_recipient_ptr), v(d_rows_ptr), v(d_proofs_ptr),
                                                       v(d_verdicts_ptr), v(d_balance_after_ptr), v(d_status_ptr), v(d_new_balances_ptr),
                                                       v(d_new_pendings_ptr), v(d_new_flags_ptr), C.byref(rounds)))
    return rounds.value


def assets_import(ctx: Context, pvk: PreparedVerifyingKey, state, txs, proofs, next_asset_id: int, new_slot_flags: int):
    """import_assets_block with the transfer rounds in one call (zk_import_assets_block).  The issue and destroy proofs
    are verified first, and asset ids and slots resolved from their verdicts, exactly as import_assets_block does; the
    rounds then run on the device between one upload and one download, with the transfer proofs checked on ctx.  Same
    arguments, result and errors, except for a key of another shape, as confidential_import."""
    slots, balances, pendings, flags = state
    slots = [(int(a), _pt32(k)) for a, k in slots]
    n = len(txs)
    proofs = _cat(proofs, 192)
    assert len(proofs) == 192 * n and len(flags) == len(slots)
    proof_rows = np.frombuffer(proofs, np.uint8).reshape(n, 192) if n else np.zeros((0, 192), np.uint8)
    kinds = np.array([t.kind for t in txs], np.uint8)
    fixed_v = np.zeros(n, np.uint8)
    fixed = np.flatnonzero(kinds != ASSET_TRANSFER)
    if len(fixed):
        pts = b"".join(txs[k].verify_points() for k in fixed.tolist())
        fixed_v[fixed] = verify_proofs_with_points(pvk, proof_rows[fixed].tobytes(), pts, CONFIDENTIAL_POINTS)
    (bal, pend, fl), asset_ids, slot_a, slot_b = _asset_slots("assets_import", slots, balances, pendings, flags, txs, fixed_v,
                                                              next_asset_id, new_slot_flags)
    n_slots = len(fl)
    rows = b"".join(t.verify_points(bytes(64)) if t.kind == ASSET_TRANSFER else bytes(32 * CONFIDENTIAL_POINTS) for t in txs)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    idx = lambda a: a if n else np.zeros(1, np.uint32)
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    v, ba, ev, ef, st = z(n), z(64 * n), z(128 * n), z(n), z(n)
    nb, npd, nf = z(64 * n_slots), z(64 * n_slots), z(n_slots)
    rounds = C.c_uint(0)
    if pvk.ctx is not ctx:
        pvk.ctx.sync()
    try:
        _ck(_lib.lib().zk_import_assets_block(ctx._h, pvk._h, n_slots, _p(buf(bal)), _p(buf(pend)), _p(buf(fl)), n, _p(buf(kinds.tobytes())),
                                              _p(idx(slot_a)), _p(idx(slot_b)), _p(buf(b"".join(t.points() for t in txs))), _p(buf(rows)),
                                              _p(buf(proofs)), _p(buf(fixed_v.tobytes())), _p(v), _p(ba), _p(ev), _p(ef), _p(st), _p(nb),
                                              _p(npd), _p(nf), C.byref(rounds)))
    except ZkError as e:
        raise _import_error("assets_import", e) from None
    events = _asset_events(kinds, ba[:64 * n].tobytes(), ev[:128 * n].tobytes(), ef[:n].tobytes(), st[:n].tobytes())
    table = (nb[:64 * n_slots].tobytes(), npd[:64 * n_slots].tobytes(), nf[:n_slots].tobytes())
    return [int(x) for x in v[:n]], asset_ids, events, (slots,) + table, rounds.value


def assets_import_device(ctx: Context, pvk: PreparedVerifyingKey, n_slots: int, d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int,
                         n_tx: int, d_kind_ptr: int, d_slot_a_ptr: int, d_slot_b_ptr: int, d_tx_points_ptr: int, d_rows_ptr: int,
                         d_proofs_ptr: int, d_fixed_verdicts_ptr: int, d_verdicts_ptr: int, d_balance_after_ptr: int, d_event_ct_ptr: int,
                         d_event_flags_ptr: int, d_status_ptr: int, d_new_balances_ptr: int, d_new_pendings_ptr: int,
                         d_new_flags_ptr: int) -> int:
    """zk_import_assets_block_device on device pointers (slots as assets_block_device; d_rows as confidential_import_device,
    read at transfers; d_fixed_verdicts: the issue and destroy verdicts).  Blocks as confidential_import_device; returns the
    number of rounds, with the outputs complete."""
    v = lambda x: C.c_void_p(x) if x else None
    rounds = C.c_uint(0)
    _ck(_lib.lib().zk_import_assets_block_device(ctx._h, pvk._h, n_slots, v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr), n_tx,
                                                 v(d_kind_ptr), v(d_slot_a_ptr), v(d_slot_b_ptr), v(d_tx_points_ptr), v(d_rows_ptr),
                                                 v(d_proofs_ptr), v(d_fixed_verdicts_ptr), v(d_verdicts_ptr), v(d_balance_after_ptr),
                                                 v(d_event_ct_ptr), v(d_event_flags_ptr), v(d_status_ptr), v(d_new_balances_ptr),
                                                 v(d_new_pendings_ptr), v(d_new_flags_ptr), C.byref(rounds)))
    return rounds.value


def _asset_section(name: str, state, txs, proofs, next_asset_id: int, new_slot_flags: int):
    """asset_calls_import's C arguments after ctx and the key, and the function that reads its result from them"""
    slots, balances, pendings, flags = state
    slots = [(int(a), _pt32(k)) for a, k in slots]
    n, ns = len(txs), len(slots)
    proofs = _cat(proofs, 192)
    assert len(proofs) == 192 * n and len(flags) == ns
    ids = [a for a, _ in slots] + [t.asset_id for t in txs if t.kind != ASSET_ISSUE] + [int(next_asset_id)]
    if any(not 0 <= a <= ASSET_ID_MAX for a in ids):
        raise ValueError("%s: asset id out of range" % name)
    rows = b"".join(t.verify_points(bytes(64)) if t.kind == ASSET_TRANSFER else t.verify_points() for t in txs)
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    u32 = lambda a: np.array(a or [0], np.uint32)
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    nr = ns + 2 * n
    v, aid, ba, ev, ef, st = z(n), u32([0] * n), z(64 * n), z(128 * n), z(n), z(n)
    nsi, nsk, nb, npd, nf = u32([0] * nr), z(32 * nr), z(64 * nr), z(64 * nr), z(nr)
    n_out, rounds = C.c_size_t(0), C.c_uint(0)
    keep = [u32([a for a, _ in slots]), buf(b"".join(k for _, k in slots)), buf(_cat(balances, 64)), buf(_cat(pendings, 64)),
            buf(bytes(flags)), buf(bytes(t.kind for t in txs)), u32([t.asset_id if t.kind != ASSET_ISSUE else 0 for t in txs]), buf(rows),
            buf(proofs)]
    args = ([ns] + [_p(a) for a in keep[:5]] + [int(next_asset_id), new_slot_flags & 0xFF, n] + [_p(a) for a in keep[5:]] +
            [_p(x) for x in (v, aid, ba, ev, ef, st, nsi, nsk, nb, npd, nf)] + [C.byref(n_out), C.byref(rounds)])

    def result():
        m = n_out.value
        kinds = bytes(t.kind for t in txs)
        verdicts = [int(x) for x in v[:n]]
        asset_ids = [int(aid[k]) if kinds[k] == ASSET_ISSUE and verdicts[k] == 1 else None for k in range(n)]
        events = _asset_events(kinds, ba[:64 * n].tobytes(), ev[:128 * n].tobytes(), ef[:n].tobytes(), st[:n].tobytes())
        grown = [(int(nsi[r]), nsk[32 * r:32 * r + 32].tobytes()) for r in range(m)]
        return verdicts, asset_ids, events, (grown, nb[:64 * m].tobytes(), npd[:64 * m].tobytes(), nf[:m].tobytes()), rounds.value
    return args, result, keep


def _asset_error(name: str, e: ZkError):
    """zk_import_asset_calls's ZK_ERR_INVALID for an id overflow or a repeated table row becomes a ValueError"""
    if e.code == -2 and ("2^32 - 1" in str(e) or "repeats" in str(e)):
        return ValueError("%s: %s" % (name, e))
    return e


def asset_calls_import(ctx: Context, pvk: PreparedVerifyingKey, state, txs, proofs, next_asset_id: int, new_slot_flags: int):
    """import_assets_block in one call (zk_import_asset_calls): the issue and destroy verification, the asset numbering, the
    slot resolution and the transfer rounds all run on the device between one upload and one download, with the proofs
    checked on ctx.  Same arguments, result and errors, plus a ValueError for a slot table that holds one (asset id, key)
    twice; a key of another shape raises as confidential_import does.  Asset ids (and next_asset_id) are AssetId = u32."""
    args, result, _keep = _asset_section("asset_calls_import", state, txs, proofs, next_asset_id, new_slot_flags)
    if pvk.ctx is not ctx:
        pvk.ctx.sync()
    try:
        _ck(_lib.lib().zk_import_asset_calls(ctx._h, pvk._h, *args))
    except ZkError as e:
        raise _asset_error("asset_calls_import", e) from None
    return result()


def asset_calls_import_device(ctx: Context, pvk: PreparedVerifyingKey, n_slots: int, d_slot_ids_ptr: int, d_slot_keys_ptr: int,
                              d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int, next_asset_id: int, new_slot_flags: int, n_tx: int,
                              d_kind_ptr: int, d_asset_id_ptr: int, d_rows_ptr: int, d_proofs_ptr: int, d_verdicts_ptr: int,
                              d_asset_ids_ptr: int, d_balance_after_ptr: int, d_event_ct_ptr: int, d_event_flags_ptr: int, d_status_ptr: int,
                              d_new_slot_ids_ptr: int, d_new_slot_keys_ptr: int, d_new_balances_ptr: int, d_new_pendings_ptr: int,
                              d_new_flags_ptr: int):
    """zk_import_asset_calls_device on device pointers (d_slot_ids, d_asset_id, d_asset_ids, d_new_slot_ids: uint32; the
    table outputs with room for n_slots + 2 n_tx rows).  Blocks on the context's stream twice before the rounds and as
    assets_import_device after; returns (rows of the grown table, rounds), with the outputs complete."""
    v = lambda x: C.c_void_p(x) if x else None
    n_out, rounds = C.c_size_t(0), C.c_uint(0)
    _ck(_lib.lib().zk_import_asset_calls_device(ctx._h, pvk._h, n_slots, v(d_slot_ids_ptr), v(d_slot_keys_ptr), v(d_balances_ptr),
                                                v(d_pendings_ptr), v(d_flags_ptr), next_asset_id, new_slot_flags & 0xFF, n_tx, v(d_kind_ptr),
                                                v(d_asset_id_ptr), v(d_rows_ptr), v(d_proofs_ptr), v(d_verdicts_ptr), v(d_asset_ids_ptr),
                                                v(d_balance_after_ptr), v(d_event_ct_ptr), v(d_event_flags_ptr), v(d_status_ptr),
                                                v(d_new_slot_ids_ptr), v(d_new_slot_keys_ptr), v(d_new_balances_ptr), v(d_new_pendings_ptr),
                                                v(d_new_flags_ptr), C.byref(n_out), C.byref(rounds)))
    return n_out.value, rounds.value


def _anon_section(name: str, accounts, txs, g_epoch, proofs):
    """anonymous_import's C arguments after ctx and the keys, and the function that reads its result from them"""
    keys, balances, pendings, flags = accounts
    n_acct, n = len(flags), len(txs)
    if any(not all(0 <= m < 2**32 for m in t.members) for t in txs):
        raise ValueError("%s: account index out of range" % name)
    proofs = _cat(proofs, 192)
    ky, bal, pend, fl, ge = _cat(keys, 32), _cat(balances, 64), _cat(pendings, 64), bytes(flags), _pt32(g_epoch)
    assert len(proofs) == 192 * n and len(ky) == 32 * n_acct and len(bal) == len(pend) == 64 * n_acct
    kind = bytes(t.kind for t in txs)
    has_issue = ANON_ISSUE in kind
    fields = b"".join(t.fee + t.balance if t.kind == ANON_ISSUE else bytes(96) for t in txs) if has_issue else b""
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    z = lambda m: np.zeros(max(m, 1), np.uint8)
    mem = np.array([t.members for t in txs] or [[0]], np.uint32).reshape(-1)
    v, eb, iss, st = z(n), z(64 * ANONIMITY_SIZE * n), z(64 * n), z(n)
    nb, npd, nf = z(64 * n_acct), z(64 * n_acct), z(n_acct)
    keep = [buf(ky), buf(bal), buf(pend), buf(fl), buf(kind), mem, buf(b"".join(t.points() for t in txs)),
            buf(b"".join(t.rvk + t.nonce for t in txs)), buf(fields), buf(ge), buf(proofs)]
    args = ([n_acct] + [_p(a) for a in keep[:4]] + [n] + [_p(a) for a in keep[4:8]] + [_p(keep[8]) if has_issue else None] +
            [_p(a) for a in keep[9:]] + [_p(x) for x in (v, eb, iss, st, nb, npd, nf)])

    def result():
        issued = [iss[64 * k:64 * k + 64].tobytes() if kind[k] == ANON_ISSUE and st[k] == BLOCK_APPLIED else None for k in range(n)]
        return ([int(x) for x in v[:n]], (nb[:64 * n_acct].tobytes(), npd[:64 * n_acct].tobytes(), nf[:n_acct].tobytes()),
                eb[:64 * ANONIMITY_SIZE * n].tobytes(), issued)
    return args, result, keep


def anonymous_import(ctx: Context, anon_pvk: PreparedVerifyingKey, conf_pvk: PreparedVerifyingKey, accounts, txs, g_epoch, proofs):
    """import_anonymous_calls_block in one call (zk_import_anonymous_block): the issue rows, both verifications, the verdict
    scatters and both state passes run on the device between one upload and one download, with the proofs checked on
    ctx.  Same arguments, result and errors (conf_pvk may be None when the block has no issue), except that a key of
    another shape raises SynthesisError(MalformedVerifyingKey) even when the block does not use it."""
    args, result, _keep = _anon_section("anonymous_import", accounts, txs, g_epoch, proofs)
    for pvk in (anon_pvk, conf_pvk):
        if pvk is not None and pvk.ctx is not ctx:
            pvk.ctx.sync()
    try:
        _ck(_lib.lib().zk_import_anonymous_block(ctx._h, anon_pvk._h, conf_pvk._h if conf_pvk is not None else None, *args))
    except ZkError as e:
        raise _import_error("anonymous_import", e) from None
    return result()


def anonymous_import_device(ctx: Context, anon_pvk: PreparedVerifyingKey, conf_pvk: PreparedVerifyingKey, n_accounts: int, d_keys_ptr: int,
                            d_balances_ptr: int, d_pendings_ptr: int, d_flags_ptr: int, n_tx: int, d_kind_ptr: int, d_members_ptr: int,
                            d_tx_points_ptr: int, d_tx_extra_ptr: int, d_issue_fields_ptr: int, d_g_epoch_ptr: int, d_proofs_ptr: int,
                            d_verdicts_ptr: int, d_enc_balances_ptr: int, d_issued_ptr: int, d_status_ptr: int, d_new_balances_ptr: int,
                            d_new_pendings_ptr: int, d_new_flags_ptr: int):
    """zk_import_anonymous_block_device on device pointers (d_members: uint32; d_kind 0 = every transaction a transfer;
    d_issue_fields: n_tx * 96 bytes, fee | balance at issues, 0 when the block has none; conf_pvk None likewise).  Blocks on
    the context's stream once, and returns with the outputs complete."""
    v = lambda x: C.c_void_p(x) if x else None
    _ck(_lib.lib().zk_import_anonymous_block_device(ctx._h, anon_pvk._h, conf_pvk._h if conf_pvk is not None else None, n_accounts,
                                                    v(d_keys_ptr), v(d_balances_ptr), v(d_pendings_ptr), v(d_flags_ptr), n_tx, v(d_kind_ptr),
                                                    v(d_members_ptr), v(d_tx_points_ptr), v(d_tx_extra_ptr), v(d_issue_fields_ptr),
                                                    v(d_g_epoch_ptr), v(d_proofs_ptr), v(d_verdicts_ptr), v(d_enc_balances_ptr),
                                                    v(d_issued_ptr), v(d_status_ptr), v(d_new_balances_ptr), v(d_new_pendings_ptr),
                                                    v(d_new_flags_ptr)))


class BadSignature(ZkError):
    """zk_import_block's ZK_ERR_BAD_SIGNATURE: extrinsic .index is the lowest whose signature fails, with the
    redjubjub_verify verdict .verdict (0 / 2 / 3 / 4).  The block is invalid and nothing of it was applied."""

    def __init__(self, code, msg, index: int, verdict: int):
        super().__init__(code, msg)
        self.index, self.verdict = index, verdict


BlockImport = collections.namedtuple("BlockImport", "confidential assets anonymous launches")
_BLOCK_SECTIONS = ("confidential", "assets", "anonymous")


def _block_error(e: ZkError, first_bad: int):
    """zk_import_block's errors as the sections' own calls raise them, with the section named"""
    msg = str(e)
    if e.code == _lib.ZK_ERR_BAD_SIGNATURE:
        m = re.search(r"verdict (\d+)", msg)
        return BadSignature(e.code, _lib.lib().zk_last_error().decode(), first_bad, int(m.group(1)))
    for sec in _BLOCK_SECTIONS:
        if ": %s: " % sec in msg:
            name = "block_import: " + sec
            return _asset_error(name, e) if sec == "assets" else _import_error(name, e)
    return e


def block_import(ctx: Context, conf_pvk: PreparedVerifyingKey, anon_pvk: PreparedVerifyingKey, signatures, confidential=None, assets=None,
                 anonymous=None) -> BlockImport:
    """A block's extrinsic signatures and the zk calls of all three pallets in one call (zk_import_block), with the
    verifier launches the sections' data allow shared between them.
    signatures: (vks, sigs, msgs, zs) as redjubjub_batch_verify takes them, one per extrinsic (zs None: drawn with
    random_batch_scalars).  confidential: (accounts, txs, proofs) as confidential_import takes them; assets: (state, txs,
    proofs, next_asset_id, new_slot_flags) as asset_calls_import; anonymous: (accounts, txs, g_epoch, proofs) as
    anonymous_import.  None: the block has no such section.  conf_pvk / anon_pvk may be None where no section uses them.
    Returns BlockImport: .confidential, .assets and .anonymous hold exactly what those functions return on their section
    (None for an absent one), .launches the verifier launches made.  Raises BadSignature when an extrinsic's signature
    fails (nothing is applied), and the sections' own errors, their ValueErrors named "block_import: <section>"."""
    vks, sigs, msgs, zs = signatures
    vk, sg = _cat(vks, 32), _cat(sigs, 64)
    n_sig = len(msgs)
    assert len(vk) == 32 * n_sig and len(sg) == 64 * n_sig
    z = random_batch_scalars(n_sig) if zs is None else _cat(zs, 32)
    assert len(z) == 32 * n_sig
    buf = lambda b: np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
    sig_keep = [buf(vk), buf(sg), buf(b"".join(bytes(m) for m in msgs)), message_offsets(msgs), buf(z)]
    sections = []
    for sec, make, name in ((confidential, _conf_section, "confidential"), (assets, _asset_section, "assets"),
                            (anonymous, _anon_section, "anonymous")):
        if sec is None:
            sections.append(None)
            continue
        sections.append(make("block_import: " + name, *sec))
    # an absent section: zero sizes and NULL pointers (the asset one's n_slots_out still written)
    n_out = C.c_size_t(0)
    empty = ([0, None, None, None, 0] + [None] * 11,
             [0] + [None] * 5 + [0, 0, 0] + [None] * 15 + [C.byref(n_out), None],
             [0, None, None, None, None, 0] + [None] * 14)
    args = []
    for s, e in zip(sections, empty):
        args += s[0] if s is not None else e
    for pvk in (conf_pvk, anon_pvk):
        if pvk is not None and pvk.ctx is not ctx:
            pvk.ctx.sync()
    first, launches = C.c_size_t(n_sig), C.c_uint(0)
    try:
        _ck(_lib.lib().zk_import_block(ctx._h, conf_pvk._h if conf_pvk is not None else None, anon_pvk._h if anon_pvk is not None else None,
                                       n_sig, *[_p(a) for a in sig_keep], *args, C.byref(first), C.byref(launches)))
    except ZkError as e:
        raise _block_error(e, first.value) from None
    out = [s[1]() if s is not None else None for s in sections]
    return BlockImport(*out, launches.value)


def block_import_device(ctx: Context, conf_pvk: PreparedVerifyingKey, anon_pvk: PreparedVerifyingKey, n_sig: int, d_vks_ptr: int,
                        d_sigs_ptr: int, d_msgs_ptr: int, d_msg_off_ptr: int, d_zs_ptr: int, confidential, assets, anonymous):
    """zk_import_block_device on device pointers.  The signatures as redjubjub_batch_verify_device takes them; confidential,
    assets and anonymous: the arguments of confidential_import_device, asset_calls_import_device and
    anonymous_import_device after their keys, as one tuple each (None: an absent section).  Blocks on the context's
    stream as zk_import_block_device documents.  Returns (confidential rounds, (asset table rows, asset rounds),
    launches), with the outputs complete; raises as block_import."""
    v = lambda x: C.c_void_p(x) if x else None
    c_rounds, a_rounds, n_out, first, launches = C.c_uint(0), C.c_uint(0), C.c_size_t(0), C.c_size_t(n_sig), C.c_uint(0)
    c = list(confidential) if confidential is not None else [0] * 15
    a = list(assets) if assets is not None else [0] * 24
    n = list(anonymous) if anonymous is not None else [0] * 20
    assert (len(c), len(a), len(n)) == (15, 24, 20)
    c_args = [c[0]] + [v(x) for x in c[1:4]] + [c[4]] + [v(x) for x in c[5:]] + [C.byref(c_rounds)]
    a_args = [a[0]] + [v(x) for x in a[1:6]] + [a[6], a[7] & 0xFF, a[8]] + [v(x) for x in a[9:]] + [C.byref(n_out), C.byref(a_rounds)]
    n_args = [n[0]] + [v(x) for x in n[1:5]] + [n[5]] + [v(x) for x in n[6:]]
    try:
        _ck(_lib.lib().zk_import_block_device(ctx._h, conf_pvk._h if conf_pvk is not None else None,
                                              anon_pvk._h if anon_pvk is not None else None, n_sig, v(d_vks_ptr), v(d_sigs_ptr), v(d_msgs_ptr),
                                              v(d_msg_off_ptr), v(d_zs_ptr), *c_args, *a_args, *n_args, C.byref(first), C.byref(launches)))
    except ZkError as e:
        raise _block_error(e, first.value) from None
    return c_rounds.value, (n_out.value, a_rounds.value), launches.value


def pairing(ctx: Context, g1_uncompressed: bytes, g2_uncompressed: bytes) -> bytes:
    """Engine::pairing for len/96 pairs; 576 bytes each in Fq12::write order."""
    n = len(g1_uncompressed) // 96
    assert len(g1_uncompressed) == 96 * n and len(g2_uncompressed) == 192 * n
    out = np.zeros(576 * max(n, 1), np.uint8)
    _ck(_lib.lib().zk_pairing_batch(ctx._h, n, _p(np.frombuffer(g1_uncompressed, np.uint8)), _p(np.frombuffer(g2_uncompressed, np.uint8)), _p(out)))
    return out[:576 * n].tobytes()


class Proof:
    """zerochain_primitives::Proof(Vec<u8>) — the wire wrapper of the 192 proof bytes (core/primitives/src/proof.rs:12-62): the
    runtime moves `Proof` SCALE-encoded (parity_codec derive: Compact<u32> length, then the bytes) and converts to / from
    bellman_verifier::Proof with Proof::read / Proof::write.  Pure byte handling: nothing here touches the device."""
    SIZE = 192

    def __init__(self, raw: bytes):
        self._b = bytes(raw)

    @staticmethod
    def from_slice(raw: bytes) -> "Proof":
        return Proof(raw)

    def as_bytes(self) -> bytes:
        return self._b

    def encode(self) -> bytes:
        """parity_codec::Encode of Vec<u8>: compact length prefix (single / two / four-byte mode), then the bytes."""
        n = len(self._b)
        if n < 1 << 6:
            pre = bytes([n << 2])
        elif n < 1 << 14:
            pre = ((n << 2) | 1).to_bytes(2, "little")
        else:
            assert n < 1 << 30
            pre = ((n << 2) | 2).to_bytes(4, "little")
        return pre + self._b

    @staticmethod
    def decode(buf: bytes) -> "Proof":
        mode = buf[0] & 3
        if mode == 0:
            n, off = buf[0] >> 2, 1
        elif mode == 1:
            n, off = int.from_bytes(buf[:2], "little") >> 2, 2
        elif mode == 2:
            n, off = int.from_bytes(buf[:4], "little") >> 2, 4
        else:
            raise ValueError("big-integer compact lengths do not occur for proofs")
        if len(buf) < off + n:
            raise ValueError("truncated Proof")
        return Proof(buf[off:off + n])

    def __eq__(self, other):
        return isinstance(other, Proof) and self._b == other._b

    def __str__(self):
        return "0x" + self._b.hex()


class ProvingAssignment:
    """What bellman's ProvingAssignment holds after `circuit.synthesize` and the input rows
    (SURVEY.md §3.2): per-constraint evaluations, assignments and the three density maps."""

    def __init__(self, a, b, c, input_assignment, aux_assignment, a_aux_density, b_input_density, b_aux_density):
        self.a, self.b, self.c = (_u64(x, (-1, 4)) for x in (a, b, c))
        self.input_assignment = _u64(input_assignment, (-1, 4))
        self.aux_assignment = _u64(aux_assignment, (-1, 4))
        self.a_aux_density = np.ascontiguousarray(a_aux_density, np.uint8)
        self.b_input_density = np.ascontiguousarray(b_input_density, np.uint8)
        self.b_aux_density = np.ascontiguousarray(b_aux_density, np.uint8)


def _fr_limbs(x: int):
    return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], np.uint64)


def create_proof(prover: ProvingAssignment, params: Parameters, r: int, s: int) -> bytes:
    """groth16::create_proof(circuit, params, r, s) below synthesis -> Proof::write bytes (192 B)."""
    out = np.zeros(192, np.uint8)
    rr, ss = _fr_limbs(r), _fr_limbs(s)
    L = _lib.lib()
    _ck(L.zk_groth16_prove(params.ctx._h, params._h, _p(prover.a), _p(prover.b), _p(prover.c), prover.a.shape[0],
                           _p(prover.input_assignment), prover.input_assignment.shape[0],
                           _p(prover.aux_assignment), prover.aux_assignment.shape[0],
                           _p(prover.a_aux_density), _p(prover.b_input_density), _p(prover.b_aux_density),
                           _p(rr), _p(ss), _p(out)))
    return out.tobytes()


def create_random_proof(prover: ProvingAssignment, params: Parameters, rng=None) -> bytes:
    """groth16::create_random_proof: draws r, s uniformly in Fr (Fr::rand, fr.rs:255-267) then create_proof."""
    draw = (lambda: secrets.randbelow(R_MODULUS)) if rng is None else (lambda: rng.randrange(R_MODULUS))
    return create_proof(prover, params, draw(), draw())


def create_proof_batch(provers, params: Parameters, rs, ss) -> bytes:
    """`len(provers)` witnesses of the same circuit in one device pass; returns batch*192 bytes."""
    p0 = provers[0]
    batch = len(provers)
    cat = lambda name: np.ascontiguousarray(np.concatenate([getattr(p, name) for p in provers], axis=0))
    a, b, c, inp, aux = (cat(k) for k in ("a", "b", "c", "input_assignment", "aux_assignment"))
    rr = np.stack([_fr_limbs(x) for x in rs]); sv = np.stack([_fr_limbs(x) for x in ss])
    out = np.zeros(192 * batch, np.uint8)
    _ck(_lib.lib().zk_groth16_prove_batch(params.ctx._h, params._h, batch, _p(a), _p(b), _p(c), p0.a.shape[0],
                                          _p(inp), p0.input_assignment.shape[0], _p(aux), p0.aux_assignment.shape[0],
                                          _p(p0.a_aux_density), _p(p0.b_input_density), _p(p0.b_aux_density),
                                          _p(rr), _p(sv), _p(out)))
    return out.tobytes()


class ConstraintSystem:
    """The fixed R1CS of a circuit resident on the device (CSR), so proofs can be made straight from assignments
    (zk_groth16_prove_witness_batch).  rows_*: per constraint a list of (variable, coefficient) with variable < n_inputs
    for inputs and n_inputs + i for aux i — the at/bt/ct that bellman's KeypairAssembly collects."""

    def __init__(self, ctx: Context, n_inputs: int, n_aux: int, rows_a, rows_b, rows_c):
        self.ctx, self.n_inputs, self.n_aux = ctx, n_inputs, n_aux
        n_c = len(rows_a)
        assert len(rows_b) == n_c and len(rows_c) == n_c
        arrs = []
        for rows in (rows_a, rows_b, rows_c):
            rp = np.zeros(n_c + 1, np.uint32)
            rp[1:] = np.cumsum([len(r) for r in rows])
            col = np.array([v for r in rows for v, _ in r] or [0], np.uint32)
            cf = np.zeros((max(1, int(rp[-1])), 4), np.uint64)
            k = 0
            for r in rows:
                for _, c in r:
                    for j in range(4):
                        cf[k, j] = (c >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
                    k += 1
            arrs += [rp, col, cf]
        self._h = C.c_void_p()
        _ck(_lib.lib().zk_r1cs_load(ctx._h, n_c, n_inputs, n_aux, *[_p(a) for a in arrs], C.byref(self._h)))

    def free(self):
        if self._h:
            _lib.lib().zk_r1cs_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def create_proof_from_witness_batch(cs: ConstraintSystem, params: Parameters, batch: int, inputs, aux, r, s) -> bytes:
    """inputs [batch][n_inputs][4], aux [batch][n_aux][4] canonical; r, s [batch][4] -> batch * 192 bytes."""
    inputs, aux = _u64(inputs, (batch, cs.n_inputs, 4)), _u64(aux, (batch, cs.n_aux, 4))
    r, s = _u64(r, (batch, 4)), _u64(s, (batch, 4))
    out = np.zeros(192 * batch, np.uint8)
    _ck(_lib.lib().zk_groth16_prove_witness_batch(params.ctx._h, params._h, cs._h, batch, _p(inputs), _p(aux), _p(r), _p(s), _p(out)))
    return out.tobytes()


def create_proof_batch_raw(params: Parameters, batch: int, a, b, c, inputs, aux, a_aux_density, b_input_density, b_aux_density, r, s) -> bytes:
    """Same as create_proof_batch with the per-proof arrays already concatenated ([batch][n][4] uint64, e.g. views
    of pinned host memory): exactly one zk_groth16_prove_batch call, no host-side copies."""
    a, b, c, inputs, aux = (_u64(x, (batch, -1, 4)) for x in (a, b, c, inputs, aux))
    r, s = _u64(r, (batch, 4)), _u64(s, (batch, 4))
    d1, d2, d3 = (np.ascontiguousarray(x, np.uint8) for x in (a_aux_density, b_input_density, b_aux_density))
    out = np.zeros(192 * batch, np.uint8)
    _ck(_lib.lib().zk_groth16_prove_batch(params.ctx._h, params._h, batch, _p(a), _p(b), _p(c), a.shape[1],
                                          _p(inputs), inputs.shape[1], _p(aux), aux.shape[1], _p(d1), _p(d2), _p(d3), _p(r), _p(s), _p(out)))
    return out.tobytes()


# ---- utilities ---------------------------------------------------------------------------------------
def scalar_mul_many(ctx: Context, group: int, base_limbs, scalars):
    s = _u64(scalars, (-1, 4))
    w = 12 if group == 1 else 24
    base = _u64(base_limbs, (w,))
    out = np.zeros((s.shape[0], w), np.uint64)
    _ck(_lib.lib().zk_scalar_mul_many(ctx._h, group, _p(base), _p(s), s.shape[0], _p(out)))
    return out


FIELD_FQ, FIELD_FR = 0, 1
OP_MUL, OP_ADD, OP_SUB, OP_SQR, OP_INV, OP_FROM_REPR, OP_INTO_REPR = range(7)


def field_op(ctx: Context, field: int, op: int, a, b=None):
    nl = 6 if field == 0 else 4
    a = _u64(a, (-1, nl))
    bb = None if b is None else _u64(b, (-1, nl))
    out = np.zeros_like(a)
    _ck(_lib.lib().zk_field_op(ctx._h, field, op, _p(a), _p(bb) if bb is not None else None, a.shape[0], _p(out)))
    return out


def bench_modmul(ctx: Context, field: int, blocks: int, threads: int, iters: int):
    per_s, ms = C.c_double(), C.c_double()
    _ck(_lib.lib().zk_bench_modmul(ctx._h, field, blocks, threads, iters, C.byref(per_s), C.byref(ms)))
    return per_s.value, ms.value


# constants of the generators in limb form (Montgomery; fq.rs:85-136) for building synthetic inputs
G1_GENERATOR = np.array([0x5cb38790fd530c16, 0x7817fc679976fff5, 0x154f95c7143ba1c1, 0xf0ae6acdf3d0e747, 0xedce6ecc21dbf440, 0x120177419e0bfb75,
                         0xbaac93d50ce72271, 0x8c22631a7918fd8e, 0xdd595f13570725ce, 0x51ac582950405194, 0x0e1c8c3fad0059c0, 0x0bbc3efc5008a26a], np.uint64)
G2_GENERATOR = np.array([0xf5f28fa202940a10, 0xb3f5fb2687b4961a, 0xa1a893b53e2ae580, 0x9894999d1a3caee9, 0x6f67b7631863366b, 0x058191924350bcd7,
                         0xa5a9c0759e23f606, 0xaaa0c59dbccd60c3, 0x3bb17e18e2867806, 0x1b1ab6cc8541b367, 0xc2b6ed0ef2158547, 0x11922a097360edf3,
                         0x4c730af860494c4a, 0x597cfa1f5e369c5a, 0xe7e6856caa0a635a, 0xbbefb5e96e0d495f, 0x07d3a975f0ef25a2, 0x0083fd8e7e80dae5,
                         0xadc0fc92df64b05d, 0x18aa270a2b1461dc, 0x86adac6a3be4eba0, 0x79495c4ec93da33a, 0xe7175850a43ccaed, 0x0b2bc2a163de1bf2], np.uint64)
