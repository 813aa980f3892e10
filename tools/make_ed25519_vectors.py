#!/usr/bin/env python3
"""Write tests/golden/ed25519_vectors.json with libsodium (PyNaCl), an implementation independent of oracle/py/ed25519.py, so
that the oracle's signing and verdict are pinned to it.  Test infrastructure only: PyNaCl is needed here, never by the product.

  honest   RFC 8032 signatures by seeded keys at message lengths where 64 + |M| (the SHA-512 input R || A || M) crosses the
           padding edges 111, 112, 127, 128, 239, 240, plus |M| = 0 and 4 KiB; each with libsodium's verdict
  reference  the reference's own test (src/crypto/ed25519.rs, test_ed25519_signature_verification): generate_keys(b"ABC")
           (secret = sha3_256(seed) with bit 255 cleared), the signature of b"salam1" accepted, the same on b"salam2" rejected
"""
import hashlib
import json
import os

import nacl
import nacl.bindings as nb

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ed25519_vectors.json")


def keypair(seed32):
    pk, _ = nb.crypto_sign_seed_keypair(seed32)
    return pk, seed32 + pk


def sign(sk64, msg):
    return nb.crypto_sign(msg, sk64)[:64]


def verdict(pk, msg, sig):
    try:
        nb.crypto_sign_open(sig + msg, pk)
        return True
    except Exception:
        return False


def main():
    out = {"source": "libsodium via PyNaCl %s (tools/make_ed25519_vectors.py)" % nacl.__version__, "honest": [], "reference": []}
    lens = [0] + [t - 64 for t in (111, 112, 127, 128, 239, 240)] + [4096]
    for i, n in enumerate(lens):
        seed = hashlib.sha256(b"ed25519-golden-%d" % i).digest()
        pk, sk = keypair(seed)
        msg = bytes((7 * j + i) & 0xFF for j in range(n))
        sig = sign(sk, msg)
        out["honest"].append({"secret": seed.hex(), "pk": pk.hex(), "msg": msg.hex(), "sig": sig.hex(), "ok": verdict(pk, msg, sig)})
    x = bytearray(hashlib.sha3_256(b"ABC").digest())
    x[31] &= 0x7F
    pk, sk = keypair(bytes(x))
    sig = sign(sk, b"salam1")
    for m in (b"salam1", b"salam2"):
        out["reference"].append({"secret": bytes(x).hex(), "pk": pk.hex(), "msg": m.hex(), "sig": sig.hex(), "ok": verdict(pk, m, sig)})
    assert [v["ok"] for v in out["reference"]] == [True, False] and all(v["ok"] for v in out["honest"])
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
