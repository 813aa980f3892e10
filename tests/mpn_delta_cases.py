"""TEST INFRASTRUCTURE: how a full node applies the MPN contract's state delta of a block, restated leaf by leaf, and the
scenarios both tiers run against bzk_mpn_state_apply_delta (csrc/mpn_host.cu).

`LeafState` is the reference's `KvStoreStateManager::update_contract` (/root/reference/src/zk/state/mod.rs:285-308) over the
sparse MPN state model of oracle/py/state.py: every entry is one `set_data` (:310-420) that re-hashes its token leaf, the token
tree path, the account leaf and the state tree path, one hash after the other; `index_mpn_accounts`
(/root/reference/src/blockchain/ops/apply_tx/mod.rs:14-56) runs first.  Plain Python, entry by entry, in the order given."""
import ctypes as ct
import random

import numpy as np

from oracle.py import state as S
from oracle.py.poseidon import poseidon as _poseidon

from bazuka_b200.mpn import native as N, update as U, wire as Wr, works as Wk
from bazuka_b200.mpn.ledger import NativeLedger

R = N.R


class Inconsistency(ValueError):
    pass


class LeafState:
    def __init__(self, A, T, hash_=_poseidon):
        self.A, self.T, self.h = A, T, hash_
        model = S.mpn_state_model(A, T)
        acct, tok = model[2], model[2][1][4]
        self.tdef = [S.compress_default(tok[2])]
        for _ in range(T):
            self.tdef.append(hash_([self.tdef[-1]] * 4))
        self.sdef = [S.compress_default(acct)]
        for _ in range(A):
            self.sdef.append(hash_([self.sdef[-1]] * 4))
        self.leaves, self.tok, self.st = {}, {}, {}   # non-zero scalars by locator; non-default tree nodes
        self.state_size, self.account_count = 0, 0
        self.index = {}                               # (x, y) -> indices recorded for it (never pruned)

    @property
    def root(self):
        return self.st.get((self.A, 0), self.sdef[self.A])

    def _put(self, tree, key, value, default):
        if value == default:
            tree.pop(key, None)
        else:
            tree[key] = value

    def set_data(self, loc, value):
        loc = tuple(loc)
        prev = self.leaves.get(loc, 0)
        if prev == value:
            return
        if value == 0:
            del self.leaves[loc]
            self.state_size -= 1
        else:
            self.leaves[loc] = value
            self.state_size += prev == 0
        i, A, T, L = loc[0], self.A, self.T, self.leaves
        if len(loc) == 4:   # the token struct, then the token list's path
            node = loc[2]
            cur = self.h([L.get((i, 4, node, 0), 0), L.get((i, 4, node, 1), 0)])
            self._put(self.tok, (i, 0, node), cur, self.tdef[0])
            for lvl in range(T):
                node >>= 2
                cur = self.h([self.tok.get((i, lvl, 4 * node + k), self.tdef[lvl]) for k in range(4)])
                self._put(self.tok, (i, lvl + 1, node), cur, self.tdef[lvl + 1])
        cur = self.h([L.get((i, f), 0) for f in range(4)] + [self.tok.get((i, T, 0), self.tdef[T])])
        node = i
        self._put(self.st, (0, node), cur, self.sdef[0])
        for lvl in range(A):
            node >>= 2
            cur = self.h([self.st.get((lvl, 4 * node + k), self.sdef[lvl]) for k in range(4)])
            self._put(self.st, (lvl + 1, node), cur, self.sdef[lvl + 1])

    def index_accounts(self, entries):
        org = {}
        for loc, v in entries:
            if len(loc) == 2 and loc[1] in (2, 3):
                org.setdefault(loc[0], {}).setdefault(loc[1], v or 0)
        for i, d in org.items():
            if 2 not in d or 3 not in d:
                raise Inconsistency(i)
        count = self.account_count
        for i in sorted(org):
            if i == count:
                count += 1
            elif i > count:
                raise Inconsistency(i)
        for i, d in org.items():
            self.index.setdefault((d[2], d[3]), set()).add(i)
        self.account_count = count

    def apply(self, entries):
        """entries: [(locator, value | None)] in the order of the map's iteration"""
        self.index_accounts(entries)
        for loc, v in entries:
            self.set_data(loc, v or 0)


def encode(entries):
    """bincode of ZkDeltaPairs with the entries in the given order; a value is None, an int (canonical) or 32 raw bytes"""
    w = Wr.Writer()
    w.u64(len(entries))
    for loc, v in entries:
        w.vec(list(loc), lambda w_, x: w_.u64(x))
        if isinstance(v, (bytes, bytearray)):
            w.u8(1)
            w.raw(v)
        else:
            w.option(v, lambda w_, x: w_.fr(x))
    return bytes(w.b)


def ptr(a):
    return ct.c_void_p(a.ctypes.data)


def wrap(ctx, h, A, T):
    led = NativeLedger.__new__(NativeLedger)
    led.ctx, led.A, led.T, led._h = ctx, A, T, h
    w = ct.c_uint32()
    ctx._check(ctx._l.bzk_mpn_update_raw_width(A, T, ct.byref(w)))
    led.n_raw = w.value
    return led


def delta_bytes(a, b):
    """bzk_mpn_state_delta(a, b) -> (image, entries)"""
    lib = a.ctx._l
    buf, ln, n = ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
    assert lib.bzk_mpn_state_delta(a._h, b._h, ct.byref(buf), ct.byref(ln), ct.byref(n)) == 0
    out = ct.string_at(buf, ln.value)
    lib.bzk_buffer_free(buf)
    return out, n.value


def apply_raw(led, image, expect_hash=None, expect_size=None):
    """-> (status, entries, last error text)"""
    ctx = led.ctx
    hb = np.frombuffer((expect_hash % R).to_bytes(32, "little"), np.uint64).copy() if expect_hash is not None else None
    sz = ct.c_uint64(expect_size) if expect_size is not None else None
    n = ct.c_uint64()
    st = ctx._l.bzk_mpn_state_apply_delta(ctx._h, led._h, image, len(image), ptr(hb) if hb is not None else None,
                                          ct.byref(sz) if sz is not None else None, ct.byref(n))
    err = ctx._l.bzk_last_error(ctx._h)
    return st, n.value, (err or b"").decode()


def same_ledger(a, b):
    """equal info and no scalar leaf differs"""
    return a.info() == b.info() and delta_bytes(a, b)[1] == 0


def load(ctx, st, A, T):
    led = NativeLedger(ctx, A, T)
    for i, a in st.accounts.items():
        led.set_account(i, a)
    return led


def oracle_of(st, A, T):
    o = LeafState(A, T)
    o.apply(list(Wk.final_delta(U.MpnState(A, T), st).items()))
    assert o.root == st.root
    return o


# ------------------------------------------------------------------ blocks through bzk_mpn_prepare_works
def run_block(ctx, led, config, deps, wds, ups, dpay=None, wpay=None):
    """bzk_mpn_prepare_works on `led` -> (GetMpnWorkResponse image, fork ledger, number of works)"""
    lib = ctx._l

    def vec(items, enc):
        w = Wr.Writer()
        w.vec(items, enc)
        return bytes(w.b)
    cw = Wr.Writer()
    Wr.enc_config(cw, config)
    cb = bytes(cw.b)
    dpay = dpay or {}
    wpay = wpay or {}
    db = vec([{"mpn_address": tuple(d.mpn_address), "payment": dpay[k]} for k, d in enumerate(deps)],
             Wr.enc_mpn_deposit) if deps else b""
    wb = vec([{"mpn_address": tuple(w.mpn_address), "mpn_withdraw_nonce": w.mpn_withdraw_nonce, "mpn_sig": {"r": tuple(w.mpn_sig["r"]), "s": w.mpn_sig["s"]},
               "payment": wpay[k]} for k, w in enumerate(wds)], Wr.enc_mpn_withdraw) if wds else b""
    ub = vec([{"nonce": t.nonce, "src_pub_key": tuple(t.src_pub_key), "dst_pub_key": tuple(t.dst_pub_key), "amount": Wk._money_w(t.amount),
               "fee": Wk._money_w(t.fee), "sig": {"r": tuple(t.sig["r"]), "s": t.sig["s"]}} for t in ups], Wr.enc_mpn_tx) if ups else b""
    rw = np.array([11, 22, 33], np.uint64)
    fee = np.frombuffer((U.ZIESHA % R).to_bytes(32, "little"), np.uint64).copy()
    fork, buf, ln, n = ct.c_void_p(), ct.c_void_p(), ct.c_size_t(), ct.c_uint64()
    ctx._check(lib.bzk_mpn_prepare_works(ctx._h, led._h, cb or None, len(cb), db or None, len(db), wb or None, len(wb), ub or None, len(ub), ptr(rw), 9,
                                         ptr(fee), ct.byref(fork), ct.byref(buf), ct.byref(ln), ct.byref(n)))
    out = ct.string_at(buf, ln.value)
    lib.bzk_buffer_free(buf)
    return out, wrap(ctx, fork, led.A, led.T), n.value


def check_block_round_trip(ctx, led, config, deps, wds, ups, dpay=None, wpay=None, next_block=None):
    """apply(clone(led), final_delta(led, fork)) equals the fork after commit_accounts; the next block's works agree byte for
    byte.  Returns the applied ledger's info."""
    _, fork, _ = run_block(ctx, led, config, deps, wds, ups, dpay, wpay)
    image, n = delta_bytes(led, fork)
    assert n > 0
    fork.commit_accounts()
    applied = led.fork()
    assert applied.apply_delta(image, expect={"state_hash": fork.info()["state_hash"], "state_size": fork.info()["state_size"]}) == n
    assert applied.info() == fork.info() and delta_bytes(applied, fork)[1] == 0
    if next_block is not None:
        a, fa, _ = run_block(ctx, applied, *next_block)
        b, fb, _ = run_block(ctx, fork, *next_block)
        assert a == b and fa.info() == fb.info()
        fa.free(); fb.free()
    info = applied.info()
    applied.free(); fork.free()
    return info


# ------------------------------------------------------------------ random deltas
def _rand_fr(rng):
    return rng.randrange(1, R)


def random_accounts(rng, n, T, A):
    st = U.MpnState(A, T)
    for i in range(n):
        toks = {s: U.Money(_rand_fr(rng), rng.randrange(0, 1 << 64)) for s in rng.sample(range(4 ** T), rng.randrange(0, 4))}
        st.set(i, U.MpnAccount(rng.randrange(0, 1 << 64), rng.randrange(0, 1 << 64), (_rand_fr(rng), _rand_fr(rng)), toks))
    return st


def random_delta(rng, st, count, T, A):
    """a valid delta over `st`: accounts created (next indices), emptied, re-keyed, nonces bumped, token slots toggled, None and
    explicit zeros -> list of (locator, value | None)"""
    d = {}
    n = count
    accs = sorted(st.accounts)
    for i in rng.sample(accs, min(len(accs), 6)):
        a = st.accounts[i]
        kind = rng.randrange(4)
        if kind == 0:                                  # emptied: every non-zero leaf removed, x / y as None or explicit 0
            for f, v in enumerate((a.tx_nonce, a.withdraw_nonce, a.address[0], a.address[1])):
                if v or f in (2, 3):
                    d[(i, f)] = rng.choice([None, 0])
            for s, m in a.tokens.items():
                d[(i, 4, s, 0)] = None
                if m.amount:
                    d[(i, 4, s, 1)] = rng.choice([None, 0])
        elif kind == 1:                                # re-keyed
            d[(i, 2)], d[(i, 3)] = _rand_fr(rng), _rand_fr(rng)
        elif kind == 2:                                # nonces
            d[(i, 0)] = rng.randrange(0, 1 << 64) or None
            d[(i, 1)] = 0
        for s in rng.sample(range(4 ** T), 2):         # token slots toggled
            if s in a.tokens:
                d[(i, 4, s, 0)] = None
                d[(i, 4, s, 1)] = rng.choice([None, 0])
            elif (i, 4, s, 0) not in d:
                d[(i, 4, s, 0)] = _rand_fr(rng)
                d[(i, 4, s, 1)] = rng.choice([rng.randrange(1, 1 << 64), 0, None])
    for i in range(n, n + rng.randrange(0, 4)):        # created
        d[(i, 2)], d[(i, 3)] = _rand_fr(rng), _rand_fr(rng)
        d[(i, 0)] = rng.randrange(1, 1 << 64)
        s = rng.randrange(4 ** T)
        d[(i, 4, s, 0)], d[(i, 4, s, 1)] = _rand_fr(rng), rng.randrange(0, 1 << 64)
    return list(d.items())


def check_random_deltas(ctx, seed, rounds, A=3, T=2):
    rng = random.Random(seed)
    st = random_accounts(rng, 12, T, A)
    led, orc = load(ctx, st, A, T), oracle_of(st, A, T)
    assert led.info()["account_count"] == orc.account_count
    for r in range(rounds):
        cur = _as_state(orc, A, T)
        entries = random_delta(rng, cur, orc.account_count, T, A)
        orc.apply(entries)
        infos = []
        for k in range(3):                             # the same delta in shuffled orders
            e = list(entries)
            rng.shuffle(e)
            c = led.fork()
            assert c.apply_delta(encode(e)) == len(e)
            infos.append(c.info())
            if k == 2:
                led.free()
                led = c
            else:
                c.free()
        assert infos[0] == infos[1] == infos[2]
        assert (infos[0]["state_hash"], infos[0]["state_size"], infos[0]["account_count"]) == (orc.root, orc.state_size, orc.account_count), r
    led.free()


def _as_state(orc, A, T):
    """the oracle's leaves as an MpnState (accounts only; for drawing the next delta)"""
    st = U.MpnState.__new__(U.MpnState)
    st.accounts = {}
    by = {}
    for loc, v in orc.leaves.items():
        by.setdefault(loc[0], {})[loc[1:]] = v
    for i, lv in by.items():
        toks = {}
        for k, v in lv.items():
            if len(k) == 3:
                toks.setdefault(k[1], [0, 0])[k[2]] = v
        st.accounts[i] = U.MpnAccount(lv.get((0,), 0), lv.get((1,), 0), (lv.get((2,), 0), lv.get((3,), 0)),
                                      {s: U.Money(t[0], t[1]) for s, t in toks.items() if t[0]})
    return st


# ------------------------------------------------------------------ refusals
def refusal_cases(A, T, count):
    """(name, image, expected substring of the error) for every refusal; `count` = the ledger's account count"""
    ok = [((0, 0), 5)]
    cases = []
    img = encode(ok)
    cases.append(("truncated", img[:-1], "truncated"))
    cases.append(("trailing", img + b"\x00", "trailing"))
    cases.append(("count beyond the image", encode([]) [:0] + (5).to_bytes(8, "little"), "truncated"))
    bad_tag = bytearray(img)
    bad_tag[8 + 8 + 16] = 2
    cases.append(("option tag", bytes(bad_tag), "option tag 2"))
    cases.append(("duplicate", encode([((0, 0), 5), ((1, 1), 2), ((0, 0), 6)]), "entry 2: duplicate locator [0, 0] (entry 0)"))
    cases.append(("short locator", encode([((0,), 5)]), "entry 0: a locator of 1 elements"))
    cases.append(("three-element locator", encode([((0, 4, 1), 5)]), "entry 0: a locator of 3 elements"))
    cases.append(("field 5", encode([((0, 0), 1), ((0, 5), 5)]), "entry 1: locator [0, 5] is not an account scalar"))
    cases.append(("token field 2", encode([((0, 4, 0, 2), 5)]), "is not a token leaf"))
    cases.append(("not a token list", encode([((0, 3, 0, 0), 5)]), "is not a token leaf"))
    cases.append(("slot out of range", encode([((0, 0), 1), ((5, 4, 4 ** T + 6, 0), 3)]), "entry 1: locator [5, 4, %d, 0] outside the token tree" % (4 ** T + 6)))
    cases.append(("account out of range", encode([((4 ** A, 0), 1)]), "outside the state tree"))
    cases.append(("non-canonical", encode([((0, 0), R.to_bytes(32, "little"))]), "not canonical"))
    cases.append(("non-canonical high", encode([((0, 2), b"\xff" * 32)]), "not canonical"))
    cases.append(("nonce >= 2^64", encode([((0, 0), 1 << 64)]), "does not fit in 64 bits"))
    cases.append(("withdraw nonce >= 2^64", encode([((1, 1), R - 1)]), "does not fit in 64 bits"))
    cases.append(("balance >= 2^64", encode([((0, 4, 3, 0), 9), ((0, 4, 3, 1), 1 << 64)]), "does not fit in 64 bits"))
    cases.append(("balance under id zero", encode([((2, 4, 7, 1), 5)]), "token slot 7 holds balance 5 under token id zero"))
    cases.append(("x without y", encode([((count, 2), 5)]), "sets its x but not its y"))
    cases.append(("y without x", encode([((0, 3), 5)]), "sets its y but not its x"))
    cases.append(("index above the count", encode([((count + 1, 2), 5), ((count + 1, 3), 6)]), "above the account count"))
    cases.append(("gap after a new index", encode([((count, 2), 5), ((count, 3), 6), ((count + 2, 2), 5), ((count + 2, 3), 6)]), "above the account count"))
    return cases


def check_refusals(ctx, led):
    """every refusal returns BZK_ERR_BAD_ARG, names its reason and leaves the ledger identical.  `led`: accounts 0..count-1 holding
    token slot 0 only (test_mpn_cpu.make_state), so that slots 3 and 7 are free"""
    before = led.fork()
    info = led.info()
    for name, image, want in refusal_cases(led.A, led.T, info["account_count"]):
        st, _, err = apply_raw(led, image)
        assert st == -1 and want in err, (name, st, err)
        assert same_ledger(led, before), name
    # the root / size check: the same valid delta with a wrong expectation
    image = encode([((0, 0), 123456)])
    probe = led.fork()
    probe.apply_delta(image)
    good = probe.info()
    probe.free()
    for h, s in ((good["state_hash"] ^ 1, None), (None, good["state_size"] + 1), (good["state_hash"] ^ 1, good["state_size"])):
        st, _, err = apply_raw(led, image, h, s)
        assert st == -1 and "expected" in err, err
        assert same_ledger(led, before)
    st, n, _ = apply_raw(led, image, good["state_hash"], good["state_size"])
    assert st == 0 and n == 1 and led.info() == good
    # a ledger with a prepare_works fork's new accounts is not the chain's ledger
    from bazuka_b200.mpn import dw as D
    fork = before.fork()
    fork.deposit_build([D.MpnDeposit(N.jj_compress(N.eddsa_keys(b"refusal-new")[0]), U.ZIESHA, 5)], 1)
    assert fork.info()["pending_accounts"] == 1
    pre = fork.fork()
    st, _, err = apply_raw(fork, encode([((0, 0), 7)]))
    assert st == -1 and "prepare_works fork" in err and same_ledger(fork, pre)
    fork.commit_accounts()
    st, _, _ = apply_raw(fork, encode([((0, 0), 7)]))
    assert st == 0
    fork.free(); pre.free(); before.free()


# ------------------------------------------------------------------ snapshots
def check_snapshot(ctx, n, A=5, T=2, seed=7):
    """a ledger built with set_account, its image bzk_mpn_state_delta(empty, ledger) applied to a fresh ledger: equal"""
    rng = random.Random(seed)
    st = random_accounts(rng, n, T, A)
    built = load(ctx, st, A, T)
    empty = NativeLedger(ctx, A, T)
    image, entries = delta_bytes(empty, built)
    assert empty.apply_delta(image) == entries
    assert empty.info() == built.info() and delta_bytes(empty, built)[1] == 0
    assert (empty.info()["state_hash"], empty.info()["state_size"]) == (st.root, st.state_size)
    # the dict form of the same snapshot
    again = NativeLedger(ctx, A, T)
    assert again.apply_delta(Wk.final_delta(U.MpnState(A, T), st)) == entries and again.info() == built.info()
    for x in (built, empty, again):
        x.free()


# ------------------------------------------------------------------ large snapshots, encoded with numpy
_R_TOP = R >> 192
_RINV = pow(1 << 256, -1, R)
_E2 = np.dtype([("len", "<u8"), ("i", "<u8"), ("f", "<u8"), ("tag", "u1"), ("v", "<u8", 4)])                         # [i, f]: 57 bytes
_E4 = np.dtype([("len", "<u8"), ("i", "<u8"), ("four", "<u8"), ("slot", "<u8"), ("k", "<u8"), ("tag", "u1"), ("v", "<u8", 4)])   # 73 bytes


def _mont_table(values):
    return np.array([list(np.frombuffer(((v << 256) % R).to_bytes(32, "little"), np.uint64)) for v in values], np.uint64)


def _mix(z):
    """SplitMix64's finaliser, elementwise (uint64 arithmetic wraps)"""
    z = (z + np.uint64(0x9E3779B97F4A7C15)) ^ ((z + np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(30))
    z = z * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _rand_limbs(key):
    """a canonical non-zero Montgomery image per key (uint64 array), a function of the key alone"""
    v = _mix(key[..., None] * np.uint64(4) + np.arange(4, dtype=np.uint64))
    v[..., 3] %= np.uint64(_R_TOP)            # below r
    v[..., 0] |= np.uint64(1)                 # non-zero
    return v


_NONCES, _AMOUNTS = _mont_table(range(1, 1001)), _mont_table(range(1, 1025))


def snapshot_accounts(lo, n, T, seed=11):
    """accounts lo .. lo+n-1 of a deterministic synthetic ledger: 1-4 tokens each; every value depends on the index only.
    -> dict of arrays (Montgomery limbs)"""
    i = np.arange(lo, lo + n, dtype=np.uint64)
    key = i * np.uint64(8) + np.uint64(seed << 40)
    ntok = (i % np.uint64(4)) + np.uint64(1)
    j = np.arange(4, dtype=np.uint64)
    slots = (i[:, None] * np.uint64(7) + j[None, :] * np.uint64(13)) % np.uint64(4 ** T)
    return {"i": i, "ntok": ntok, "slots": slots, "x": _rand_limbs(key), "y": _rand_limbs(key + np.uint64(1)),
            "ids": _rand_limbs(key[:, None] + np.uint64(2) + np.arange(4, dtype=np.uint64)[None, :]),
            "tx": _NONCES[i % np.uint64(1000)], "wd": _NONCES[(i * np.uint64(7)) % np.uint64(1000)],
            "amt": _AMOUNTS[(i[:, None] + j[None, :] * np.uint64(101)) % np.uint64(1024)]}


def snapshot_image(lo, n, T, seed=11):
    """bincode ZkDeltaPairs that creates accounts lo .. lo+n-1 of snapshot_accounts (every leaf Some)"""
    a = snapshot_accounts(lo, n, T, seed)
    e2 = np.zeros((n, 4), _E2)
    e2["len"], e2["tag"] = 2, 1
    e2["i"] = a["i"][:, None]
    e2["f"] = np.arange(4, dtype=np.uint64)[None, :]
    for f, key in enumerate(("tx", "wd", "x", "y")):
        e2["v"][:, f] = a[key]
    mask = np.arange(4)[None, :] < a["ntok"][:, None].astype(np.int64)
    e4 = np.zeros((n, 4, 2), _E4)
    e4["len"], e4["four"], e4["tag"] = 4, 4, 1
    e4["i"] = a["i"][:, None, None]
    e4["slot"] = a["slots"][:, :, None]
    e4["k"] = np.arange(2, dtype=np.uint64)[None, None, :]
    e4["v"][:, :, 0] = a["ids"]
    e4["v"][:, :, 1] = a["amt"]
    e4 = e4[mask]
    count = np.array([4 * n + 2 * len(e4)], np.uint64)
    return count.tobytes() + e2.tobytes() + e4.tobytes()


def _canon_of(limbs):
    return int.from_bytes(np.ascontiguousarray(limbs, np.uint64).tobytes(), "little") * _RINV % R


def snapshot_mpn_accounts(lo, n, T, seed=11):
    """the same accounts as update.MpnAccount (for set_account)"""
    a = snapshot_accounts(lo, n, T, seed)
    out = {}
    for k in range(n):
        toks = {int(a["slots"][k, j]): U.Money(_canon_of(a["ids"][k, j]), _canon_of(a["amt"][k, j])) for j in range(int(a["ntok"][k]))}
        out[int(a["i"][k])] = U.MpnAccount(_canon_of(a["tx"][k]), _canon_of(a["wd"][k]), (_canon_of(a["x"][k]), _canon_of(a["y"][k])), toks)
    return out


def parse(image):
    """bincode ZkDeltaPairs -> [(locator, value | None)] (values canonical)"""
    import struct
    o, out = 8, []
    for _ in range(struct.unpack_from("<Q", image, 0)[0]):
        L = struct.unpack_from("<Q", image, o)[0]
        loc = struct.unpack_from("<%dQ" % L, image, o + 8)
        o += 8 + 8 * L
        tag = image[o]
        o += 1
        v = None
        if tag:
            v = int.from_bytes(image[o:o + 32], "little") * _RINV % R
            o += 32
        out.append((tuple(loc), v))
    assert o == len(image)
    return out
