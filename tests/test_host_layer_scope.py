"""acu._Scope, the owner of what one Context call allocates, against a fake context that records every allocation and
release: everything is released in reverse order on normal exit and when the body raises, a failing release never
replaces the exception in flight, and filter-plan handles that were never set are not destroyed."""
import ctypes as C

import numpy as np
import pytest

import acu


class FakeLib:
    def __init__(self, log):
        self.log = log

    def acu_filter_plan_destroy(self, h, plan):
        self.log.append(("destroy", plan.value))


class FakeContext:
    """malloc / free / h2d and the plan destructor; free(p) fails for p in `bad`."""

    def __init__(self, bad=()):
        self.log, self.bad, self.next, self.h = [], set(bad), 0x1000, None
        self.lib = FakeLib(self.log)

    def malloc(self, nbytes):
        p, self.next = self.next, self.next + 0x100
        self.log.append(("malloc", p))
        return p

    def free(self, p):
        self.log.append(("free", p))
        if p in self.bad:
            raise acu.ArrowError(1, f"free {p:#x} failed")

    def h2d(self, p, arr):
        self.log.append(("h2d", p))

    def released(self):
        return [x for x in self.log if x[0] in ("free", "destroy")]


def fill(s):
    """Register one of each kind: allocated and appended pointers, an ArrayOut, a set plan, an unset plan, a host object."""
    a = s.malloc(8)
    b = s.append(0x42)
    out = s.out(16, 10)
    plan = s.plan()
    plan.value = 0xBEEF
    s.plan()
    s.keep.append(object())
    return [("free", a), ("free", b), ("free", out.values), ("free", out.validity), ("destroy", 0xBEEF)]


def test_releases_everything_in_reverse_order():
    ctx = FakeContext()
    with acu._Scope(ctx) as s:
        made = fill(s)
        assert ctx.released() == []
    assert ctx.released() == made[::-1]
    assert s.keep == []


def test_releases_everything_when_the_body_raises():
    ctx = FakeContext()
    with pytest.raises(ValueError, match="body"):
        with acu._Scope(ctx) as s:
            made = fill(s)
            raise ValueError("body")
    assert ctx.released() == made[::-1]


def test_failing_release_does_not_replace_the_exception_in_flight():
    ctx = FakeContext(bad={0x1000, 0x1100})
    with pytest.raises(ValueError, match="body"):
        with acu._Scope(ctx) as s:
            made = fill(s)
            raise ValueError("body")
    assert ctx.released() == made[::-1]


def test_first_failing_release_is_raised_after_the_others():
    ctx = FakeContext(bad={0x1000, 0x1100})
    with pytest.raises(acu.ArrowError) as e:
        with acu._Scope(ctx) as s:
            made = fill(s)
    assert ctx.released() == made[::-1]
    assert str(e.value) == "free 0x1100 failed"  # released before 0x1000


def test_unset_plan_is_not_destroyed():
    ctx = FakeContext()
    with acu._Scope(ctx) as s:
        plan = s.plan()
        assert isinstance(plan, C.c_void_p) and not plan
    assert ctx.released() == []


def test_nested_scopes_release_independently():
    ctx = FakeContext()
    with acu._Scope(ctx) as outer:
        a = outer.malloc(8)
        with pytest.raises(ValueError):
            with acu._Scope(ctx) as inner:
                b = inner.malloc(8)
                raise ValueError("inner")
        assert ctx.released() == [("free", b)]
        c = outer.malloc(8)
    assert ctx.released() == [("free", b), ("free", c), ("free", a)]


def test_a_scope_stands_where_a_pointer_list_did():
    """The upload helpers append the device pointers they allocate to a list or to a scope alike."""
    ctx = FakeContext()
    arr = np.arange(4, dtype=np.int32)
    owned = []
    p = acu.Context._copy_in(ctx, arr, owned)
    with acu._Scope(ctx) as s:
        q = acu.Context._copy_in(ctx, arr, s)
    assert owned == [p] and ("h2d", p) in ctx.log and ("h2d", q) in ctx.log
    assert ctx.released() == [("free", q)]
