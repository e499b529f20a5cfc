"""tests/oracle_filter_take.py against the reference's literal struct and union cases (tests/golden/union_vectors.json), and its
error order, on the CPU."""
import numpy as np
import pytest

from acu import HostArray, ListColumn, StructColumn, UnionColumn
from acu import _abi as abi

import oracle_filter_take as oft
import union_util as uu

CASES = uu.golden_cases()


def _filter(col, pred):
    return oft.filter(col, oft.filter_mask(pred))


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{k}" for k, c in enumerate(CASES)])
def test_oracle_matches_golden(i):
    case = CASES[i]
    uu.check(case, uu.run_case(case, _filter, oft.take_host))


def test_golden_covers_every_reference_test():
    names = {c["name"] for c in CASES}
    assert names == {
        "test_filter_union_array_dense", "test_filter_union_array_sparse", "test_filter_run_union_array_dense",
        "test_filter_union_array_dense_with_nulls", "test_filter_union_array_sparse_with_nulls", "test_filter_struct",
        "test_filter_empty_struct", "test_take_struct", "test_take_struct_with_null_indices", "test_take_union_sparse",
        "test_take_union_dense", "test_take_union_dense_using_builder", "test_take_union_dense_all_match_issue_6206"}


def _dense():
    return UnionColumn(abi.UNION_DENSE, [3, 7], [HostArray.from_list(abi.I32, [1, 2]), HostArray.from_list(abi.I64, [5])],
                       [3, 7, 3], [0, 0, 1])


def test_null_out_of_bounds_index_gives_type_id_zero_and_fails_validation():
    idx = HostArray.from_list(abi.U32, [0, None])
    idx.values[1] = 99
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(_dense(), idx)
    assert e.value.status == abi.ERR_INVALID_ARGUMENT and e.value.message.endswith(oft.UNION_TYPE_IDS)


def test_child_error_comes_before_the_validation():
    # type id 0 names a field whose child is empty: the child's take panics first
    u = UnionColumn(abi.UNION_DENSE, [0], [HostArray.from_list(abi.I32, [])], [0], [0])
    idx = HostArray.from_list(abi.U32, [None])
    idx.values[0] = 5
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(u, idx)
    assert e.value.status == abi.ERR_PANIC_OUT_OF_BOUNDS


def test_struct_take_reads_a_validity_buffer_without_nulls():
    s = StructColumn([HostArray.from_list(abi.I32, [1, 2])], oft.nulls_of([True, True], force=True))
    idx = HostArray.from_list(abi.U32, [None, 0])
    idx.values[0] = 9
    assert oft.take_host(s, idx).nulls.valid_mask().tolist() == [False, True]
    with pytest.raises(oft.OracleError) as e:  # the field's own panic comes first
        oft.take_host(s, HostArray.from_list(abi.U32, [0, 9]))
    assert e.value.message.startswith("Out-of-bounds index")
    s0 = StructColumn([], oft.nulls_of([True, True], force=True))
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(s0, HostArray.from_list(abi.U32, [0, 9]))
    assert e.value.message == oft.BIT_LEN and e.value.index == 1
    # without a validity buffer no row is read
    s1 = StructColumn([], oft.nulls_of([True, True]))
    assert oft.take_host(s1, HostArray.from_list(abi.U32, [0, 9])).length == 2


def test_dense_filter_under_a_list_extends_every_row():
    u = _dense()
    lst = ListColumn(np.array([0, 2, 3], np.int32), u, oft.nulls_of([True, True]))
    got = oft.filter(lst, np.array([False, True]))
    # the list's child step extends row 2 of the union: child 3's row 1 becomes its only row
    assert oft.to_pylist(got) == [[[3, 2]]]
    assert [int(x) for x in got.child.offsets] == [0]
