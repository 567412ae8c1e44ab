"""QueryBatch marshalling of per-query doc filters (TQ_QUERY_FILTER): the flag and filter_id land in the tq_query row, queries
without a filter keep both zero, and a filter that is not a u32 id is refused before anything reaches the library."""
import numpy as np
import pytest

from tantivy_b200._abi import (TQ_OP_OR, TQ_QUERY_COUNT_HITS, TQ_QUERY_FILTER, TQ_QUERY_HAS_THRESHOLD, Query, QUERY_DTYPE,
                               QueryBatch)


def _q(**extra):
    q = dict(op=TQ_OP_OR, k=10, weights=[1.0, 2.0], avg_fieldnorm=[3.0, 3.0], term_segs=[(0, 5, 0, 10, 0, 40), (1, 5, 0, 7, 40, 70)])
    q.update(extra)
    return q


def test_filter_sets_flag_and_id():
    qb = QueryBatch([_q(), _q(filter=7), _q(filter=0, threshold=1.5, count_hits=True), _q(filter=np.uint32(2**32 - 1))])
    rows = qb.q[:qb.nq]
    assert list(rows["flags"]) == [0, TQ_QUERY_FILTER, TQ_QUERY_HAS_THRESHOLD | TQ_QUERY_COUNT_HITS | TQ_QUERY_FILTER, TQ_QUERY_FILTER]
    assert list(rows["filter_id"]) == [0, 7, 0, 2**32 - 1]
    assert QUERY_DTYPE.fields["filter_id"][1] == Query.filter_id.offset == 104


@pytest.mark.parametrize("bad", [-1, 2**32, 1.5, True, "3"])
def test_filter_must_be_a_u32_id(bad):
    with pytest.raises(ValueError, match="filter"):
        QueryBatch([_q(), _q(filter=bad)])
