"""tantivy_b200 — H100-native execution of tantivy's posting decode -> AND/OR -> BM25 -> top-k path.

Importing this package loads the CUDA library (tantivy_b200/_lib/libtantivy_b200.so) and fails
loudly if it has not been built; there is no CPU fallback."""
from ._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_BOOL, TERMINATED, TQ_MAX_K, TQ_MAX_TERMS, TQ_OP_AND, TQ_OP_OR, TQ_OP_PHRASE, TQ_OP_TERM, TQ_ORDER_ASC, TQ_ORDER_DESC,
                   TQ_FAST_BOOL, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64,
                   TQ_METRIC_COUNT_ONLY, TQ_METRIC_EMPTY, TQ_METRIC_MISSING, TQ_METRICS_MAX_COLUMNS,
                   TQ_TERMS_BY_COUNT, TQ_TERMS_BY_KEY, TQ_TERMS_BY_METRIC, TQ_TERMS_MISSING_AFTER_MAX, TQ_TERMS_MISSING_IMAGE, TQ_TERMS_MISSING_NONE,
                   TQ_RECORD_BASIC, TQ_RECORD_FREQS, TQ_RECORD_FREQS_POSITIONS, QueryBatch)
from .lib import (Batch, Context, FieldWriter, MultiContext, SynthIndex, TqError, bm25_idf, bm25_tf_cache, bm25_weight, fast_value_to_u64, fieldnorm_to_id,
                  id_to_fieldnorm, u64_to_fast_value)
from . import terms  # noqa: E402  (the terms aggregation's request and result side)
from .terms import TermsRefused  # noqa: E402
from . import metrics  # noqa: E402  (the metric aggregations' request and result side)
from .metrics import MetricsRefused  # noqa: E402
from . import hist_metrics  # noqa: E402  (histograms with metric sub-aggregations: request and result side)
from .hist_metrics import HistMetricsRefused  # noqa: E402
from . import terms_metrics  # noqa: E402  (terms with metric sub-aggregations: request and result side)
from .terms_metrics import TermsMetricsRefused  # noqa: E402
from . import ranges  # noqa: E402  (range aggregations, with or without metric sub-aggregations: request and result side)
from .ranges import RangeRefused  # noqa: E402
from . import terms_hist  # noqa: E402  (terms with one histogram sub-aggregation: request and result side)
from .terms_hist import TermsHistRefused  # noqa: E402
from . import hist_terms  # noqa: E402  (a histogram with one terms sub-aggregation: request and result side)
from .hist_terms import HistTermsRefused  # noqa: E402
