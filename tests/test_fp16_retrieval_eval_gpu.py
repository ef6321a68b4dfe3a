"""evaluate_retrieval on an fp16 model (its search in fp16 operands) against recall_at_k over the same index:
the checks of tests/test_retrieval_eval_gpu.py, run on dtype='fp16' models, on the same validation shards
(a distractor first, distractors at the tail)."""
import pytest

import test_retrieval_eval_gpu as RE
from test_retrieval_eval_gpu import shards  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("embedding_size,return_embedding", [(32, True), (0, False)])
def test_fp16_evaluate_retrieval_equals_recall_at_k(shards, embedding_size, return_embedding):  # noqa: F811
    RE.test_evaluate_retrieval_equals_recall_at_k_on_pil_batches(shards, "fp16", embedding_size, return_embedding)
