"""visualbert_b200 — the VisualBERT encoder hot path as hand-written sm_90a (H100) CUDA kernels behind the
reference's `TrainVisualBERTObjective` / `BertVisualModel` interface. See DESIGN.md."""
from .modeling import (BertConfig, BertLayerNorm, BertVisualModel, BertEmbeddingsWithVisualEmbedding,  # noqa: F401
                       BertEncoder, BertLayer, BertPooler, BertPreTrainingHeads, PreTrainedBertModel,
                       TrainVisualBERTObjective)

__version__ = "0.1.0"
from .optimization import BertAdam, WarmupLinearSchedule  # noqa: F401,E402
