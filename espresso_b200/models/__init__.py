from .transformer import (  # noqa: F401
    SpeechTransformerConfig,
    SpeechTransformerDecoderBase,
    SpeechTransformerEncoderForPrediction,
    SpeechTransformerEncoderModel,
    SpeechTransformerModel,
    SpeechTransformerModelBase,
    SpeechTransformerTransducerModelBase,
)
from .speech_lstm import SpeechLSTMModel, SpeechLSTMModelConfig  # noqa: F401,E402
from .lstm_lm import LSTMLanguageModelEspresso, LSTMLanguageModelEspressoConfig  # noqa: F401,E402
from .tensorized_lookahead_language_model import TensorizedLookaheadLanguageModel  # noqa: F401,E402
from .external_language_model import MultiLevelLanguageModel  # noqa: F401,E402
from .ngram_lm import LexiconTrie, NgramLanguageModel  # noqa: F401,E402
