# mirrors decoders/__init__.py for the recognition heads, the EAST head and the DB detector head (SegDetector + its losses)
from .attention_decoder import AttentionDecoder  # noqa: F401
from .ctc_decoder import CTCDecoder  # noqa: F401
from .crnn import CRNNDecoder  # noqa: F401
from .ctc_decoder2d import CTCDecoder2D  # noqa: F401
from .ctc_loss2d import CTCLoss2D, CTC2DLoss  # noqa: F401
from .east import EASTDecoder  # noqa: F401
from .dice_loss import DiceLoss  # noqa: F401
from .l1_loss import MaskL1Loss  # noqa: F401
from .balance_cross_entropy_loss import BalanceCrossEntropyLoss  # noqa: F401
from .seg_detector import SegDetector  # noqa: F401
