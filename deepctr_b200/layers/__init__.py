"""deepctr.layers surface for the hot path (deepctr/layers/__init__.py:3-54 lists the reference's)."""
from ..engine import Layer, Dense, Flatten, Reshape, Concatenate, Add, Lambda, Input, Conv2D
from .activation import Dice, Activation, activation_layer
from .core import DNN, LocalActivationUnit, PredictionLayer, RegulationModule
from .interaction import (AFMLayer, BiInteractionPooling, BilinearInteraction, FM, CrossNet, CIN, InteractingLayer,
                          SENETLayer, FwFMLayer, FEFMLayer, InnerProductLayer, OutterProductLayer, BridgeModule,
                          FieldWiseBiInteraction)
from .normalization import BatchNormalization, Dropout, LayerNormalization
from .sequence import (SequencePoolingLayer, WeightedSequenceLayer, AttentionSequencePoolingLayer, Transformer,
                       PositionEncoding, KMaxPooling)
from .utils import (NoMask, Hash, Linear, Concat, _Add, concat_func, add_func, combined_dnn_input,
                    reduce_sum, reduce_mean, reduce_max, div, softmax)

custom_objects = {
    'DNN': DNN, 'PredictionLayer': PredictionLayer, 'LocalActivationUnit': LocalActivationUnit,
    'AFMLayer': AFMLayer, 'BiInteractionPooling': BiInteractionPooling,
    'SENETLayer': SENETLayer, 'BilinearInteraction': BilinearInteraction,
    'FwFMLayer': FwFMLayer, 'FEFMLayer': FEFMLayer,
    'InnerProductLayer': InnerProductLayer, 'OutterProductLayer': OutterProductLayer,
    'FM': FM, 'CrossNet': CrossNet, 'CIN': CIN, 'InteractingLayer': InteractingLayer,
    'SequencePoolingLayer': SequencePoolingLayer, 'WeightedSequenceLayer': WeightedSequenceLayer,
    'AttentionSequencePoolingLayer': AttentionSequencePoolingLayer, 'Dice': Dice, 'Hash': Hash,
    'Linear': Linear, 'Concat': Concat, 'NoMask': NoMask, '_Add': _Add,
    'Transformer': Transformer, 'PositionEncoding': PositionEncoding, 'LayerNormalization': LayerNormalization,
    'RegulationModule': RegulationModule, 'BridgeModule': BridgeModule, 'KMaxPooling': KMaxPooling,
    'FieldWiseBiInteraction': FieldWiseBiInteraction,
}
