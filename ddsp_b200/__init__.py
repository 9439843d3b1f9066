"""ddsp_b200 - H100-native (sm_90a) Harmonic + FilteredNoise DDSP decoder.

Drop-in for the signal-generation layer of magenta/ddsp: `Processor`,
`ProcessorGroup`, `Harmonic`, `FilteredNoise`, `Add` with the reference's API,
backed by hand-written CUDA kernels behind a ctypes C ABI (include/ddsp_b200.h).
"""
from ddsp_b200 import _lib
from ddsp_b200 import colab_utils
from ddsp_b200 import core
from ddsp_b200 import dags
from ddsp_b200 import decoders
from ddsp_b200 import effects
from ddsp_b200 import encoders
from ddsp_b200 import heuristics
from ddsp_b200 import host
from ddsp_b200 import models
from ddsp_b200 import nn
from ddsp_b200 import postprocessing
from ddsp_b200 import preprocessing
from ddsp_b200 import processors
from ddsp_b200 import synthetic_data
from ddsp_b200 import synths
from ddsp_b200.decoders import DilatedConvDecoder, MidiToHarmonicDecoder, RnnFcDecoder
from ddsp_b200.effects import (ExpDecayReverb, FIRFilter, FilteredNoiseReverb,
                               ModDelay, Reverb)
from ddsp_b200.encoders import (ExpressionEncoder, HarmonicToMidiEncoder, OneHotEncoder,
                                ResnetSinusoidalEncoder, SinusoidalToHarmonicEncoder)
from ddsp_b200.host import HostDecoder
from ddsp_b200.models import InverseSynthesis, MidiAutoencoder, ZMidiAutoencoder
from ddsp_b200.processors import Add, Crop, Mix, Processor, ProcessorGroup
from ddsp_b200.synths import (FilteredNoise, Harmonic, Sinusoidal, TensorToAudio,
                              Wavetable)

__version__ = '0.1.0'
