"""megatts2_b200: H100-native (sm_90a) implementation of the Mega-TTS 2 synthesis hot path.

Drop-in surface = the reference's nn.Module API (LSimon95/megatts2, SURVEY.md §8b):
``megatts2_b200.modules.{transformer,convnet,mrte,vqpe,embedding,tokenizer,quantization}``
and ``megatts2_b200.models.megatts2.{MegaG,MegaPLM,MegaADM,Megatts}`` keep the reference's
class names, constructor kwargs, state_dict keys and forward/infer signatures; all device
work goes through ``lib/libmegatts2_b200.so`` (C ABI in ``include/megatts2_b200.h``).
"""
__version__ = "0.1.0"
