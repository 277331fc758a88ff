"""llava/conversation.py — only what `llava.cli.infer` touches: the conversation-mode registry.  The
sm_90a path tokenises through the tokenizer's chat template (SeparatorStyle.AUTO in the reference,
llava/utils/tokenizer.py:83-115), so a mode is just a name here."""
from types import SimpleNamespace


class _Conv(SimpleNamespace):
    def copy(self):
        return _Conv(**self.__dict__)


conv_templates = {name: _Conv(name=name, sep_style="AUTO") for name in ("auto", "vicuna_v1", "llama_3", "hermes-2")}
default_conversation = conv_templates["auto"].copy()


def auto_set_conversation_mode(model_name_or_path: str) -> None:
    global default_conversation
    default_conversation = conv_templates["auto"].copy()
