"""OpenAI-style chat-completions server on the sm_90a hot path (SURVEY §8 f3).

Mirrors the request / response shapes of the reference's `serving/server.py` (`ChatCompletionRequest`
:84-95, content parts :45-62, `/chat/completions` :209-300: `data: {chunk}\n\n` server-sent events when
`stream` is set, one `chat.completion` object otherwise) on top of `generate_content(prompt, stream=...)`.
The reference serialises requests with a global lock; here non-streaming requests that arrive while the
engine is busy are grouped (up to `slots`) and decoded together by `LlavaLlamaModel.generate_batch`
(continuous batching over the shared paged pool, vila_b200/serving.py).  With --sample every request is sampled
on the device with its own temperature, top_p and seed: non-streaming ones through generate_batch, streaming ones
on the single-stream graph decoder (generate_content(stream=True) with a sampling generation config).  Without it
every request is decoded greedily.  With --prefix-cache every non-streaming request goes to the batched engine, which
the model keeps between batches together with the K/V pages of the prompt blocks it has seen: a request that starts
like an earlier one (another question about the same video or image) prefills only what follows the shared blocks.
A non-streaming request with `logprobs` (and optionally `top_logprobs`, 0..20) is always decoded by the batched engine,
which computes each token's log-probability and its top alternatives on the device (vila_b200/logprobs.py); its
choice carries OpenAI's `logprobs.content` list.  A non-streaming request with a non-zero `presence_penalty` or
`frequency_penalty` (each in [-2, 2]) is likewise always decoded by the batched engine, which applies OpenAI's penalties
over the request's generated ids on the device (vila_b200/penalties.py), greedily unless --sample is set.  A streaming
request with logprobs or a non-zero penalty is decoded by the single-stream graph decoder through the model's
`stream_content`, which computes both on the device as well: each SSE chunk carries `choices[0].logprobs.content` for
the ids it was decoded from (every id once, in order, the stop token excluded), even when those ids decode to no text.
With a model that has no `stream_content`, such streaming requests are refused.
A request with a `response_format` of type `json_object` or `json_schema` (structured output), streamed or not, is
decoded alone by the single-stream graph decoder through `stream_content(..., response_format=...)`, which masks every
logits row with the grammar's token bitmask on the device (vila_b200/grammar.py); it never joins a batch, and it
combines with --sample, logprobs and penalties.  A non-streaming one gets the chunks collected into one
`chat.completion`.  `type: "text"` is no constraint, as in OpenAI's API.  A schema that is not JSON, or that the model's
grammar compiler rejects, fails the request before anything is decoded or streamed.

    python -m vila_b200.server --model-path <dir> --port 8000
"""
from __future__ import annotations

import argparse
import asyncio
import base64
import copy
import json
import re
import time
import uuid
from io import BytesIO
from typing import Any, Dict, List, Literal, Optional, Union

from pydantic import BaseModel

from llava.model.configuration_llava import ResponseFormat

IMAGE_B64 = re.compile(r"^data:image/(png|jpe?g);base64,(.*)$")
VIDEO_B64 = re.compile(r"^data:video/(mp4);base64,(.*)$")


class MediaURL(BaseModel):
    url: str


class TextContent(BaseModel):
    type: Literal["text"]
    text: str


class ImageContent(BaseModel):
    type: Literal["image_url"]
    image_url: MediaURL


class VideoContent(BaseModel):
    type: Literal["video_url"]
    video_url: MediaURL
    frames: Optional[int] = 8


class ChatMessage(BaseModel):
    role: Literal["user", "assistant"]
    content: Union[str, List[Union[TextContent, ImageContent, VideoContent]]]


class ChatCompletionRequest(BaseModel):
    model: str
    messages: List[ChatMessage]
    max_tokens: Optional[int] = 512
    top_p: Optional[float] = 0.9
    temperature: Optional[float] = 0.2
    stream: Optional[bool] = False
    use_cache: Optional[bool] = True
    num_beams: Optional[int] = 1
    client: Optional[dict] = None
    seed: Optional[int] = None
    logprobs: Optional[bool] = False
    top_logprobs: Optional[int] = None
    presence_penalty: Optional[float] = 0.0
    frequency_penalty: Optional[float] = 0.0
    response_format: Optional[ResponseFormat] = None


def load_image(url: str):
    from PIL import Image
    m = IMAGE_B64.match(url)
    if m is None:
        if url.startswith("http"):
            raise ValueError("remote image URLs need network access; send base64 data URLs")
        return Image.open(url).convert("RGB")
    return Image.open(BytesIO(base64.b64decode(m.groups()[1]))).convert("RGB")


def load_video(url: str) -> str:
    """A `video_url` -> a file on disk (serving/server.py:124-143: base64 mp4 data URL or http(s)
    download).  A path that exists locally is accepted as it is (no network on a serving box)."""
    import os
    import tempfile
    if url.startswith("http"):
        import requests
        payload = requests.get(url).content
    else:
        m = VIDEO_B64.match(url)
        if m is None:
            if os.path.exists(url):
                return url
            raise ValueError(f"Invalid video url: {url[:64]}")
        payload = base64.b64decode(m.groups()[1])
    path = os.path.join(tempfile.mkdtemp(prefix="vila_serving_"), f"{uuid.uuid5(uuid.NAMESPACE_DNS, url)}.mp4")
    with open(path, "wb") as f:
        f.write(payload)
    return path


def sample_frames_from_video(path: str, num_frames: int = 8) -> list:
    """The server's own sampling rule (serving/server.py:106-122), not `_load_video`'s: frame i of n sits at
    index int(total / n * i); unreadable frames are dropped; a directory of frames is sampled the same way."""
    import os
    from PIL import Image
    if os.path.isdir(path):
        files = sorted(os.path.join(path, f) for f in os.listdir(path))
        return [Image.open(files[int(len(files) / num_frames * i)]).convert("RGB") for i in range(num_frames)]
    import cv2
    cap = cv2.VideoCapture(path)
    total = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
    frames = []
    for i in range(num_frames):
        cap.set(cv2.CAP_PROP_POS_FRAMES, int(total / num_frames * i))
        ok, frame = cap.read()
        if ok:
            frames.append(Image.fromarray(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB)))
    cap.release()
    return frames


def build_prompt(messages: List[ChatMessage], num_video_frames: int = 8) -> list:
    """messages -> the prompt list generate_content takes (serving/server.py:234-256): strings and text
    parts as they come, images decoded to PIL, a video replaced by its sampled frames (as images)."""
    prompt: list = []
    for message in messages:
        if isinstance(message.content, str):
            prompt.append(message.content)
            continue
        for part in message.content:
            if part.type == "text":
                prompt.append(part.text)
            elif part.type == "image_url":
                prompt.append(load_image(part.image_url.url))
            elif part.type == "video_url":
                prompt += sample_frames_from_video(load_video(part.video_url.url), part.frames or num_video_frames)
            else:
                raise NotImplementedError(f"Unsupported content type: {part.type}")
    return prompt


class Engine:
    """One model, one asyncio lock (the GPU is a single queue): streaming requests hold the lock while
    their generator runs; non-streaming requests waiting for it are batched together."""

    def __init__(self, model, model_name: str, slots: int = 8, kv_cache: str = "bf16", sample: bool = False, *,
                 prefix_cache: bool = False, max_tokens_per_slot: int = 20480):
        self.model, self.model_name, self.slots = model, model_name, slots
        self.kv_cache = kv_cache
        if sample and not hasattr(model, "generate_batch"):
            raise ValueError("sample=True needs a model with generate_batch (the batched engine draws the tokens)")
        if prefix_cache and not hasattr(model, "generate_batch"):
            raise ValueError("prefix_cache=True needs a model with generate_batch (the batched engine caches prompts)")
        if prefix_cache and kv_cache == "fp8":
            raise ValueError("prefix caching is not supported with the fp8 KV cache")
        self.sample = sample  # every request sampled with its own parameters (batched engine / graph decoder)
        self.prefix_cache, self.max_tokens_per_slot = prefix_cache, max_tokens_per_slot
        self.lock = asyncio.Lock()
        self.pending: List[Any] = []

    def _gen_config(self, req: ChatCompletionRequest):
        gc = self.model.default_generation_config
        gc.max_new_tokens = req.max_tokens
        return gc

    async def complete(self, req: ChatCompletionRequest) -> Dict[str, Any]:
        if req.model != self.model_name:
            raise ValueError(f"The endpoint is configured to use the model {self.model_name}, "
                             f"but the request model is {req.model}")
        # checked before the request joins a batch: a bad value fails this request only
        rf = self._response_format(req)
        if rf is not None:
            return await self._complete_constrained(req, rf)
        params = self._sampling(req) if self.sample else None
        top = self._top_logprobs(req)
        if top is not None and not hasattr(self.model, "generate_batch"):
            raise ValueError("logprobs need a model with generate_batch (the batched engine computes them)")
        pen = self._penalties(req)
        if pen is not None and not hasattr(self.model, "generate_batch"):
            raise ValueError("presence / frequency penalties need a model with generate_batch (the batched engine "
                             "applies them)")
        loop = asyncio.get_running_loop()
        fut = loop.create_future()
        self.pending.append((req, fut, params, top, pen))
        async with self.lock:
            if not fut.done():  # this task drains the queue for everyone that piled up behind the lock
                batch, self.pending = self.pending[:self.slots], self.pending[self.slots:]
                try:
                    results = await loop.run_in_executor(None, self._run_batch, [b[0] for b in batch],
                                                         [b[2] for b in batch] if self.sample else None,
                                                         [b[3] for b in batch], [b[4] for b in batch])
                except Exception as e:  # every request of the failed batch gets the error, none is left waiting
                    for b in batch:
                        if not b[1].done():
                            b[1].set_exception(e)
                else:
                    for b, res in zip(batch, results):
                        if not b[1].done():
                            b[1].set_result(res)
        text, content = await fut
        return self._completion(req, text, content)

    @staticmethod
    def _completion(req: ChatCompletionRequest, text: str, content) -> Dict[str, Any]:
        choice = {"message": {"role": "assistant", "content": text}}
        if content is not None:
            choice["logprobs"] = {"content": content}
        return {"id": uuid.uuid4().hex, "object": "chat.completion", "created": int(time.time()),
                "model": req.model, "index": 0, "choices": [choice]}

    def _response_format(self, req: ChatCompletionRequest):
        """a request's ResponseFormat, None for none or type "text"; a json_schema without a schema or a schema that
        is not a JSON document raises.  Cheap: the grammar is compiled in a worker thread (check_stream, or the
        decode's own executor call for a non-streaming request)"""
        rf = req.response_format
        if rf is None or rf.type == "text":
            return None
        if not hasattr(self.model, "stream_content"):
            raise ValueError("response_format needs a model with stream_content (the graph decoder applies the "
                             "grammar)")
        if rf.type == "json_schema":
            if rf.json_schema is None:
                raise ValueError("response_format of type json_schema needs json_schema.schema")
            try:
                json.loads(rf.json_schema.schema_)
            except ValueError as e:
                raise ValueError(f"response_format: the schema is not valid JSON: {e}") from None
        return rf

    async def check_stream(self, req: ChatCompletionRequest) -> None:
        """a streaming request's values, checked before its stream starts: sampling, logprobs and penalties
        (_stream_config), and its response_format, whose grammar is compiled here in a worker thread, so a schema the
        model's grammar compiler rejects fails the request first and the event loop is not blocked while it compiles
        (the compiler caches the result for the decode)"""
        self._stream_config(req)
        rf = self._response_format(req)
        if rf is not None and hasattr(self.model, "compile_response_format"):
            await asyncio.get_running_loop().run_in_executor(None, self.model.compile_response_format, rf)

    async def _complete_constrained(self, req: ChatCompletionRequest, rf) -> Dict[str, Any]:
        """a non-streaming request with a response_format: decoded alone under the lock by stream_content in a worker
        thread, its chunks collected into one completion.  The grammar is compiled there too, before anything is
        decoded, so a schema the compiler rejects fails the request without blocking the event loop"""
        gc = self._stream_config(req)
        top, pen = self._top_logprobs(req), self._penalties(req)

        def run():
            ids, entries = [], []
            for chunk, chunk_entries in self.model.stream_content(build_prompt(req.messages), generation_config=gc,
                                                                  logprobs=top, penalties=pen, response_format=rf):
                ids += chunk
                entries += chunk_entries or []
            text = self.model.tokenizer.decode(ids, skip_special_tokens=True).strip()
            return text, None if top is None else self._logprobs_content(ids, entries, top)

        async with self.lock:
            text, content = await asyncio.get_running_loop().run_in_executor(None, run)
        return self._completion(req, text, content)

    @staticmethod
    def _top_logprobs(req: ChatCompletionRequest) -> Optional[int]:
        """a request's number of top alternatives per token (None: no logprobs); a bad combination raises"""
        if req.top_logprobs is not None and not req.logprobs:
            raise ValueError("top_logprobs needs logprobs=true")
        if not req.logprobs:
            return None
        n = 0 if req.top_logprobs is None else req.top_logprobs
        if not isinstance(n, int) or isinstance(n, bool) or not 0 <= n <= 20:
            raise ValueError(f"top_logprobs must be an integer in 0..20, got {n!r}")
        return n

    @staticmethod
    def _penalties(req: ChatCompletionRequest):
        """a request's PenaltyParams, None when both penalties are 0 (None counts as 0); a bad value raises"""
        from .penalties import PenaltyParams
        p = PenaltyParams(presence=0.0 if req.presence_penalty is None else req.presence_penalty,
                          frequency=0.0 if req.frequency_penalty is None else req.frequency_penalty)
        return None if p.off else p

    def _logprobs_content(self, ids: List[int], entries, n: int) -> List[Dict[str, Any]]:
        """OpenAI's logprobs.content: one entry per id the text was decoded from (the stop token excluded)"""
        tok = self.model.tokenizer
        stop = set(getattr(tok, "stop_token_ids", None) or ())
        if ids and ids[-1] in stop:
            ids = ids[:-1]

        def item(i: int, lp: float) -> Dict[str, Any]:
            text = tok.decode([i])
            return {"token": text, "logprob": lp, "bytes": list(text.encode("utf-8"))}

        return [dict(item(e.token, e.logprob), top_logprobs=[item(i, lp) for i, lp in e.top[:n]])
                for e in entries[:len(ids)]]

    def _run_batch(self, reqs: List[ChatCompletionRequest], sampling: Optional[list] = None,
                   top: Optional[list] = None, penalties: Optional[list] = None) -> List[tuple]:
        """sampling: one SamplingParams per request (Engine(sample=True)), or None for greedy decoding; top: each
        request's top_logprobs count, None where it did not ask for logprobs; penalties: each request's PenaltyParams,
        None where it asked for none.  -> (text, logprobs content or None) per request"""
        m = self.model
        top = top if top is not None else [None] * len(reqs)
        want_lp = any(n is not None for n in top)
        want_pen = penalties is not None and any(p is not None for p in penalties)
        if (sampling is None and not self.prefix_cache and not want_lp and not want_pen
                and (len(reqs) == 1 or not hasattr(m, "generate_batch"))):
            return [(m.generate_content(build_prompt(r.messages), generation_config=self._gen_config(r)), None)
                    for r in reqs]
        prepared = [m._prepare_content(build_prompt(r.messages)) for r in reqs]
        # the default is not passed: a model whose generate_batch predates the kv_cache argument keeps working
        kw = {} if self.kv_cache == "bf16" else {"kv_cache": self.kv_cache}
        if sampling is not None:
            kw["sampling"] = sampling
        if self.prefix_cache:
            kw.update(prefix_cache=True, max_tokens_per_slot=self.max_tokens_per_slot)
        if want_lp:  # as kv_cache: only passed when asked for
            kw["logprobs"] = max(n for n in top if n is not None)
        if want_pen:  # likewise
            kw["penalties"] = list(penalties)
        res = m.generate_batch([{"input_ids": i, "media": md, "media_config": mc} for i, md, mc in prepared],
                               max_new_tokens=max(r.max_tokens or 512 for r in reqs), slots=self.slots, **kw)
        ids, lps = res if want_lp else (res, None)
        outs = []
        for k, (r, g) in enumerate(zip(reqs, ids)):
            g = g[:r.max_tokens or 512]
            text = m.tokenizer.decode(g, skip_special_tokens=True).strip()
            outs.append((text, None if top[k] is None else self._logprobs_content(g, lps[k], top[k])))
        return outs

    @staticmethod
    def _sampling(req: ChatCompletionRequest):
        """a request's SamplingParams: temperature None or 0 is greedy, top_p None is off; bad values raise"""
        from .sampling import SamplingParams
        return SamplingParams(temperature=float(req.temperature or 0.0),
                              top_p=float(req.top_p) if req.top_p is not None else 1.0, seed=req.seed)

    def _stream_config(self, req: ChatCompletionRequest):
        """a streamed request's generation config: a copy of the model's default with the request's max_tokens,
        and do_sample set explicitly: with --sample the request's temperature, top_p (top_k 0) and seed, else
        greedy whatever the checkpoint's config says.  Bad values raise."""
        if not hasattr(self.model, "stream_content"):
            if req.logprobs or req.top_logprobs is not None:
                raise ValueError("logprobs are not supported with stream=true: the single-stream decoder that serves "
                                 "streaming requests does not compute them yet; send the request without stream")
            if self._penalties(req) is not None:
                raise ValueError("presence / frequency penalties are not supported with stream=true: the "
                                 "single-stream decoder that serves streaming requests does not apply them yet; send "
                                 "the request without stream")
        else:  # bad values fail the request here, before streaming starts
            self._top_logprobs(req)
            self._penalties(req)
        gc = copy.copy(self.model.default_generation_config)
        gc.max_new_tokens = req.max_tokens
        gc.do_sample = False
        if self.sample:
            p = self._sampling(req)
            gc.do_sample = not p.greedy
            gc.temperature, gc.top_k, gc.top_p, gc.seed = p.temperature, 0, p.top_p, p.seed
        return gc

    @staticmethod
    def _sse_chunk(req: ChatCompletionRequest, chunk_id: int, text: str, content=None) -> str:
        """one streamed chat.completion.chunk event: the text delta, and OpenAI's logprobs.content when given"""
        choice: Dict[str, Any] = {"delta": {"content": text}}
        if content is not None:
            choice["logprobs"] = {"content": content}
        chunk = {"id": str(chunk_id), "object": "chat.completion.chunk", "created": int(time.time()),
                 "model": req.model, "choices": [choice]}
        return f"data: {json.dumps(chunk)}\n\n"

    async def stream(self, req: ChatCompletionRequest):
        if req.model != self.model_name:
            raise ValueError(f"The endpoint is configured to use the model {self.model_name}, "
                             f"but the request model is {req.model}")
        gc = self._stream_config(req)  # a bad value fails this request before it takes the lock
        top, pen, rf = self._top_logprobs(req), self._penalties(req), self._response_format(req)
        if top is not None or pen is not None or rf is not None:
            kw = {} if rf is None else {"response_format": rf}  # as in _run_batch: only passed when asked for
            async with self.lock:
                gen = self.model.stream_content(build_prompt(req.messages), generation_config=gc, logprobs=top,
                                                penalties=pen, **kw)
                for chunk_id, (ids, entries) in enumerate(gen):
                    text = self.model.tokenizer.decode(ids, skip_special_tokens=True)
                    content = None if top is None else self._logprobs_content(ids, entries, top)
                    if text or content:  # a chunk with entries is sent even when its ids decode to no text
                        yield self._sse_chunk(req, chunk_id, text, content)
                    await asyncio.sleep(0)
                yield "data: [DONE]\n\n"
            return
        async with self.lock:
            gen = self.model.generate_content(build_prompt(req.messages), generation_config=gc, stream=True)
            for chunk_id, new_text in enumerate(gen):
                if len(new_text):
                    yield self._sse_chunk(req, chunk_id, new_text)
                await asyncio.sleep(0)
            yield "data: [DONE]\n\n"


def create_app(model, model_name: str, slots: int = 8, kv_cache: str = "bf16", sample: bool = False, *,
               prefix_cache: bool = False, max_tokens_per_slot: int = 20480):
    from fastapi import FastAPI
    from fastapi.responses import JSONResponse, StreamingResponse
    app = FastAPI()
    engine = Engine(model, model_name, slots, kv_cache, sample, prefix_cache=prefix_cache,
                    max_tokens_per_slot=max_tokens_per_slot)
    app.state.engine = engine

    @app.get("/")
    async def read_root():
        return {"message": "vila_b200 chat-completions endpoint: POST /chat/completions"}

    @app.post("/chat/completions")
    async def chat_completions(request: ChatCompletionRequest):
        try:
            if request.stream:
                await engine.check_stream(request)  # bad values or schemas fail this request before it streams
                return StreamingResponse(engine.stream(request), media_type="text/event-stream")
            return await engine.complete(request)
        except Exception as e:  # the reference answers 500 with the message (server.py:302-306)
            return JSONResponse(status_code=500, content={"error": str(e)})

    return app


def main() -> None:
    import uvicorn

    import llava
    from llava.mm_utils import get_model_name_from_path
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", type=str, default="0.0.0.0")
    ap.add_argument("--port", type=int, default=8000)
    ap.add_argument("--model-path", type=str, required=True)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--decode-weights", choices=("bf16", "fp8", "w4a16"), default="bf16",
                    help="weights of the single-stream greedy decoder (fp8: e4m3 with per-row scales; w4a16: "
                         "4-bit with group-128 scales and zero points, lm_head e4m3), and of the engine that "
                         "batches queued requests; the prefill stays bf16)")
    ap.add_argument("--kv-cache", choices=("bf16", "fp8"), default="bf16",
                    help="K/V format of the engine that batches queued requests (fp8: e4m3 with one fp32 scale "
                         "per token and KV head, about half the bytes; the single-stream decoder stays bf16)")
    ap.add_argument("--sample", action="store_true",
                    help="sample every request with its own temperature, top_p and seed on the device: "
                         "non-streaming requests on the batched engine (vila_sample_batch), even one that arrives "
                         "alone, streaming requests on the single-stream graph decoder (vila_sample_finalize); "
                         "without it every request is decoded greedily")
    ap.add_argument("--prefix-cache", action="store_true",
                    help="send every non-streaming request, even one that arrives alone, to the batched engine and "
                         "keep that engine between batches with the K/V pages of the full 128-token prompt blocks it "
                         "has seen, so that a request starting like an earlier one (another question about the same "
                         "video or image) prefills only what follows.  The kept pool is slots x "
                         "--max-tokens-per-slot x the K/V bytes per token (57,344 B for NVILA-8B: 9.4 GB at 8 x "
                         "20,480).  Not with --kv-cache fp8; streaming requests are unchanged")
    ap.add_argument("--max-tokens-per-slot", type=int, default=20480,
                    help="tokens per slot of the kept engine of --prefix-cache (prompt + new tokens + 8)")
    args = ap.parse_args()
    if args.prefix_cache and args.kv_cache == "fp8":
        ap.error("--prefix-cache is not supported with --kv-cache fp8")
    model = llava.load(args.model_path, decode_weights=args.decode_weights)
    uvicorn.run(create_app(model, get_model_name_from_path(args.model_path), args.slots, args.kv_cache, args.sample,
                           prefix_cache=args.prefix_cache, max_tokens_per_slot=args.max_tokens_per_slot),
                host=args.host, port=args.port)


if __name__ == "__main__":
    main()
