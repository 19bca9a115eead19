"""The synthetic Llama models of the eval-step tests, and the bar their logits are held to.

* `toy`: vocab 320, n_embd 256, n_ff 512, Q4_0 layers, a Q4_0 or Q6_K lm_head, its CPU graph (oracle/llama_model.py) and the jig
  graph: the same graph with every embedding value moved by +-64 ulp.
* `llama2_7b_shaped`: n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000, two Q4_0 layers and the full Q4_0 output head,
  drawn from the caller's generator, and the reference engine: oracle.RefNeLlama where oracle/_ref is built, else the CPU graph.
* `smooth`: the toy's shapes with BesTLA int4 weights evaluated in fp32, whose logits are a smooth function of the attention
  output, so that two attention kernels can be compared tightly through the whole engine.

Every engine is loaded by neural_speed_b200.gguf_loader.load_into_engine, as a model read from a file is.

The bar (DESIGN.md section 2).  Each Q8_0 activation quantisation is a rounding discontinuity, so the CPU graph differs from its
own jig by a measurable amount: the conditioning floor of the graph.  A device step has to stay within the north star 1e-2, or
1.5 x that floor where it is larger, and within 2.5e-2 outright, all relative to max(1, max|want|).  The floor is either the
largest distance seen so far in the test (`RunningBar`: the floor is a property of the model, not of one step) or that of one
evaluation (`bar(distance(jig_want, want))`)."""
import numpy as np

import neural_speed_b200 as ns
import oracle
from neural_speed_b200 import gguf_loader
from oracle.llama_model import OracleLlama, greedy


def _hparams(n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx):
    return dict(n_vocab=n_vocab, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_layer=n_layer, n_ff=n_ff, n_ctx=n_ctx,
                norm_eps=1e-5, rope_theta=10000.0, rope_scale=1.0)


def _shapes(hp):
    E, FF = hp["n_embd"], hp["n_ff"]
    kvd = E // hp["n_head"] * hp["n_head_kv"]
    return dict(wq=(E, E), wk=(kvd, E), wv=(kvd, E), wo=(E, E), w1=(FF, E), w2=(E, FF), w3=(FF, E))


def _norm(rng, n):
    return rng.uniform(0.5, 1.5, n).astype(np.float32)


def _moved(tok, signs):
    """the embedding table with every value moved by sign x 64 ulp"""
    return (tok.view(np.int32) + signs * 64).view(np.float32)


class Llama:
    """fp32 embeddings and norms; per layer the seven matmul payloads of type `fmt`, and the lm_head's of type `out_fmt`
    (gguf_loader's "q4_0", "q6_K" or "btla")"""

    tok_jig = None

    def __init__(self, hp, tok, out_norm, out_rows, layers, out_fmt="q4_0", fmt="q4_0"):
        self.hp, self.tok, self.out_norm, self.out_rows, self.layers = hp, tok, out_norm, out_rows, layers
        self.out_fmt, self.fmt = out_fmt, fmt

    def draw_jig(self, rng):
        """the 7B-shaped model's jig table, signs drawn from the caller's generator wherever the test draws them"""
        self.tok_jig = _moved(self.tok, rng.integers(0, 2, self.tok.shape, dtype=np.int8).astype(np.int32) * 2 - 1)

    def graph(self, jig=False):
        """a fresh CPU graph (its own KV cache: one per sequence), on the jig table with jig=True"""
        return OracleLlama(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers, fmt=self.out_fmt)

    def reference(self, jig=False):
        """the reference's own graph engine where oracle/_ref is built, else the CPU graph (bit-identical to it)"""
        if oracle.ref_ne() is None:
            return self.graph(jig)
        return oracle.RefNeLlama(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def engine(self, n_seq=1):
        """a device engine with every tensor set, and n_seq KV blocks"""
        layers = [{k: v if k.endswith("norm") else (self.fmt, v) for k, v in L.items()} for L in self.layers]
        model = gguf_loader.GGUFLlama(self.hp, self.tok, self.out_norm, (self.out_fmt, self.out_rows), layers)
        eng = gguf_loader.load_into_engine(model)
        if n_seq != 1:
            eng.set_sequences(n_seq)
        return eng


def toy(n_head=4, n_head_kv=4, out_fmt="q4_0", seed=0, n_layer=2, n_ctx=48):
    rng = np.random.default_rng(seed)
    hp = _hparams(320, 256, n_head, n_head_kv, n_layer, 512, n_ctx)
    E, V = 256, 320

    def w(n, k):
        return rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32)

    tok = rng.normal(0, 1, (V, E)).astype(np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = oracle.quantize_q4_0(w(n, k))
        layers.append(L)
    wout = w(V, E)
    out_rows = oracle.quantize_q6_K(wout) if out_fmt == "q6_K" else oracle.quantize_q4_0(wout)
    m = Llama(hp, tok, out_norm, out_rows, layers, out_fmt)
    m.tok_jig = _moved(tok, (np.random.default_rng(99).integers(0, 2, tok.shape) * 2 - 1).astype(np.int32))
    return m


def llama2_7b_shaped(rng, n_ctx):
    """Q4_0 weights drawn from rng; the jig (Llama.draw_jig) is a separate draw"""
    hp = _hparams(32000, 4096, 32, 32, 2, 11008, n_ctx)
    E, V = 4096, 32000

    def qw(n, k):
        return oracle.quantize_q4_0(rng.standard_normal((n, k), dtype=np.float32) * np.float32(1.0 / np.sqrt(k)))

    tok = rng.standard_normal((V, E), dtype=np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(hp["n_layer"]):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = qw(n, k)
        layers.append(L)
    return Llama(hp, tok, out_norm, qw(V, E), layers)


def smooth(n_head, n_head_kv, n_ctx, seed=0, n_layer=2):
    """BesTLA int4 (group 32, symmetric, fp32 scales) weights with fp32 compute: no activation quantiser.  The lm_head is drawn
    before the layers."""
    rng = np.random.default_rng(seed)
    hp = _hparams(320, 256, n_head, n_head_kv, n_layer, 512, n_ctx)
    E, V = 256, 320

    def blob(n, k):
        return ns.np_bestla_quantize(rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32), "int4", 32, "sym", "fp32", "fp32")

    tok = rng.normal(0, 1, (V, E)).astype(np.float32)
    out_norm = _norm(rng, E)
    out = blob(V, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = blob(n, k)
        layers.append(L)
    return Llama(hp, tok, out_norm, out, layers, out_fmt="btla", fmt="btla")


def close(*graphs):
    """free the reference engines among graphs (a CPU graph holds nothing to free)"""
    for g in graphs:
        if hasattr(g, "close"):
            g.close()


def rows(graph, tokens, n_past):
    """the reference's logits_all rows of one segment, [len(tokens)][n_vocab]: row r is the last-token logits of the same sequence
    evaluated one token at a time up to token r -- model_eval's graph is row-wise apart from the causal attention, which reads
    the K/V rows the earlier tokens appended"""
    return np.stack([graph.eval([t], n_past + j) for j, t in enumerate(tokens)])


# ------------------------------------------------------------------------------------------------------------- the bar
def scale(want):
    return max(1.0, float(np.abs(want).max()))


def distance(got, want):
    """max |got - want| relative to max(1, max|want|)"""
    return float(np.abs(got - want).max()) / scale(want)


def bar(floor):
    """the north star 1e-2, or 1.5 x the conditioning floor where that is larger, never more than 2.5e-2"""
    return min(max(1e-2, 1.5 * floor), 2.5e-2)


class RunningBar:
    """the bar on the largest distance of the CPU graph to its jig seen so far in the test"""

    def __init__(self):
        self.floor = 0.0

    def __call__(self, want, jig_want):
        self.floor = max(self.floor, distance(jig_want, want))
        return bar(self.floor)


class SeqOracle:
    """one sequence on the CPU graph and on its jig: eval() returns the logits and the running bar after that step"""

    def __init__(self, model, running):
        self.orc, self.jig, self.running = model.graph(), model.graph(jig=True), running

    def eval(self, tokens, n_past):
        want = self.orc.eval(tokens, n_past)
        return want, self.running(want, self.jig.eval(tokens, n_past))


def unambiguous(want, tol=2e-2):
    """want's top-2 margin exceeds tol x max(1, max|want|)"""
    top = np.sort(want)[-2:]
    return top[1] - top[0] > tol * scale(want)


def check_logits(got, want, tol=1e-2):
    """got within tol of want, and its argmax the greedy pick wherever want's top-2 margin exceeds twice that"""
    s = scale(want)
    err = float(np.abs(got - want).max())
    assert err <= tol * s, (err / s, tol)
    if unambiguous(want, 2 * tol):
        assert int(np.argmax(got)) == greedy(want)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)
