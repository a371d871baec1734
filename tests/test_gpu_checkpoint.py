"""Checkpoints on the GPU: sampler.checkpoint() / sampler.restore() (amwg_checkpoint_save / amwg_checkpoint_load).

A run that is checkpointed, closed and restored into a new sampler must be the run that never stopped: draws, state, log_post and
info bit for bit, on every kernel path, at any point of the adaptation schedule, on any sharding of the chains, from either host.
A refused restore must leave the handle exactly as it was."""
import numpy as np
import pytest

import ckpt_ref
import models
from conftest import config2_data, config3_data
from test_gpu_inits import PATHS, _bits_equal, _case, env

pytestmark = pytest.mark.gpu


def _out(s):
    return {"state": s.state, "log_post": s.log_post(), "info": s.info()}


# the calls of a run, split at the checkpoint: (calls before, calls after)
POINTS = {
    "mid_batch": ([("burn", 75)], [("sample", 40), ("burn", 60), ("sample", 30)]),
    "batch_boundary": ([("burn", 100)], [("sample", 30), ("burn", 50), ("sample", 20)]),
    "adaptation_stopped": ([("burn", 60), ("stop", 0), ("burn", 15)], [("sample", 20), ("start", 0), ("burn", 70), ("sample", 20)]),
}


def _do(s, calls):
    got = []
    for op, n in calls:
        if op == "burn":
            s.burn(n)
        elif op == "sample":
            got.append(s.sample(n))
        elif op == "stop":
            s.stop_adaptation()
        elif op == "start":
            s.start_adaptation()
    return {"draws": got, **_out(s)}


@pytest.mark.parametrize("point", list(POINTS))
@pytest.mark.parametrize("name", PATHS)
def test_resume_equals_never_stopping_on_every_kernel_path(gpu_pkg, name, point):
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, check = _case(gpu_pkg, name)
    before, after = POINTS[point]
    with env(**envs):
        a = mcmc.AmwgSampler(params, lp, data, dict(opts))
        b = mcmc.AmwgSampler(params, lp, data, dict(opts))
        _do(a, before)
        _do(b, before)
        at_a = _out(a)
        img = b.checkpoint()
        b.close()
        c = mcmc.AmwgSampler(params, lp, data, dict(opts, seed=opts["seed"] + 1000))
        c.restore(img)
    assert check(a) and check(c) and a.jit_status()[0] == c.jit_status()[0], (name, c.jit_status())
    assert c.seed == opts["seed"]
    _bits_equal(_out(c), at_a, name + " at the checkpoint")
    _bits_equal(_do(c, after), _do(a, after), name + " " + point)


@pytest.mark.parametrize("name", PATHS)
def test_set_state_and_restore_to_the_current_run_mid_batch_change_nothing(gpu_pkg, name):
    """burn(75) ends in the middle of an adaptation batch. Putting the chains back where they are (set_state), or restoring the image
    just taken into the same handle, re-evaluates log_post and the term cache from the state: both must be exactly what the sweep
    kernels carried."""
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, check = _case(gpu_pkg, name)
    with env(**envs):
        hs = [mcmc.AmwgSampler(params, lp, data, dict(opts)) for _ in range(3)]
    out = []
    for k, s in enumerate(hs):
        s.burn(75)
        if k == 1:
            s.set_state({n: v for n, v in s.state.items() if n in params})
        if k == 2:
            s.restore(s.checkpoint())
        out.append({"lp0": s.log_post(), **_do(s, [("sample", 50), ("burn", 30)])})
    _bits_equal(out[0], out[1], name + " set_state")
    _bits_equal(out[0], out[2], name + " restore")


def _wide(ld):
    P = 18
    params = {"t%d" % k: ({"type": "real"} if k % 3 else {"type": "int", "lower": -50, "upper": 50}) for k in range(P)}
    params["x"] = {"type": "real", "dim": [300]}
    params["m"] = {"type": "binary"}

    def lp(state, d=None):
        l = 0
        for k in range(P):
            l += ld.norm(state["t%d" % k], 0.5 * k, 1 + 0.1 * k)
        for j in range(300):
            l += ld.norm(state.x[j], 0.01 * j, 2)
        l += ld.bern(state.m, 0.3)
        state.tsum = state.t1 + state.t2
        return l
    return params, lp


def test_wide_models_resume_and_reshard(gpu_pkg):
    """20 named parameters (the substepper order is one byte per parameter), a dim-300 parameter (its visiting order lives in global
    memory), int and binary components and a derived quantity. Every handle holds whole CTAs of the phase-synchronised term-cache
    sweep (128 chains): in a ragged last CTA the threads past the last chain shadow it, and on this model that chain does not repeat
    bit for bit from one run to the next, with or without a checkpoint."""
    mcmc = gpu_pkg.mcmc
    params, lp = _wide(gpu_pkg.ld)
    opts = {"chains": 256, "seed": 12}
    a = mcmc.AmwgSampler(params, lp, None, dict(opts))
    parts = [mcmc.AmwgSampler(params, lp, None, dict(opts, chains=128, first_chain=f)) for f in (0, 128)]
    for s in [a] + parts:
        s.burn(75)
    imgs = [p.checkpoint() for p in parts]
    assert len(imgs[0]) == 56 + 24 * 319 + 128 * (20 * 319 + 8 + 20) + 8          # D = 18 + 300 + 1, P = 20
    for p in parts:
        p.close()
    b = mcmc.AmwgSampler(params, lp, None, dict(opts, seed=1))
    b.restore(imgs[::-1])
    after = [("sample", 30), ("burn", 30), ("sample", 10)]
    ra, rb = _do(a, after), _do(b, after)
    _bits_equal(rb, ra, "wide")
    assert set(np.unique(np.asarray(ra["draws"][0]["m"]))) <= {0.0, 1.0} and "tsum" in ra["state"]


def test_rewind_continues_like_a_fresh_handle_restored_from_the_image(gpu_pkg):
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, _check = _case(gpu_pkg, "term_cache")
    s = mcmc.AmwgSampler(params, lp, data, dict(opts))
    s.burn(75)
    img = s.checkpoint()
    s.sample(40)
    s.stop_adaptation()
    s.burn(33)
    s.restore(img)
    f = mcmc.AmwgSampler(params, lp, data, dict(opts, seed=77))
    f.restore(img)
    after = [("sample", 40), ("burn", 60), ("sample", 10)]
    _bits_equal(_do(s, after), _do(f, after), "rewind")


def _norm(pkg, x, **opts):
    return pkg.mcmc.AmwgSampler(models.PARAMS_NORM, models.norm_post_readme(pkg.ld), x, dict({"seed": 31}, **opts))


def test_resharding_resumes_bit_for_bit(gpu_pkg):
    x = config2_data().tolist()
    total = 8229
    after = [("sample", 30), ("burn", 50), ("sample", 20)]
    with env(AMWG_JIT="1"):                           # every handle size runs the specialised statistics sweep
        whole = _norm(gpu_pkg, x, chains=total)
        halves = [_norm(gpu_pkg, x, chains=n, first_chain=f) for f, n in ((0, 3000), (3000, total - 3000))]
        for s in [whole] + halves:
            s.burn(75)
        img_whole = whole.checkpoint()
        imgs = [h.checkpoint() for h in halves]
        joined = _norm(gpu_pkg, x, chains=total, seed=5)
        joined.restore(imgs)
        thirds = [_norm(gpu_pkg, x, chains=n, first_chain=f, seed=6) for f, n in ((0, 1000), (1000, 4321), (5321, total - 5321))]
        for t in thirds:
            t.restore(img_whole)
    assert all(s.jit_status()[0] and "specialised sweep" in s.jit_status()[1] for s in [whole, joined] + thirds), whole.jit_status()
    want = _do(whole, after)
    _bits_equal(_do(joined, after), want, "two images into one handle")
    got = [_do(t, after) for t in thirds]
    for k in ("state", "log_post"):
        cat = {n: np.concatenate([np.asarray(g[k][n]) for g in got]) for n in want[k]} if k == "state" else np.concatenate([g[k] for g in got])
        _bits_equal(cat, want[k], "one image into three handles: " + k)
    for r in range(2):
        for n in ("mu", "sigma"):
            _bits_equal(np.concatenate([g["draws"][r][n] for g in got], axis=1), want["draws"][r][n], "draws %d %s" % (r, n))


def test_full_program_model_reshards_across_the_specialisation_threshold(gpu_pkg):
    """Full-program models take the same bits on the specialised sweep (>= 4096 chains by default) and the interpreter: one 5000-chain
    handle's image continues in two handles below the threshold."""
    mcmc, ld = gpu_pkg.mcmc, gpu_pkg.ld
    y = {"x": config3_data().tolist()}
    params, lp = models.PARAMS_SPIKE, models.spike_bern(ld, mcmc)
    whole = mcmc.AmwgSampler(params, lp, y, {"chains": 5000, "seed": 8})
    whole.burn(75)
    img = whole.checkpoint()
    parts = [mcmc.AmwgSampler(params, lp, y, {"chains": n, "first_chain": f, "seed": 9}) for f, n in ((0, 2500), (2500, 2500))]
    for p in parts:
        p.restore(img)
    assert whole.jit_status()[0] and "full-program" in whole.jit_status()[1] and not any(p.jit_status()[0] for p in parts)
    after = [("sample", 30), ("burn", 50), ("sample", 20)]
    want = _do(whole, after)
    got = [_do(p, after) for p in parts]
    for r in range(2):
        for n in ("theta", "m"):
            _bits_equal(np.concatenate([g["draws"][r][n] for g in got], axis=1), want["draws"][r][n], "draws %d %s" % (r, n))
    _bits_equal(np.concatenate([g["log_post"] for g in got]), want["log_post"], "log_post")


JS_NORM = r"""
var readme_norm_post = function(state, data) {
  var log_post = 0;
  log_post += ld.norm(state.mu, 0, 100);
  log_post += ld.unif(state.sigma, 0, 100);
  for(var i = 0; i < data.length; i++) {
    log_post += ld.norm(data[i], state.mu, state.sigma);
  }
  return log_post;
};
"""


def test_images_move_between_the_python_and_javascript_hosts(gpu_pkg):
    from js_host import JsHost, to_py
    from js_native_checkpoint import CheckpointDeviceNative, as_image, image_of
    from oracle.minijs.minijs import to_js
    h = JsHost(native=CheckpointDeviceNative(gpu_pkg))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.it.set_global("ld", h.load("distributions"))
    h.run(JS_NORM)
    x = config2_data()
    h.it.set_global("the_data", to_js(h.it, [float(v) for v in x]))
    Cn = 512
    with env(AMWG_JIT="1"):
        py = _norm(gpu_pkg, x.tolist(), chains=Cn, seed=4)
        py.burn(75)
        h.it.set_global("py_image", as_image(h.it, py.checkpoint()))
        h.run("""
          var S = new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, readme_norm_post, the_data, {chains: 512, seed: 99});
          S.restore(py_image);
          var s_seed = S.model.seed;
          var d1 = S.sample(20);
          var T = new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, readme_norm_post, the_data, {chains: 512, seed: 4});
          T.burn(75);
          var t_image = T.checkpoint();
          T.burn(10);
          var d2 = T.sample(20);
        """)
        p1 = py.sample(20)
        q = _norm(gpu_pkg, x.tolist(), chains=Cn, seed=123)
        q.restore(image_of(h.get("t_image")))
        q.burn(10)
        p2 = q.sample(20)
    assert h.get("s_seed") == 4.0
    for js, pd in ((to_py(h.get("d1")), p1), (to_py(h.get("d2")), p2)):
        for k in ("mu", "sigma"):
            _bits_equal(np.asarray(js[k], np.float64), np.asarray(pd[k], np.float64), k)


def test_refused_restores_leave_the_handle_unchanged(gpu_pkg):
    mcmc = gpu_pkg.mcmc
    params, lp, data, opts, envs, _check = _case(gpu_pkg, "term_cache")
    s = mcmc.AmwgSampler(params, lp, data, dict(opts))
    twin = mcmc.AmwgSampler(params, lp, data, dict(opts))
    for h in (s, twin):
        h.burn(75)
    other = mcmc.AmwgSampler(params, lp, dict(data, x=[6] + list(data["x"][1:])), dict(opts))       # one data value differs
    src = mcmc.AmwgSampler(params, lp, data, dict(opts, seed=50))
    src.burn(20)
    good = src.checkpoint()
    part = mcmc.AmwgSampler(params, lp, data, dict(opts, chains=100))
    part.burn(20)
    D, Cn = s.n_comp, opts["chains"]
    perm_off = 56 + 24 * D + 16 * D * Cn
    bad_perm = bytearray(good)
    bad_perm[perm_off + 8 * 17: perm_off + 8 * 18] = (0).to_bytes(8, "little")
    bad_perm = bytes(bad_perm[:-8]) + ckpt_ref.checksum(bytes(bad_perm[:-8])).to_bytes(8, "little")
    damaged = bytearray(good)
    damaged[1000] ^= 4
    cases = [(other.checkpoint(), "restore: the image was taken with a different model, data or options"),
             (part.checkpoint(), "restore: chains [100, %d) are not covered by the images" % Cn),
             (bytes(damaged), "restore: the image is damaged (checksum mismatch)"),
             (bad_perm, "restore: chain 17 has an invalid substepper order")]
    for img, msg in cases:
        with pytest.raises(mcmc.JsThrow) as e:
            s.restore(img)
        assert str(e.value) == msg
    assert s.seed == twin.seed
    after = [("sample", 40), ("burn", 60), ("sample", 10)]
    _bits_equal(_do(s, after), _do(twin, after), "after refusals")


def test_round_trip_at_config2_size(gpu_pkg):
    """2^20 chains, the headline model (BASELINE config 2): the image is 58.7 MB."""
    x = config2_data().tolist()
    a = _norm(gpu_pkg, x, chains=1 << 20)
    a.burn(75)
    img = a.checkpoint()
    assert len(img) == 56 + 24 * 2 + (1 << 20) * 56 + 8
    b = _norm(gpu_pkg, x, chains=1 << 20, seed=2)
    b.restore([memoryview(img)])
    assert a.jit_status()[0] and len({h.jit_status()[1].replace(" (cubin from the disk cache)", "") for h in (a, b)}) == 1
    after = [("burn", 25), ("sample", 4)]
    _bits_equal(_do(b, after), _do(a, after), "config 2")
