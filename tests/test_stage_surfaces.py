"""CPU tier: the pipeline-stage range on the public surfaces — manifest schema (models[].layers), `kuke model plan --layers` and the pool
registry's Entry."""
import io
import json
import os

import pytest

from kukeon_b200 import cli, registry, schema
from kukeon_b200.schema import Err, SchemaError, validate_models
from tools import synth


def _ok(p):
    return None


def test_layers_accepted_and_carried_on_the_spec():
    specs = validate_models([{"name": "a", "source": "/m", "layers": [0, 16]}, {"name": "b", "source": "/m", "layers": [16, 32]},
                             {"name": "c", "source": "/m"}], stat=_ok)
    assert [s.layers for s in specs] == [(0, 16), (16, 32), None]


@pytest.mark.parametrize("bad", [[4, 4], [5, 2], [-1, 3], [0], [0, 1, 2], [True, 3], [0, False], [0.0, 2], ["0", "2"], "0:2", 7, {"b": 0}, [0, 2**32]])
def test_layers_rejections_carry_the_sentinel(bad):
    with pytest.raises(SchemaError) as e:
        validate_models([{"name": "a", "source": "/m", "devices": [0], "layers": bad}], stat=_ok)
    assert e.value.sentinel == Err.ModelLayersInvalid
    assert str(e.value).endswith(f"(model[0] layers {bad!r})")


def test_layers_are_checked_after_devices():
    with pytest.raises(SchemaError) as e:
        validate_models([{"name": "a", "source": "/m", "devices": [0, 0], "layers": [3, 1]}], stat=_ok)
    assert e.value.sentinel == Err.ModelDevicesInvalid
    with pytest.raises(SchemaError) as e:
        validate_models([{"name": "a", "source": "/m", "layers": [3, 1], "options": {"nope": True}}], stat=_ok)
    assert e.value.sentinel == Err.ModelLayersInvalid


@pytest.fixture(scope="module")
def gguf(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("plan") / "mixtral.gguf")
    synth.write_gguf(p, synth.mixtral_gguf_tensors(hidden=256, ffn=512, layers=4, experts=2, vocab=320, kv_dim=128), 5)
    return p


def run(argv):
    out = io.StringIO()
    rc = cli.main(argv, out)
    return rc, out.getvalue()


def test_model_plan_layers_table_and_json(gguf, capsys):
    rc, whole = run(["model", "plan", gguf, "-o", "json"])
    assert rc == 0
    whole = json.loads(whole)
    assert "layers" not in whole and "nLayers" not in whole
    stages = []
    for b, e in ((0, 2), (2, 4)):
        rc, txt = run(["model", "plan", gguf, "--layers", f"{b}:{e}", "-o", "json"])
        assert rc == 0
        doc = json.loads(txt)
        assert doc["layers"] == [b, e] and doc["nLayers"] == 4
        stages.append(doc)
    assert stages[0]["fileBytes"] + stages[1]["fileBytes"] == whole["fileBytes"]  # no tied embedding and no every-stage tensor here
    assert stages[0]["tensors"] + stages[1]["tensors"] == whole["tensors"]
    assert max(s["poolBytesPerGpu"][0] for s in stages) < whole["poolBytesPerGpu"][0]
    rc, txt = run(["model", "plan", gguf, "--layers", "2:4", "--mode", "broadcast", "--gpus", "2"])
    assert rc == 0
    assert txt.splitlines()[0].split() == ["GPU", "INGESTS", "POOL"] and len(txt.splitlines()) == 4
    assert txt.rstrip().endswith("mode broadcast, layers 2-3 of 4")
    rc, txt = run(["model", "plan", gguf, "--layers", "0:2", "-o", "yaml"])
    assert rc == 0 and "nLayers: 4" in txt and "layers:\n- 0\n- 2" in txt
    rc, txt = run(["model", "plan", gguf, "--layers", "0:2", "-o", "json", "--full"])
    assert rc == 0 and json.loads(txt)["layers"] == [0, 2] and json.loads(txt)["n_layers"] == 4
    # out of range: the library's error, exit 1
    rc, _ = run(["model", "plan", gguf, "--layers", "2:5"])
    assert rc == 1 and "4 layers" in capsys.readouterr().err
    for bad in ("3:3", "4:2", "2", "a:b", "-1:2", ":3"):
        with pytest.raises(SystemExit) as e:
            run(["model", "plan", gguf, "--layers", bad])
        assert e.value.code == 2


def test_registry_entry_round_trip_with_and_without_a_range(tmp_path):
    run_path = str(tmp_path / "run")
    shard = tmp_path / "m.gguf"
    shard.write_bytes(b"x" * 10)
    r = registry.PoolRegistry(run_path, epoch="boot:1:1")
    r.reconcile()
    r.record("whole", "/models/m", 0, 10, 256, [0], [str(shard)])
    r.record("stage1", "/models/m", 0, 5, 256, [1], [str(shard)], layers=(16, 32))
    doc = json.load(open(os.path.join(run_path, registry.FILE_NAME)))
    by_key = {m["key"]: m for m in doc["models"]}
    assert "layers" not in by_key["whole"], "a whole-checkpoint entry is written as before"
    assert by_key["stage1"]["layers"] == [16, 32]
    # a restarted daemon gets the stage back, so it reloads [16, 32) and not the whole model
    stale = {e.key: e for e in registry.PoolRegistry(run_path, epoch="boot:2:2").reconcile()}
    assert stale["stage1"].layers == [16, 32] and stale["whole"].layers is None
    assert registry.Entry.from_json(stale["stage1"].to_json()) == stale["stage1"]
    assert registry.Entry.from_json(stale["whole"].to_json()) == stale["whole"]
