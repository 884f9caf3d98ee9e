"""Writes suggest_shard.json: the three resources of the reference's nidx_tests/src/lib.rs that tests/integration/suggest.rs indexes
(little_prince, thus_spoke_zarathustra, people_and_places), as data: per resource its labels, text fields, paragraphs (field, start,
end) and relations (field, source, relation type, target as (value, type, subtype)).  Resource ids are fixed here (the reference draws
them at random).  Usage: python make_suggest_shard.py"""
import json
import os

ENTITY, LABEL, RESOURCE, USER = 0, 1, 2, 3            # utils.RelationNode.NodeType
COLAB_REL, ENTITY_REL = 3, 2                          # utils.Relation.RelationType

LITTLE_PRINCE = "0b7a5bd2c6d04b1e9b6f8a9c1d2e3f40"
ZARATHUSTRA = "1c8b6ce3d7e15c2fa07f9bad2e3f4051"
PEOPLE_AND_PLACES = "2d9c7df4e8f26d30b1809cbe3f405162"

SUMMARY = ("The story follows a young prince who visits various planets in space, including Earth, and addresses themes of loneliness, "
           "friendship, love, and loss.")


def resources():
    pap_nodes = [("Anastasia", USER, "", COLAB_REL), ("Irene", USER, "", COLAB_REL)]
    pap_nodes += [(p, ENTITY, "person", ENTITY_REL) for p in ("Anna", "Anthony", "Bárcenas", "Ben", "John")]
    pap_nodes += [(c, ENTITY, "city", ENTITY_REL) for c in ("Barcelona", "New York", "York")]
    pap_nodes += [(c, ENTITY, "country", ENTITY_REL) for c in ("Israel", "Netherlands", "Solomon Islands")]
    return [
        {"name": "little prince", "uuid": LITTLE_PRINCE, "labels": ["/s/p/en"],
         "texts": {"a/title": "The little prince", "a/summary": SUMMARY},
         "paragraphs": [["a/title", 0, 17], ["a/summary", 0, 150]], "relations": []},
        {"name": "zarathustra", "uuid": ZARATHUSTRA, "labels": ["/s/p/de"],
         "texts": {"a/title": "Thus Spoke Zarathustra", "a/summary": "Philosophical book written by Frederich Nietzche"},
         "paragraphs": [["a/title", 0, 22], ["a/summary", 0, 48]], "relations": []},
        {"name": "pap", "uuid": PEOPLE_AND_PLACES, "labels": [],
         "texts": {f"{PEOPLE_AND_PLACES}/title": "People and places",
                   f"{PEOPLE_AND_PLACES}/summary": "Test entities to validate suggest on relations index"},
         "paragraphs": [],
         "relations": [["a/metadata", [PEOPLE_AND_PLACES, RESOURCE, ""], rel, [v, t, s]] for v, t, s, rel in pap_nodes]},
    ]


if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "suggest_shard.json"), "w") as f:
        json.dump({"resources": resources()}, f, indent=1, ensure_ascii=False)
        f.write("\n")
