"""CPU oracle for the IGMC hot path — TEST INFRASTRUCTURE ONLY.

Nothing in the shipped package ``igmc_b200`` may import this package.  Only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs use it, and only as the checker / the timed CPU arm.

Contents
--------
ref_shim        imports the *unmodified* reference ``util_functions.py`` from
                oracle/_ref/ (built by ``make_ref.py``) to pin ``extract_np``
                and to generate ``tests/golden``.
extract_np      numpy restatement of ``subgraph_extraction_labeling`` +
                ``construct_pyg_graph`` + PyG collate, in canonical form.
pyg_restated    pure-torch restatement of PyG 1.4.2 ``RGCNConv`` / ``dropout_adj``
                / ``IGMC.forward`` / the train-step loss (PARITY UNPINNED: PyG is
                not installable here and the reference ships no tests).
"""
