"""Hardware harness scripts that compare the engine with the CPU oracle (run on a GPU machine by hand)."""
