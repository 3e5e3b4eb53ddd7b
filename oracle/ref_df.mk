# oracle/ref_df.mk -- builds the DarkForest-plane search shim (test-only checker) on top of Makefile's
# reference libraries:
#   make -f ref_df.mk ref_df : oracle/_ref/libref_mcts_df{19,9}.so from ref_mcts_df_shim.cc, linked against
#                              oracle/_ref/libref_go{19,9}.so (found next to it at run time)
include Makefile

.PHONY: ref_df
ref_df: $(OUT)/libref_mcts_df19.so $(OUT)/libref_mcts_df9.so

$(OUT)/libref_mcts_df19.so: ref_mcts_df_shim.cc $(OUT)/libref_go19.so
	g++ $(CXXFLAGS) $(INC) -shared -o $@ ref_mcts_df_shim.cc -L$(OUT) -lref_go19 -Wl,-rpath,'$$ORIGIN'

$(OUT)/libref_mcts_df9.so: ref_mcts_df_shim.cc $(OUT)/libref_go9.so
	g++ $(CXXFLAGS) -DBOARD9x9 $(INC) -shared -o $@ ref_mcts_df_shim.cc -L$(OUT) -lref_go9 -Wl,-rpath,'$$ORIGIN'
