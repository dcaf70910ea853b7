// The variables behind b200mol_set_option / b200mol_get_option (the table in options.cu). Each is defined in the file
// whose code it steers, next to the reasons for its default; include/b200mol.h documents the keys.
#pragma once

namespace b200 {

// similarity passes (options.cu, tanimoto_tc.cu)
extern long long          g_tensorMinPairs;
extern int                g_tensorCluster;
extern int                g_superpose;
extern int                g_superposeCols;
extern int                g_superposeAuto;
extern int                g_pipelineChunks;
extern int                g_popcountBand;
extern int                g_superposeLast;
extern unsigned long long g_candidatesLast;
extern unsigned long long g_unitsPlanned;
// top-k search (topk.cu)
extern long long          g_topkSlabCols;
extern unsigned long long g_topkSlabsLast;
// MaxMin picking (maxmin.cu)
extern int                g_maxminMode;
extern long long          g_maxminResidentRows;
extern int                g_maxminResidentLast;
// Leader picking (leader.cu)
extern long long          g_leaderWindowRows;
extern long long          g_leaderWindowsLast;
extern unsigned long long g_leaderBulkPairsLast;
// conformer RMSD matrices (conformer_rmsd.cu)
extern long long g_rmsdMatchChunk;
extern long long g_rmsdMatchChunksLast;
// Morgan fingerprints (morgan.cu)
extern long long g_morganGlobalSlabLast;
// Butina clustering (butina.cu)
extern int g_butinaMinCommits;
// minimiser and embedder (bfgs.cu, etkdg.cu)
extern int g_bfgsCtasPerSm;
extern int g_bfgsL2Persist;
extern int g_etkdgHessianFp64;

// Word i of a file's device statistics counters, as the last call left them (synchronises the device).
unsigned long long readWalkCounter(int i);  // tanimoto_tc.cu: [0] units, [1] tiles the count passes walked
unsigned long long readTopkStat(int i);     // topk.cu: [0] candidates listed, [1] rows redone
unsigned long long readMaxminStat(int i);   // maxmin.cu: [0] distances evaluated, [1] skipped by the popcount bound
unsigned long long readLeaderStat(int i);   // leader.cu: [0] pairs compared in a window, [1] in a block
unsigned long long readCountStat(int i);    // count_similarity.cu: [0] pairs the neighbour pass compared

}  // namespace b200
