//go:build b200

package kzg_test

import (
	"crypto/sha256"
	"math/big"
	"testing"

	bls12381 "github.com/consensys/gnark-crypto/ecc/bls12-381"
	frbls "github.com/consensys/gnark-crypto/ecc/bls12-381/fr"
	kzgbls "github.com/consensys/gnark-crypto/ecc/bls12-381/kzg"
	"github.com/consensys/gnark-crypto/ecc/bn254"
	frbn "github.com/consensys/gnark-crypto/ecc/bn254/fr"
	kzgbn "github.com/consensys/gnark-crypto/ecc/bn254/kzg"
	b200kzgbls "github.com/consensys/gnark/backend/accelerated/b200/kzg/bls12-381"
	b200kzgbn "github.com/consensys/gnark/backend/accelerated/b200/kzg/bn254"
)

// Commitments, openings (one and a batch, a zero point among them) and a batch opening at one point on a small SRS:
// every result is checked with gnark-crypto's own verifier, and every commitment equals gnark-crypto's kzg.Commit.
func TestDeviceKeyBN254(t *testing.T) {
	srs, err := kzgbn.NewSRS(300, big.NewInt(-1))
	if err != nil {
		t.Fatal(err)
	}
	key, err := b200kzgbn.NewDeviceKey(srs.Pk)
	if err != nil {
		t.Fatal(err)
	}
	defer key.Free()
	ps := make([][]frbn.Element, 5)
	points := make([]frbn.Element, len(ps))
	for i := range ps {
		ps[i] = make([]frbn.Element, 100+40*i)
		for j := range ps[i] {
			ps[i][j].SetRandom()
		}
		if i != 2 {
			points[i].SetRandom()
		}
	}
	digests, err := key.CommitBatch(ps)
	if err != nil {
		t.Fatal(err)
	}
	for i := range ps {
		want, err := kzgbn.Commit(ps[i], srs.Pk)
		if err != nil {
			t.Fatal(err)
		}
		if !want.Equal(&digests[i]) {
			t.Fatalf("commitment %d differs from kzg.Commit", i)
		}
		one, err := key.Commit(ps[i])
		if err != nil || !one.Equal(&digests[i]) {
			t.Fatalf("Commit %d differs from CommitBatch: %v", i, err)
		}
	}
	proofs, err := key.OpenBatch(ps, points)
	if err != nil {
		t.Fatal(err)
	}
	for i := range ps {
		if err := kzgbn.Verify(&digests[i], &proofs[i], points[i], srs.Vk); err != nil {
			t.Fatalf("opening %d: %v", i, err)
		}
	}
	single, err := key.Open(ps[0], points[0])
	if err != nil || kzgbn.Verify(&digests[0], &single, points[0], srs.Vk) != nil {
		t.Fatalf("Open: %v", err)
	}
	batch, err := key.BatchOpenSinglePoint(ps, digests, points[0], sha256.New(), []byte("data"))
	if err != nil {
		t.Fatal(err)
	}
	if err := kzgbn.BatchVerifySinglePoint(digests, &batch, points[0], sha256.New(), srs.Vk, []byte("data")); err != nil {
		t.Fatal(err)
	}
	if _, err := key.Commit(make([]frbn.Element, 301)); err == nil {
		t.Fatal("a polynomial longer than the SRS was committed")
	}
	if _, err := key.BatchOpenSinglePoint(ps, digests[:4], points[0], sha256.New()); err == nil {
		t.Fatal("BatchOpenSinglePoint accepted fewer digests than polynomials")
	}
	_ = bn254.G1Affine{}
}

// The same on BLS12-381 with a larger batch.
func TestDeviceKeyBLS12381(t *testing.T) {
	srs, err := kzgbls.NewSRS(1<<12, big.NewInt(-1))
	if err != nil {
		t.Fatal(err)
	}
	key, err := b200kzgbls.NewDeviceKey(srs.Pk)
	if err != nil {
		t.Fatal(err)
	}
	defer key.Free()
	ps := make([][]frbls.Element, 16)
	points := make([]frbls.Element, len(ps))
	for i := range ps {
		ps[i] = make([]frbls.Element, 1<<12)
		for j := range ps[i] {
			ps[i][j].SetRandom()
		}
		points[i].SetRandom()
	}
	digests, err := key.CommitBatch(ps)
	if err != nil {
		t.Fatal(err)
	}
	proofs, err := key.OpenBatch(ps, points)
	if err != nil {
		t.Fatal(err)
	}
	for i := range ps {
		if err := kzgbls.Verify(&digests[i], &proofs[i], points[i], srs.Vk); err != nil {
			t.Fatalf("opening %d: %v", i, err)
		}
	}
	batch, err := key.BatchOpenSinglePoint(ps, digests, points[3], sha256.New())
	if err != nil {
		t.Fatal(err)
	}
	if err := kzgbls.BatchVerifySinglePoint(digests, &batch, points[3], sha256.New(), srs.Vk); err != nil {
		t.Fatal(err)
	}
	_ = bls12381.G1Affine{}
}
